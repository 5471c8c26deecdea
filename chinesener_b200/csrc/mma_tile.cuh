// Warp-level tensor-core tiles of the head-dim-64 kernels (attention.cu, attention_bwd.cu, global_pointer.cu):
// mma.sync.m16n8k16 (bf16 in, fp32 accumulate) on operands staged in shared memory as [rows][PITCH] bf16 matrices.
// A warp owns 16 rows; its accumulator is a 16 x 64 tile in C-fragment layout, float[8][4] (8 n-tiles of 8 columns).
#pragma once
#include "common.cuh"

namespace mma_tile {

using nerdev::smem_u32;

constexpr int D = 64;         // head dim: the k extent of A . B^T and the column count of P . B
constexpr int PITCH = D + 8;  // bf16 per smem row (144 B): conflict-free fragment loads / ldmatrix

__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldsm_x2_trans(uint32_t& r0, uint32_t& r1, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(smem_u32(p)));
}
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ uint32_t lds32(const __nv_bfloat16* p) { return *reinterpret_cast<const uint32_t*>(p); }

__device__ __forceinline__ void clear_tile(float (&acc)[8][4]) {
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
}

// A-operand fragments (16 rows x 64 k) of rows r0 / r0 + 8 of a [rows][PITCH] smem matrix
__device__ __forceinline__ void load_a_frags(uint32_t (&a)[4][4], const __nv_bfloat16* base, int r0, int cq) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    a[ks][0] = lds32(base + r0 * PITCH + ks * 16 + cq);
    a[ks][1] = lds32(base + (r0 + 8) * PITCH + ks * 16 + cq);
    a[ks][2] = lds32(base + r0 * PITCH + ks * 16 + 8 + cq);
    a[ks][3] = lds32(base + (r0 + 8) * PITCH + ks * 16 + 8 + cq);
  }
}
// acc[nt] (16 x 64 cols in 8 n-tiles) += A(16 x 64) . Bm[n0 .. n0+64]^T, Bm a [cols][PITCH] smem matrix (rows = n index)
__device__ __forceinline__ void mma_a_bt(float (&acc)[8][4], const uint32_t (&a)[4][4], const __nv_bfloat16* Bm, int n0,
                                         int lane, int cq) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const __nv_bfloat16* p = Bm + (n0 + nt * 8 + (lane >> 2)) * PITCH + ks * 16 + cq;
      mma16816(acc[nt], a[ks], lds32(p), lds32(p + 8));
    }
}
// out[dt] (16 x 64 dims) += P(16 x 64, C-fragment layout in p) . Bm[n0 .. n0+64][dims]
__device__ __forceinline__ void mma_p_b(float (&out)[8][4], const float (&p)[8][4], const __nv_bfloat16* Bm, int n0,
                                        int lane) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    uint32_t pa[4];
    pa[0] = pack2(p[2 * kk][0], p[2 * kk][1]);
    pa[1] = pack2(p[2 * kk][2], p[2 * kk][3]);
    pa[2] = pack2(p[2 * kk + 1][0], p[2 * kk + 1][1]);
    pa[3] = pack2(p[2 * kk + 1][2], p[2 * kk + 1][3]);
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
      uint32_t b0, b1;
      ldsm_x2_trans(b0, b1, Bm + (n0 + kk * 16 + (lane & 15)) * PITCH + dt * 8);
      mma16816(out[dt], pa, b0, b1);
    }
  }
}

}  // namespace mma_tile
