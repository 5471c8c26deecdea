// Backward of the BERT self-attention core (sm_90a), head_dim 64, padded layout:
//   given qkv (bf16 [B*L, 3*NH*64]), the forward context O (bf16) and dO (bf16), produce
//   d_qkv (bf16, same layout as qkv).  This is the gradient tf.gradients derives through
//   attention_layer() of bert_base.bert.modeling (reference tools/train_utils.py:314).
//
// Up to L = 384: one CTA per (batch row, head).  Q, K, V and dO of the head are staged once in shared memory;
// nothing of size L x L is ever written anywhere: the scores are recomputed from Q/K with warp-level
// mma.sync.m16n8k16 (bf16 in, fp32 accumulate), flash-attention style, in two phases.
//   phase A (a warp owns 16 query rows):  row max / 1/sum / D = rowsum(dO*O), then
//           dS = P o (dO V^T - D),  dQ = scale * dS K                       (no cross-warp reduction)
//   phase B (a warp owns 16 key rows):    S^T = K Q^T so keys are the accumulator rows,
//           dV = P^T dO,  dK = scale * dS^T Q                               (no cross-warp reduction)
// Longer sequences, where the head does not fit in shared memory, take the key-tiled kernels further down.
#include "common.cuh"
#include "mma_tile.cuh"

namespace {

using namespace nerdev;
using namespace mma_tile;

constexpr int NW = 8;  // warps per CTA

// Same attention_probs dropout factor as the forward kernel (attention.cu): z in {0, 1/keep}.
// With O = (P o z) V:  dV = (P o z)^T dO,  dS = P o (z o dP - D),  D = rowsum(dO o O) unchanged.
__device__ __forceinline__ float attn_drop(uint32_t sa, uint32_t sb, int q, int k, uint32_t thr, float inv_keep) {
  return hash3(sa, (uint32_t)q, (uint32_t)k ^ sb) < thr ? inv_keep : 0.f;
}

template <bool DROP>
__global__ void __launch_bounds__(NW * 32)
bert_attention_bwd_kernel(const __nv_bfloat16* __restrict__ qkv, const int32_t* __restrict__ mask,
                          const __nv_bfloat16* __restrict__ ctx, const __nv_bfloat16* __restrict__ dctx,
                          __nv_bfloat16* __restrict__ dqkv, int Lpad, int NH, int Lp_max, float scale, float mask_add,
                          const int32_t* __restrict__ cu_seqlens, float keep, uint32_t seed_lo, uint32_t seed_hi) {
  const uint32_t dsa = seed_lo ^ ((uint32_t)(blockIdx.y * NH + blockIdx.x) * 0x9E3779B1u), dthr = keep_threshold(keep);
  const float dik = 1.f / keep;
  // padded mode: rows [b*L, (b+1)*L), keys masked by `mask`; packed mode: rows [cu[b], cu[b+1]), all keys valid and the
  // tile loops stop at the sequence's own length (same convention as the forward kernel, attention.cu)
  const size_t row_base = cu_seqlens ? (size_t)cu_seqlens[blockIdx.y] : (size_t)blockIdx.y * Lpad;
  const int L = cu_seqlens ? (cu_seqlens[blockIdx.y + 1] - cu_seqlens[blockIdx.y]) : Lpad;
  const int Lp = cu_seqlens ? (L + 63) / 64 * 64 : Lp_max;
  if (L == 0) return;
  extern __shared__ __align__(16) uint8_t smraw[];
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(smraw);
  __nv_bfloat16* Ks = Qs + (size_t)Lp * PITCH;
  __nv_bfloat16* Vs = Ks + (size_t)Lp * PITCH;
  __nv_bfloat16* Os = Vs + (size_t)Lp * PITCH;  // dO
  float* s_madd = reinterpret_cast<float*>(Os + (size_t)Lp * PITCH);
  float* s_m = s_madd + Lp;
  float* s_li = s_m + Lp;
  float* s_D = s_li + Lp;

  const int b = blockIdx.y, h = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int HD = NH * D;
  const size_t rs = (size_t)3 * HD;
  const __nv_bfloat16* base = qkv + row_base * rs + h * D;
  const __nv_bfloat16* obase = ctx + row_base * HD + h * D;
  const __nv_bfloat16* dobase = dctx + row_base * HD + h * D;

  for (int idx = tid; idx < Lp * 8; idx += NW * 32) {
    const int row = idx >> 3, ch = idx & 7;
    if (row < L) {
      cp_async16(Qs + row * PITCH + ch * 8, base + (size_t)row * rs + ch * 8);
      cp_async16(Ks + row * PITCH + ch * 8, base + (size_t)row * rs + HD + ch * 8);
      cp_async16(Vs + row * PITCH + ch * 8, base + (size_t)row * rs + 2 * HD + ch * 8);
      cp_async16(Os + row * PITCH + ch * 8, dobase + (size_t)row * HD + ch * 8);
    } else {
      const uint4 z = make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(Qs + row * PITCH + ch * 8) = z;
      *reinterpret_cast<uint4*>(Ks + row * PITCH + ch * 8) = z;
      *reinterpret_cast<uint4*>(Vs + row * PITCH + ch * 8) = z;
      *reinterpret_cast<uint4*>(Os + row * PITCH + ch * 8) = z;
    }
  }
  cp_async_commit();
  for (int k = tid; k < Lp; k += NW * 32) {
    s_madd[k] = (k < L) ? (cu_seqlens ? 0.f : (1.f - (float)mask[(size_t)b * Lpad + k]) * mask_add) : -1e30f;
    s_m[k] = 0.f;
    s_li[k] = 0.f;
    s_D[k] = 0.f;
  }
  cp_async_wait<0>();
  __syncthreads();

  constexpr float kLog2e = 1.4426950408889634f;
  const int cq = 2 * (lane & 3);

  // ------------------------------------------------------------------ phase A: query rows
  for (int qb = warp; qb * 16 < L; qb += NW) {
    const int r0 = qb * 16 + (lane >> 2), r1 = r0 + 8;
    uint32_t qa[4][4], da[4][4];
    load_a_frags(qa, Qs, r0, cq);
    load_a_frags(da, Os, r0, cq);
    // D = rowsum(dO * O)
    float d0 = 0.f, d1 = 0.f;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int col = ks * 16 + hh * 8 + cq;
        const __nv_bfloat162 g0 = *reinterpret_cast<const __nv_bfloat162*>(&da[ks][hh * 2 + 0]);
        const __nv_bfloat162 g1 = *reinterpret_cast<const __nv_bfloat162*>(&da[ks][hh * 2 + 1]);
        if (r0 < L) {
          const __nv_bfloat162 o = *reinterpret_cast<const __nv_bfloat162*>(obase + (size_t)r0 * HD + col);
          d0 += __low2float(g0) * __low2float(o) + __high2float(g0) * __high2float(o);
        }
        if (r1 < L) {
          const __nv_bfloat162 o = *reinterpret_cast<const __nv_bfloat162*>(obase + (size_t)r1 * HD + col);
          d1 += __low2float(g1) * __low2float(o) + __high2float(g1) * __high2float(o);
        }
      }
    d0 += __shfl_xor_sync(0xffffffffu, d0, 1);
    d0 += __shfl_xor_sync(0xffffffffu, d0, 2);
    d1 += __shfl_xor_sync(0xffffffffu, d1, 1);
    d1 += __shfl_xor_sync(0xffffffffu, d1, 2);
    // pass 1: row max and sum
    float m0 = -1e30f, m1 = -1e30f, l0 = 0.f, l1 = 0.f;
    for (int kb = 0; kb < Lp; kb += 64) {
      float s[8][4];
      clear_tile(s);
      mma_a_bt(s, qa, Ks, kb, lane, cq);
      float mx0 = -1e30f, mx1 = -1e30f;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const float a0 = s_madd[kb + nt * 8 + cq], a1 = s_madd[kb + nt * 8 + cq + 1];
        s[nt][0] = s[nt][0] * scale + a0;
        s[nt][1] = s[nt][1] * scale + a1;
        s[nt][2] = s[nt][2] * scale + a0;
        s[nt][3] = s[nt][3] * scale + a1;
        mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
        mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float n0 = fmaxf(m0, mx0), n1 = fmaxf(m1, mx1);
      float p0 = 0.f, p1 = 0.f;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        p0 += exp2f((s[nt][0] - n0) * kLog2e) + exp2f((s[nt][1] - n0) * kLog2e);
        p1 += exp2f((s[nt][2] - n1) * kLog2e) + exp2f((s[nt][3] - n1) * kLog2e);
      }
      l0 = l0 * exp2f((m0 - n0) * kLog2e) + p0;
      l1 = l1 * exp2f((m1 - n1) * kLog2e) + p1;
      m0 = n0;
      m1 = n1;
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float li0 = 1.f / l0, li1 = 1.f / l1;
    if ((lane & 3) == 0) {
      if (r0 < L) { s_m[r0] = m0; s_li[r0] = li0; s_D[r0] = d0; }
      if (r1 < L) { s_m[r1] = m1; s_li[r1] = li1; s_D[r1] = d1; }
    }
    // pass 2: dS and dQ
    float dq[8][4];
    clear_tile(dq);
    for (int kb = 0; kb < Lp; kb += 64) {
      float s[8][4], dp[8][4];
      clear_tile(s);
      clear_tile(dp);
      mma_a_bt(s, qa, Ks, kb, lane, cq);
      mma_a_bt(dp, da, Vs, kb, lane, cq);
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const float a0 = s_madd[kb + nt * 8 + cq], a1 = s_madd[kb + nt * 8 + cq + 1];
        const float p00 = exp2f((s[nt][0] * scale + a0 - m0) * kLog2e) * li0;
        const float p01 = exp2f((s[nt][1] * scale + a1 - m0) * kLog2e) * li0;
        const float p10 = exp2f((s[nt][2] * scale + a0 - m1) * kLog2e) * li1;
        const float p11 = exp2f((s[nt][3] * scale + a1 - m1) * kLog2e) * li1;
        if (DROP) {
          const int k = kb + nt * 8 + cq;
          dp[nt][0] *= attn_drop(dsa, seed_hi, r0, k, dthr, dik);
          dp[nt][1] *= attn_drop(dsa, seed_hi, r0, k + 1, dthr, dik);
          dp[nt][2] *= attn_drop(dsa, seed_hi, r1, k, dthr, dik);
          dp[nt][3] *= attn_drop(dsa, seed_hi, r1, k + 1, dthr, dik);
        }
        s[nt][0] = p00 * (dp[nt][0] - d0);
        s[nt][1] = p01 * (dp[nt][1] - d0);
        s[nt][2] = p10 * (dp[nt][2] - d1);
        s[nt][3] = p11 * (dp[nt][3] - d1);
      }
      mma_p_b(dq, s, Ks, kb, lane);
    }
    __nv_bfloat16* dqb = dqkv + row_base * rs + h * D;
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
      if (r0 < L) *reinterpret_cast<uint32_t*>(dqb + (size_t)r0 * rs + dt * 8 + cq) = pack2(dq[dt][0] * scale, dq[dt][1] * scale);
      if (r1 < L) *reinterpret_cast<uint32_t*>(dqb + (size_t)r1 * rs + dt * 8 + cq) = pack2(dq[dt][2] * scale, dq[dt][3] * scale);
    }
  }
  __syncthreads();

  // ------------------------------------------------------------------ phase B: key rows
  for (int kb16 = warp; kb16 * 16 < L; kb16 += NW) {
    const int k0 = kb16 * 16 + (lane >> 2), k1 = k0 + 8;
    uint32_t ka[4][4], va[4][4];
    load_a_frags(ka, Ks, k0, cq);
    load_a_frags(va, Vs, k0, cq);
    const float ma0 = s_madd[k0], ma1 = s_madd[k1];
    float dk[8][4], dv[8][4];
    clear_tile(dk);
    clear_tile(dv);
    for (int qb = 0; qb < Lp; qb += 64) {
      float st[8][4], dpt[8][4];
      clear_tile(st);
      clear_tile(dpt);
      mma_a_bt(st, ka, Qs, qb, lane, cq);   // S^T  = K Q^T      (rows: keys, cols: queries)
      mma_a_bt(dpt, va, Os, qb, lane, cq);  // dP^T = V dO^T
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int q0 = qb + nt * 8 + cq, q1 = q0 + 1;
        const float mq0 = s_m[q0], mq1 = s_m[q1], lq0 = s_li[q0], lq1 = s_li[q1], dq0 = s_D[q0], dq1 = s_D[q1];
        const float p00 = exp2f((st[nt][0] * scale + ma0 - mq0) * kLog2e) * lq0;
        const float p01 = exp2f((st[nt][1] * scale + ma0 - mq1) * kLog2e) * lq1;
        const float p10 = exp2f((st[nt][2] * scale + ma1 - mq0) * kLog2e) * lq0;
        const float p11 = exp2f((st[nt][3] * scale + ma1 - mq1) * kLog2e) * lq1;
        float z00 = 1.f, z01 = 1.f, z10 = 1.f, z11 = 1.f;
        if (DROP) {
          z00 = attn_drop(dsa, seed_hi, q0, k0, dthr, dik);
          z01 = attn_drop(dsa, seed_hi, q1, k0, dthr, dik);
          z10 = attn_drop(dsa, seed_hi, q0, k1, dthr, dik);
          z11 = attn_drop(dsa, seed_hi, q1, k1, dthr, dik);
        }
        st[nt][0] = p00 * z00;
        st[nt][1] = p01 * z01;
        st[nt][2] = p10 * z10;
        st[nt][3] = p11 * z11;
        dpt[nt][0] = p00 * (z00 * dpt[nt][0] - dq0);
        dpt[nt][1] = p01 * (z01 * dpt[nt][1] - dq1);
        dpt[nt][2] = p10 * (z10 * dpt[nt][2] - dq0);
        dpt[nt][3] = p11 * (z11 * dpt[nt][3] - dq1);
      }
      mma_p_b(dv, st, Os, qb, lane);   // dV += P^T dO
      mma_p_b(dk, dpt, Qs, qb, lane);  // dK += dS^T Q
    }
    __nv_bfloat16* dkb = dqkv + row_base * rs + HD + h * D;
    __nv_bfloat16* dvb = dqkv + row_base * rs + 2 * HD + h * D;
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
      if (k0 < L) {
        *reinterpret_cast<uint32_t*>(dkb + (size_t)k0 * rs + dt * 8 + cq) = pack2(dk[dt][0] * scale, dk[dt][1] * scale);
        *reinterpret_cast<uint32_t*>(dvb + (size_t)k0 * rs + dt * 8 + cq) = pack2(dv[dt][0], dv[dt][1]);
      }
      if (k1 < L) {
        *reinterpret_cast<uint32_t*>(dkb + (size_t)k1 * rs + dt * 8 + cq) = pack2(dk[dt][2] * scale, dk[dt][3] * scale);
        *reinterpret_cast<uint32_t*>(dvb + (size_t)k1 * rs + dt * 8 + cq) = pack2(dv[dt][2], dv[dt][3]);
      }
    }
  }
}

// ------------------------------------------------------------------ key-tiled backward (sequences too long for the kernel above)
// Three launches in stream order, each CTA owning one 64-row tile of one (sequence, head), 4 warps x 16 rows; the other
// operand streams through a cp.async double buffer, so shared memory does not depend on L:
//   stats  (per query tile, streams K):      lse = m + log(sum exp), D = rowsum(dO o O), stored as fp32 (lse, D) in the
//                                            first 8 bytes of the row's dQ slot in d_qkv
//   dK/dV  (per key tile, streams Q, dO):    phase B above, P rebuilt from the stored lse, D read back
//   dQ     (per query tile, streams K, V):   phase A pass 2 above; reads its rows' statistics, then overwrites the slot
// Every output slot is written by exactly one CTA of one launch: no atomics, no workspace, repeat calls are bit-identical.
// Needs d_qkv not to alias qkv / ctx / dctx.
constexpr int TQ = 64;  // rows per tile
constexpr int TW = 4;   // warps per CTA
constexpr int TILE = TQ * PITCH;
constexpr size_t KV_SMEM = (size_t)6 * TILE * 2 + (size_t)2 * TQ * 8;  // K, V + 2 x (Q, dO) + 2 x stats
constexpr size_t DQ_SMEM = (size_t)6 * TILE * 2 + (size_t)2 * TQ * 4;  // Q, dO + 2 x (K, V) + 2 x key mask terms

__device__ __forceinline__ void cp_async8(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(smem_u32(smem)), "l"(gmem));
}
// rows [row0, row0 + 64) of a row-major bf16 matrix (64 columns used, row stride `stride`) -> [64][PITCH] smem, zero past L
__device__ __forceinline__ void tile_async(__nv_bfloat16* dst, const __nv_bfloat16* src, size_t stride, int row0, int L,
                                           int tid) {
#pragma unroll
  for (int i = 0; i < TQ * 8 / (TW * 32); ++i) {
    const int idx = tid + i * TW * 32, r = idx >> 3, ch = idx & 7;
    if (row0 + r < L)
      cp_async16(dst + r * PITCH + ch * 8, src + (size_t)(row0 + r) * stride + ch * 8);
    else
      *reinterpret_cast<uint4*>(dst + r * PITCH + ch * 8) = make_uint4(0, 0, 0, 0);
  }
}
// additive score term of key k: mask_add on padded [PAD] keys, 0 on valid keys, -1e30 past the sequence
__device__ __forceinline__ float key_add(const int32_t* mask, const int32_t* cu_seqlens, int b, int Lpad, int L, int k,
                                         float mask_add) {
  if (k >= L) return -1e30f;
  return cu_seqlens ? 0.f : (1.f - (float)mask[(size_t)b * Lpad + k]) * mask_add;
}
__device__ __forceinline__ void stage_key_add(float* dst, const int32_t* mask, const int32_t* cu_seqlens, int b, int Lpad,
                                              int L, int k0, float mask_add, int tid) {
  if (tid < TQ) dst[tid] = key_add(mask, cu_seqlens, b, Lpad, L, k0 + tid, mask_add);
}

__global__ void __launch_bounds__(TW * 32)
bert_attention_bwd_stats_kernel(const __nv_bfloat16* __restrict__ qkv, const int32_t* __restrict__ mask,
                                const __nv_bfloat16* __restrict__ ctx, const __nv_bfloat16* __restrict__ dctx,
                                __nv_bfloat16* __restrict__ dqkv, int Lpad, int NH, float scale, float mask_add,
                                const int32_t* __restrict__ cu_seqlens) {
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * TQ;
  const size_t row_base = cu_seqlens ? (size_t)cu_seqlens[b] : (size_t)b * Lpad;
  const int L = cu_seqlens ? (cu_seqlens[b + 1] - cu_seqlens[b]) : Lpad;
  if (q0 >= L) return;
  __shared__ __align__(16) __nv_bfloat16 Qs[TILE];
  __shared__ __align__(16) __nv_bfloat16 Ks[2][TILE];
  __shared__ float s_madd[2][TQ];
  __shared__ float s_D[TQ];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, cq = 2 * (lane & 3);
  const int HD = NH * D;
  const size_t rs = (size_t)3 * HD;
  const __nv_bfloat16* base = qkv + row_base * rs + h * D;
  const __nv_bfloat16* obase = ctx + row_base * HD + h * D;
  const __nv_bfloat16* dobase = dctx + row_base * HD + h * D;
  const int nkt = (L + TQ - 1) / TQ;

  tile_async(Qs, base, rs, q0, L, tid);
  tile_async(Ks[0], base + HD, rs, 0, L, tid);
  stage_key_add(s_madd[0], mask, cu_seqlens, b, Lpad, L, 0, mask_add, tid);
  cp_async_commit();
  // D = rowsum(dO o O): 8 lanes per row, 16 B each
#pragma unroll
  for (int i = 0; i < TQ / (TW * 4); ++i) {
    const int r = i * TW * 4 + warp * 4 + (lane >> 3), ch = lane & 7;
    float d = 0.f;
    if (q0 + r < L) {
      const uint4 g = *reinterpret_cast<const uint4*>(dobase + (size_t)(q0 + r) * HD + ch * 8);
      const uint4 o = *reinterpret_cast<const uint4*>(obase + (size_t)(q0 + r) * HD + ch * 8);
      const __nv_bfloat162* g2 = reinterpret_cast<const __nv_bfloat162*>(&g);
      const __nv_bfloat162* o2 = reinterpret_cast<const __nv_bfloat162*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j)
        d += __low2float(g2[j]) * __low2float(o2[j]) + __high2float(g2[j]) * __high2float(o2[j]);
    }
    d += __shfl_xor_sync(0xffffffffu, d, 1);
    d += __shfl_xor_sync(0xffffffffu, d, 2);
    d += __shfl_xor_sync(0xffffffffu, d, 4);
    if ((lane & 7) == 0) s_D[r] = d;
  }
  cp_async_wait<0>();
  __syncthreads();

  constexpr float kLog2e = 1.4426950408889634f;
  const int rl0 = warp * 16 + (lane >> 2), rl1 = rl0 + 8;
  uint32_t qa[4][4];
  load_a_frags(qa, Qs, rl0, cq);
  float m0 = -1e30f, m1 = -1e30f, l0 = 0.f, l1 = 0.f;
  for (int t = 0; t < nkt; ++t) {
    const int buf = t & 1;
    if (t + 1 < nkt) {
      tile_async(Ks[buf ^ 1], base + HD, rs, (t + 1) * TQ, L, tid);
      stage_key_add(s_madd[buf ^ 1], mask, cu_seqlens, b, Lpad, L, (t + 1) * TQ, mask_add, tid);
      cp_async_commit();
    }
    float s[8][4];
    clear_tile(s);
    mma_a_bt(s, qa, Ks[buf], 0, lane, cq);
    float mx0 = -1e30f, mx1 = -1e30f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float a0 = s_madd[buf][nt * 8 + cq], a1 = s_madd[buf][nt * 8 + cq + 1];
      s[nt][0] = s[nt][0] * scale + a0;
      s[nt][1] = s[nt][1] * scale + a1;
      s[nt][2] = s[nt][2] * scale + a0;
      s[nt][3] = s[nt][3] * scale + a1;
      mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float n0 = fmaxf(m0, mx0), n1 = fmaxf(m1, mx1);
    float p0 = 0.f, p1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      p0 += exp2f((s[nt][0] - n0) * kLog2e) + exp2f((s[nt][1] - n0) * kLog2e);
      p1 += exp2f((s[nt][2] - n1) * kLog2e) + exp2f((s[nt][3] - n1) * kLog2e);
    }
    l0 = l0 * exp2f((m0 - n0) * kLog2e) + p0;
    l1 = l1 * exp2f((m1 - n1) * kLog2e) + p1;
    m0 = n0;
    m1 = n1;
    if (t + 1 < nkt) cp_async_wait<0>();
    __syncthreads();
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  if ((lane & 3) == 0) {
    __nv_bfloat16* st = dqkv + row_base * rs + h * D;
    if (q0 + rl0 < L) *reinterpret_cast<float2*>(st + (size_t)(q0 + rl0) * rs) = make_float2(m0 + logf(l0), s_D[rl0]);
    if (q0 + rl1 < L) *reinterpret_cast<float2*>(st + (size_t)(q0 + rl1) * rs) = make_float2(m1 + logf(l1), s_D[rl1]);
  }
}

template <bool DROP>
__global__ void __launch_bounds__(TW * 32)
bert_attention_bwd_dkdv_kernel(const __nv_bfloat16* __restrict__ qkv, const int32_t* __restrict__ mask,
                               const __nv_bfloat16* __restrict__ dctx, __nv_bfloat16* __restrict__ dqkv, int Lpad, int NH,
                               float scale, float mask_add, const int32_t* __restrict__ cu_seqlens, float keep,
                               uint32_t seed_lo, uint32_t seed_hi) {
  const int b = blockIdx.z, h = blockIdx.y, kt0 = blockIdx.x * TQ;
  const size_t row_base = cu_seqlens ? (size_t)cu_seqlens[b] : (size_t)b * Lpad;
  const int L = cu_seqlens ? (cu_seqlens[b + 1] - cu_seqlens[b]) : Lpad;
  if (kt0 >= L) return;
  const uint32_t dsa = seed_lo ^ ((uint32_t)(b * NH + h) * 0x9E3779B1u), dthr = keep_threshold(keep);
  const float dik = 1.f / keep;
  extern __shared__ __align__(16) uint8_t smraw[];
  __nv_bfloat16* Ks = reinterpret_cast<__nv_bfloat16*>(smraw);
  __nv_bfloat16* Vs = Ks + TILE;
  __nv_bfloat16* Qs = Vs + TILE;      // [2][TILE]
  __nv_bfloat16* Os = Qs + 2 * TILE;  // dO, [2][TILE]
  float2* s_st = reinterpret_cast<float2*>(Os + 2 * TILE);  // [2][TQ] (lse, D)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, cq = 2 * (lane & 3);
  const int HD = NH * D;
  const size_t rs = (size_t)3 * HD;
  const __nv_bfloat16* base = qkv + row_base * rs + h * D;
  const __nv_bfloat16* dobase = dctx + row_base * HD + h * D;
  const __nv_bfloat16* stbase = dqkv + row_base * rs + h * D;
  const int nqt = (L + TQ - 1) / TQ;
  auto stage_q = [&](int buf, int qt0) {
    tile_async(Qs + buf * TILE, base, rs, qt0, L, tid);
    tile_async(Os + buf * TILE, dobase, HD, qt0, L, tid);
    if (tid < TQ) {
      if (qt0 + tid < L) cp_async8(s_st + buf * TQ + tid, stbase + (size_t)(qt0 + tid) * rs);
      else s_st[buf * TQ + tid] = make_float2(INFINITY, 0.f);  // no such query: P = 0
    }
  };

  tile_async(Ks, base + HD, rs, kt0, L, tid);
  tile_async(Vs, base + 2 * HD, rs, kt0, L, tid);
  stage_q(0, 0);
  cp_async_commit();
  const int kl0 = warp * 16 + (lane >> 2);
  const int k0 = kt0 + kl0, k1 = k0 + 8;
  const float ma0 = key_add(mask, cu_seqlens, b, Lpad, L, k0, mask_add);
  const float ma1 = key_add(mask, cu_seqlens, b, Lpad, L, k1, mask_add);
  cp_async_wait<0>();
  __syncthreads();

  constexpr float kLog2e = 1.4426950408889634f;
  uint32_t ka[4][4], va[4][4];
  load_a_frags(ka, Ks, kl0, cq);
  load_a_frags(va, Vs, kl0, cq);
  float dk[8][4], dv[8][4];
  clear_tile(dk);
  clear_tile(dv);
  for (int t = 0; t < nqt; ++t) {
    const int buf = t & 1;
    if (t + 1 < nqt) {
      stage_q(buf ^ 1, (t + 1) * TQ);
      cp_async_commit();
    }
    const __nv_bfloat16* Qb = Qs + buf * TILE;
    const __nv_bfloat16* Ob = Os + buf * TILE;
    const float2* stb = s_st + buf * TQ;
    float st[8][4], dpt[8][4];
    clear_tile(st);
    clear_tile(dpt);
    mma_a_bt(st, ka, Qb, 0, lane, cq);   // S^T  = K Q^T      (rows: keys, cols: queries)
    mma_a_bt(dpt, va, Ob, 0, lane, cq);  // dP^T = V dO^T
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int q0 = t * TQ + nt * 8 + cq, q1 = q0 + 1;
      const float2 s0 = stb[nt * 8 + cq], s1 = stb[nt * 8 + cq + 1];
      const float p00 = exp2f((st[nt][0] * scale + ma0 - s0.x) * kLog2e);
      const float p01 = exp2f((st[nt][1] * scale + ma0 - s1.x) * kLog2e);
      const float p10 = exp2f((st[nt][2] * scale + ma1 - s0.x) * kLog2e);
      const float p11 = exp2f((st[nt][3] * scale + ma1 - s1.x) * kLog2e);
      float z00 = 1.f, z01 = 1.f, z10 = 1.f, z11 = 1.f;
      if (DROP) {
        z00 = attn_drop(dsa, seed_hi, q0, k0, dthr, dik);
        z01 = attn_drop(dsa, seed_hi, q1, k0, dthr, dik);
        z10 = attn_drop(dsa, seed_hi, q0, k1, dthr, dik);
        z11 = attn_drop(dsa, seed_hi, q1, k1, dthr, dik);
      }
      st[nt][0] = p00 * z00;
      st[nt][1] = p01 * z01;
      st[nt][2] = p10 * z10;
      st[nt][3] = p11 * z11;
      dpt[nt][0] = p00 * (z00 * dpt[nt][0] - s0.y);
      dpt[nt][1] = p01 * (z01 * dpt[nt][1] - s1.y);
      dpt[nt][2] = p10 * (z10 * dpt[nt][2] - s0.y);
      dpt[nt][3] = p11 * (z11 * dpt[nt][3] - s1.y);
    }
    mma_p_b(dv, st, Ob, 0, lane);   // dV += P^T dO
    mma_p_b(dk, dpt, Qb, 0, lane);  // dK += dS^T Q
    if (t + 1 < nqt) cp_async_wait<0>();
    __syncthreads();
  }
  __nv_bfloat16* dkb = dqkv + row_base * rs + HD + h * D;
  __nv_bfloat16* dvb = dqkv + row_base * rs + 2 * HD + h * D;
#pragma unroll
  for (int dt = 0; dt < 8; ++dt) {
    if (k0 < L) {
      *reinterpret_cast<uint32_t*>(dkb + (size_t)k0 * rs + dt * 8 + cq) = pack2(dk[dt][0] * scale, dk[dt][1] * scale);
      *reinterpret_cast<uint32_t*>(dvb + (size_t)k0 * rs + dt * 8 + cq) = pack2(dv[dt][0], dv[dt][1]);
    }
    if (k1 < L) {
      *reinterpret_cast<uint32_t*>(dkb + (size_t)k1 * rs + dt * 8 + cq) = pack2(dk[dt][2] * scale, dk[dt][3] * scale);
      *reinterpret_cast<uint32_t*>(dvb + (size_t)k1 * rs + dt * 8 + cq) = pack2(dv[dt][2], dv[dt][3]);
    }
  }
}

template <bool DROP>
__global__ void __launch_bounds__(TW * 32)
bert_attention_bwd_dq_kernel(const __nv_bfloat16* __restrict__ qkv, const int32_t* __restrict__ mask,
                             const __nv_bfloat16* __restrict__ dctx, __nv_bfloat16* __restrict__ dqkv, int Lpad, int NH,
                             float scale, float mask_add, const int32_t* __restrict__ cu_seqlens, float keep,
                             uint32_t seed_lo, uint32_t seed_hi) {
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * TQ;
  const size_t row_base = cu_seqlens ? (size_t)cu_seqlens[b] : (size_t)b * Lpad;
  const int L = cu_seqlens ? (cu_seqlens[b + 1] - cu_seqlens[b]) : Lpad;
  if (q0 >= L) return;
  const uint32_t dsa = seed_lo ^ ((uint32_t)(b * NH + h) * 0x9E3779B1u), dthr = keep_threshold(keep);
  const float dik = 1.f / keep;
  extern __shared__ __align__(16) uint8_t smraw[];
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(smraw);
  __nv_bfloat16* Os = Qs + TILE;      // dO
  __nv_bfloat16* Ks = Os + TILE;      // [2][TILE]
  __nv_bfloat16* Vs = Ks + 2 * TILE;  // [2][TILE]
  float* s_madd = reinterpret_cast<float*>(Vs + 2 * TILE);  // [2][TQ]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, cq = 2 * (lane & 3);
  const int HD = NH * D;
  const size_t rs = (size_t)3 * HD;
  const __nv_bfloat16* base = qkv + row_base * rs + h * D;
  const __nv_bfloat16* dobase = dctx + row_base * HD + h * D;
  __nv_bfloat16* dqb = dqkv + row_base * rs + h * D;
  const int nkt = (L + TQ - 1) / TQ;
  auto stage_k = [&](int buf, int kt0) {
    tile_async(Ks + buf * TILE, base + HD, rs, kt0, L, tid);
    tile_async(Vs + buf * TILE, base + 2 * HD, rs, kt0, L, tid);
    stage_key_add(s_madd + buf * TQ, mask, cu_seqlens, b, Lpad, L, kt0, mask_add, tid);
  };

  tile_async(Qs, base, rs, q0, L, tid);
  tile_async(Os, dobase, HD, q0, L, tid);
  stage_k(0, 0);
  cp_async_commit();
  const int rl0 = warp * 16 + (lane >> 2);
  const int r0 = q0 + rl0, r1 = r0 + 8;
  // this CTA's own rows' (lse, D), read before the dQ stores below overwrite them
  float2 st0 = make_float2(0.f, 0.f), st1 = make_float2(0.f, 0.f);
  if (r0 < L) st0 = *reinterpret_cast<const float2*>(dqb + (size_t)r0 * rs);
  if (r1 < L) st1 = *reinterpret_cast<const float2*>(dqb + (size_t)r1 * rs);
  cp_async_wait<0>();
  __syncthreads();

  constexpr float kLog2e = 1.4426950408889634f;
  uint32_t qa[4][4], da[4][4];
  load_a_frags(qa, Qs, rl0, cq);
  load_a_frags(da, Os, rl0, cq);
  float dq[8][4];
  clear_tile(dq);
  for (int t = 0; t < nkt; ++t) {
    const int buf = t & 1;
    if (t + 1 < nkt) {
      stage_k(buf ^ 1, (t + 1) * TQ);
      cp_async_commit();
    }
    const __nv_bfloat16* Kb = Ks + buf * TILE;
    const __nv_bfloat16* Vb = Vs + buf * TILE;
    const float* mb = s_madd + buf * TQ;
    float s[8][4], dp[8][4];
    clear_tile(s);
    clear_tile(dp);
    mma_a_bt(s, qa, Kb, 0, lane, cq);
    mma_a_bt(dp, da, Vb, 0, lane, cq);
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float a0 = mb[nt * 8 + cq], a1 = mb[nt * 8 + cq + 1];
      const float p00 = exp2f((s[nt][0] * scale + a0 - st0.x) * kLog2e);
      const float p01 = exp2f((s[nt][1] * scale + a1 - st0.x) * kLog2e);
      const float p10 = exp2f((s[nt][2] * scale + a0 - st1.x) * kLog2e);
      const float p11 = exp2f((s[nt][3] * scale + a1 - st1.x) * kLog2e);
      if (DROP) {
        const int k = t * TQ + nt * 8 + cq;
        dp[nt][0] *= attn_drop(dsa, seed_hi, r0, k, dthr, dik);
        dp[nt][1] *= attn_drop(dsa, seed_hi, r0, k + 1, dthr, dik);
        dp[nt][2] *= attn_drop(dsa, seed_hi, r1, k, dthr, dik);
        dp[nt][3] *= attn_drop(dsa, seed_hi, r1, k + 1, dthr, dik);
      }
      s[nt][0] = p00 * (dp[nt][0] - st0.y);
      s[nt][1] = p01 * (dp[nt][1] - st0.y);
      s[nt][2] = p10 * (dp[nt][2] - st1.y);
      s[nt][3] = p11 * (dp[nt][3] - st1.y);
    }
    mma_p_b(dq, s, Kb, 0, lane);
    if (t + 1 < nkt) cp_async_wait<0>();
    __syncthreads();
  }
#pragma unroll
  for (int dt = 0; dt < 8; ++dt) {
    if (r0 < L) *reinterpret_cast<uint32_t*>(dqb + (size_t)r0 * rs + dt * 8 + cq) = pack2(dq[dt][0] * scale, dq[dt][1] * scale);
    if (r1 < L) *reinterpret_cast<uint32_t*>(dqb + (size_t)r1 * rs + dt * 8 + cq) = pack2(dq[dt][2] * scale, dq[dt][3] * scale);
  }
}

}  // namespace

static int attention_bwd_tiled(const __nv_bfloat16* qkv, const int32_t* mask, const __nv_bfloat16* ctx,
                               const __nv_bfloat16* dctx, __nv_bfloat16* dqkv, int B, int L, int num_heads, float scale,
                               float mask_add, const int32_t* cu_seqlens, float keep_prob, uint64_t seed, cudaStream_t st) {
  auto dkdv = keep_prob < 1.f ? bert_attention_bwd_dkdv_kernel<true> : bert_attention_bwd_dkdv_kernel<false>;
  auto dq = keep_prob < 1.f ? bert_attention_bwd_dq_kernel<true> : bert_attention_bwd_dq_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(dkdv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)KV_SMEM);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(dq, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DQ_SMEM);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  const dim3 grid((L + TQ - 1) / TQ, num_heads, B), block(TW * 32);
  const uint32_t lo = (uint32_t)seed, hi = (uint32_t)(seed >> 32);
  bert_attention_bwd_stats_kernel<<<grid, block, 0, st>>>(qkv, mask, ctx, dctx, dqkv, L, num_heads, scale, mask_add,
                                                          cu_seqlens);
  if ((e = cudaGetLastError()) != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  dkdv<<<grid, block, KV_SMEM, st>>>(qkv, mask, dctx, dqkv, L, num_heads, scale, mask_add, cu_seqlens, keep_prob, lo, hi);
  if ((e = cudaGetLastError()) != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  dq<<<grid, block, DQ_SMEM, st>>>(qkv, mask, dctx, dqkv, L, num_heads, scale, mask_add, cu_seqlens, keep_prob, lo, hi);
  return ner_launch_status();
}

static int attention_bwd_launch(const void* qkv_bf16, const int32_t* mask, const void* ctx_bf16, const void* dctx_bf16,
                                void* dqkv_bf16, int B, int L, int num_heads, int head_dim, float scale, float mask_add,
                                const int32_t* cu_seqlens, float keep_prob, uint64_t seed, ner_stream_t stream) {
  if (B < 0 || L < 1 || num_heads < 1 || !(keep_prob > 0.f)) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!qkv_bf16 || (!mask && !cu_seqlens) || !ctx_bf16 || !dctx_bf16 || !dqkv_bf16) return NER_ERR_INVALID_ARG;
  if (head_dim != D) return NER_ERR_UNSUPPORTED;
  const int Lp = (L + 63) / 64 * 64;
  const size_t smem = (size_t)4 * Lp * PITCH * 2 + (size_t)4 * Lp * 4;
  if (smem > 227 * 1024)  // the whole head fits up to L = 384; longer sequences take the key-tiled kernels
    return attention_bwd_tiled(static_cast<const __nv_bfloat16*>(qkv_bf16), mask, static_cast<const __nv_bfloat16*>(ctx_bf16),
                               static_cast<const __nv_bfloat16*>(dctx_bf16), static_cast<__nv_bfloat16*>(dqkv_bf16), B, L,
                               num_heads, scale, mask_add, cu_seqlens, keep_prob, seed, static_cast<cudaStream_t>(stream));
  auto kern = keep_prob < 1.f ? bert_attention_bwd_kernel<true> : bert_attention_bwd_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  dim3 grid(num_heads, B);
  kern<<<grid, NW * 32, smem, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(qkv_bf16), mask, static_cast<const __nv_bfloat16*>(ctx_bf16),
      static_cast<const __nv_bfloat16*>(dctx_bf16), static_cast<__nv_bfloat16*>(dqkv_bf16), L, num_heads, Lp, scale,
      mask_add, cu_seqlens, keep_prob, (uint32_t)seed, (uint32_t)(seed >> 32));
  return ner_launch_status();
}

extern "C" int ner_bert_attention_bwd(const void* qkv_bf16, const int32_t* mask, const void* ctx_bf16,
                                      const void* dctx_bf16, void* dqkv_bf16, int B, int L, int num_heads,
                                      int head_dim, float scale, float mask_add, float keep_prob, uint64_t seed,
                                      ner_stream_t stream) {
  if (!mask) return B == 0 ? NER_OK : NER_ERR_INVALID_ARG;
  return attention_bwd_launch(qkv_bf16, mask, ctx_bf16, dctx_bf16, dqkv_bf16, B, L, num_heads, head_dim, scale, mask_add,
                              nullptr, keep_prob, seed, stream);
}

extern "C" int ner_bert_attention_bwd_packed(const void* qkv_bf16, const int32_t* cu_seqlens, const void* ctx_bf16,
                                             const void* dctx_bf16, void* dqkv_bf16, int B, int L, int num_heads,
                                             int head_dim, float scale, float keep_prob, uint64_t seed,
                                             ner_stream_t stream) {
  if (!cu_seqlens) return B == 0 ? NER_OK : NER_ERR_INVALID_ARG;
  return attention_bwd_launch(qkv_bf16, nullptr, ctx_bf16, dctx_bf16, dqkv_bf16, B, L, num_heads, head_dim, scale, 0.f,
                              cu_seqlens, keep_prob, seed, stream);
}
