// BERT self-attention core on the Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a, inference path:
//   ctx = softmax(Q K^T * scale + (1 - mask) * mask_add) V     per (sequence, head), head_dim = 64
// (attention_layer() of bert_base.bert.modeling as executed from reference tools/layer.py:68-77; SURVEY Appendix A.3).
//
// One CTA = one warpgroup = one (sequence b, head h, tile of 64 query rows); sequences of up to 256 keys are handled in
// ONE pass.  A short sequence (<= 64 tokens, most of an MSRA batch) is one CTA per head with no idle warps; tiles past a
// packed sequence's end exit at once, so the host sizes the grid from B, NH and the longest length alone.
//   thread 0 TMA: Q tile, K rows and V rows of the head come from the fused [rows, 3H] QKV matrix as 64-row x 64-column
//            bf16 boxes (CU_TENSOR_MAP_SWIZZLE_128B) into shared memory, mbarrier transaction counts
//   MMA 1    S[64, N] = Q K^T — four wgmma.m64nNk16 (K = 16 each) from K-major SWIZZLE_128B descriptors, fp32
//            accumulator in registers; N = the sequence's key count rounded up to 64 (<= NKMAX)
//   softmax  in registers (row max / sum over the 4 lanes that share a row); the unnormalised probabilities go to
//            shared memory as bf16 in the canonical K-major SWIZZLE_128B A-operand layout (over the space Q and K
//            occupied, after every warp finished reading them)
//   MMA 2    O[64, 64] = P V — V stays as TMA delivered it ([key][d], d contiguous) and is consumed as an MN-MAJOR
//            ("transposed") B operand (8-key swizzle atoms 1024 B apart), N/16 MMAs
//   store    O rows times 1 / row sum, bf16, staged in shared memory by stmatrix and written to ctx as whole rows
// Shared memory 41 KB (NKMAX 128, five CTAs per SM) / 73 KB (NKMAX 256, three).  Nothing L x L leaves the SM.  Rows of
// other sequences that ride along in a 64-row box are masked as keys (probability exactly 0, V rows >= L zeroed in shared
// memory) and never stored as queries.
#include <stdlib.h>

#include "tc_common.cuh"

namespace {

using namespace tc;
using nerdev::fast_ex2;

constexpr int D = 64;          // head_dim
constexpr int QT = 64;         // query rows per work item (one wgmma M = 64 warpgroup)
constexpr int BOX_ROWS = 64;   // rows per TMA box
constexpr int BOX_BYTES = BOX_ROWS * D * 2;   // 8 KB
constexpr int THREADS = 128;

template <int NKMAX>
struct ACfg {
  static constexpr int KV_BYTES = NKMAX * D * 2;
  // Q tile + K rows; once S is complete, P [N/64][64 rows][128 B] from offset 0 and the 64 x 64 bf16 output tile after
  // the largest P (exactly where the last 64 K rows were)
  static constexpr int REGION_A = QT * D * 2 + KV_BYTES;
  static constexpr int O_OFFSET = QT * NKMAX * 2;
  static_assert(O_OFFSET + QT * D * 2 <= REGION_A, "P and the output tile must fit over Q and K");
  static constexpr size_t SMEM = (size_t)REGION_A + KV_BYTES + 64 + NKMAX * 4;
  // resident CTAs per SM the registers are budgeted for, which shared memory also admits (41 KB / 73 KB per CTA)
  static constexpr int MIN_CTAS = NKMAX == 128 ? 5 : 3;
};

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

// S = Q K^T for the item's 64 query rows over N key columns, softmax numerators into the P tile, then O = P V and the
// normalised store.  r_lo = this thread's first row within the tile (the second is r_lo + 8).  PACKED: every key < L is
// valid and s_madd is not read (its entries are 0 there).
template <int N, bool PACKED>
__device__ __forceinline__ void attend(uint8_t* s_q, uint8_t* s_k, uint8_t* s_p, uint8_t* s_v, uint8_t* s_o, const float* s_madd, int r_lo,
                                       int L, float sc, uint64_t* v_bar, __nv_bfloat16* ctx,
                                       size_t out_row0, int HD, int h, int q0) {
  const int lane = threadIdx.x & 31;
  constexpr float kLog2e = 1.4426950408889634f;
  float s[N / 2];
  float lsum[2] = {0.f, 0.f};
  {
    const uint32_t qa = smem_u32(s_q), ka = smem_u32(s_k);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < D / 16; ++k)
      wgmma_bf16<N, 0, 0>(s, make_wgmma_desc_sw128(qa + k * 32), make_wgmma_desc_sw128(ka + k * 32), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    // scores in the log2 domain: x = s*scale*log2e + madd*log2e (packed: madd = 0, and fmaf(s, sc, 0) rounds like
    // s * sc); columns >= L (other sequences' or never loaded key rows) are excluded by a select, so whatever their score
    // holds (NaN included) never reaches the max, the sum or P.  N rounds L up to 64, so only the last 64 columns can
    // be >= L.
    float mx[2] = {-3.0e38f, -3.0e38f};
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int c = 8 * j + 2 * (lane & 3) + (e & 1);
        const float x = PACKED ? s[4 * j + e] * sc : fmaf(s[4 * j + e], sc, s_madd[c] * kLog2e);
        s[4 * j + e] = x;
        if (8 * j < N - 64 || c < L) mx[e >> 1] = fmaxf(mx[e >> 1], x);
      }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
    }
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int c = 8 * j + 2 * (lane & 3) + (e & 1);
        const float p = (8 * j < N - 64 || c < L) ? fast_ex2(s[4 * j + e] - mx[e >> 1]) : 0.f;
        s[4 * j + e] = p;
        lsum[e >> 1] += p;
      }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      lsum[hh] += __shfl_xor_sync(0xffffffffu, lsum[hh], 1);
      lsum[hh] += __shfl_xor_sync(0xffffffffu, lsum[hh], 2);
    }
  }
  __syncthreads();                             // every warp is done reading Q and K: P may overwrite them
#pragma unroll
  for (int j = 0; j < N / 8; ++j)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int r = r_lo + 8 * hh, c = 8 * j + 2 * (lane & 3);
      uint8_t* blk = s_p + (c >> 6) * (QT * 128) + (r >> 3) * 1024 + (r & 7) * 128;
      *reinterpret_cast<uint32_t*>(blk + ((((c & 63) >> 3) ^ (r & 7)) << 4) + (c & 7) * 2) =
          pack_bf16x2(s[4 * j + 2 * hh], s[4 * j + 2 * hh + 1]);
    }
  // V rows [L, N) belong to other sequences (or were never loaded): zero them so that 0 * x stays 0
  mbar_wait(v_bar, 0);
  for (int idx = threadIdx.x; idx < (N - L) * 8; idx += THREADS)
    *reinterpret_cast<uint4*>(s_v + (size_t)(L + (idx >> 3)) * 128 + ((idx & 7) << 4)) = make_uint4(0, 0, 0, 0);
  fence_proxy_async();                         // P and the zeroed V rows: generic-proxy writes -> visible to wgmma
  __syncthreads();

  float o[D / 2];
  {
    const uint32_t pa = smem_u32(s_p), va = smem_u32(s_v);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < N / 16; ++ks)
      wgmma_bf16<D, 0, 1>(o, make_wgmma_desc_sw128(pa + (ks >> 2) * (QT * 128) + (ks & 3) * 32),
                          make_wgmma_desc_sw128(va + ks * 2048), ks > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
  }
  // O times 1 / row sum as bf16 into this warp's 16 rows of s_o (stmatrix; the 16-byte chunks of row r sit at chunk ^
  // (r & 7), so that neither these stores nor the reads below conflict), then whole 128-byte rows to ctx: full 32-byte
  // sectors instead of 16-byte pieces of eight rows per store
  const int warp = threadIdx.x >> 5;
  const float inv0 = 1.f / lsum[0], inv1 = 1.f / lsum[1];
  const uint32_t so = smem_u32(s_o);
#pragma unroll
  for (int j = 0; j < D / 8; j += 2) {
    const int i = lane >> 3, jj = j + (i >> 1), r = 16 * warp + 8 * (i & 1) + (lane & 7);
    stmatrix_x4(so + r * 128 + ((jj ^ (r & 7)) << 4),
                pack_bf16x2(o[4 * j] * inv0, o[4 * j + 1] * inv0), pack_bf16x2(o[4 * j + 2] * inv1, o[4 * j + 3] * inv1),
                pack_bf16x2(o[4 * j + 4] * inv0, o[4 * j + 5] * inv0), pack_bf16x2(o[4 * j + 6] * inv1, o[4 * j + 7] * inv1));
  }
  __syncwarp();
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int r = 16 * warp + 4 * it + (lane >> 3), ch = lane & 7;
    if (q0 + r < L)
      *reinterpret_cast<uint4*>(ctx + (out_row0 + r) * HD + h * D + ch * 8) =
          *reinterpret_cast<const uint4*>(s_o + r * 128 + ((ch ^ (r & 7)) << 4));
  }
}

// PACKED: rows and lengths from cu_seqlens; otherwise padded rows and the additive mask
template <int NKMAX, bool PACKED>
__global__ void __launch_bounds__(THREADS, ACfg<NKMAX>::MIN_CTAS)
bert_attention_tc_kernel(const __grid_constant__ CUtensorMap tma_qkv, const int32_t* __restrict__ mask,
                         __nv_bfloat16* __restrict__ ctx, int Lpad, int NH, float scale, float mask_add,
                         const int32_t* __restrict__ cu_seqlens) {
  using C = ACfg<NKMAX>;
  nerdev::pdl_launch_dependents();
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0u) __trap();
  uint8_t* s_q = smem;                         // [64 rows][128 B]   (SW128, 8-row groups of 1 KB)
  uint8_t* s_k = smem + QT * D * 2;            // [Nk rows][128 B]
  uint8_t* s_p = smem;                         // [Nk/64 blocks][64 rows][128 B] — written after S is complete
  uint8_t* s_v = smem + C::REGION_A;           // [Nk rows][128 B]
  uint8_t* s_o = smem + C::O_OFFSET;           // [64 rows][128 B]: bf16 context rows on their way to ctx, after S
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_v + C::KV_BYTES);   // qk, v
  float* s_madd = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 64);

  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * QT;
  const int tid = threadIdx.x;
  const int HD = NH * D;

  if (tid == 0) {
    tma_prefetch_desc(&tma_qkv);
    for (int i = 0; i < 2; ++i) mbar_init(&bars[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  nerdev::pdl_wait();                         // QKV comes from the GEMM just before this kernel in the stream

  // padded mode: rows [b*Lpad, (b+1)*Lpad), keys masked by `mask`; packed mode: rows [cu[b], cu[b+1]), all keys valid
  const int row_base = PACKED ? cu_seqlens[b] : b * Lpad;
  const int L = PACKED ? (cu_seqlens[b + 1] - row_base) : Lpad;
  if (q0 >= L) return;                        // uniform over the CTA
  const int n64 = (L + 63) & ~63;             // wgmma N of S = K extent of P V (multiple of 64, <= NKMAX)
  const int kv_boxes = n64 / BOX_ROWS;

  if (tid == 0) {
    mbar_arrive_expect_tx(&bars[0], (uint32_t)((1 + kv_boxes) * BOX_BYTES));
    tma_load_2d(s_q, &tma_qkv, &bars[0], h * D, row_base + q0);
    for (int i = 0; i < kv_boxes; ++i) tma_load_2d(s_k + i * BOX_BYTES, &tma_qkv, &bars[0], HD + h * D, row_base + i * BOX_ROWS);
    mbar_arrive_expect_tx(&bars[1], (uint32_t)(kv_boxes * BOX_BYTES));
    for (int i = 0; i < kv_boxes; ++i) tma_load_2d(s_v + i * BOX_BYTES, &tma_qkv, &bars[1], 2 * HD + h * D, row_base + i * BOX_ROWS);
  }
  if constexpr (!PACKED) {
    for (int k = tid; k < n64; k += THREADS)
      s_madd[k] = (k < L) ? (1.f - (float)mask[(size_t)b * Lpad + k]) * mask_add : -1e30f;
    __syncthreads();                          // s_madd visible
  }
  mbar_wait(&bars[0], 0);

  constexpr float kLog2e = 1.4426950408889634f;
  const float sc = scale * kLog2e;
  const int r_lo = ((tid >> 5) & 3) * 16 + ((tid & 31) >> 2);
  const size_t out_row0 = (size_t)row_base + q0;
  if (n64 <= 64) attend<64, PACKED>(s_q, s_k, s_p, s_v, s_o, s_madd, r_lo, L, sc, &bars[1], ctx, out_row0, HD, h, q0);
  else if (n64 <= 128 || NKMAX == 128)
    attend<128, PACKED>(s_q, s_k, s_p, s_v, s_o, s_madd, r_lo, L, sc, &bars[1], ctx, out_row0, HD, h, q0);
  else if constexpr (NKMAX == 256) {
    if (n64 <= 192) attend<192, PACKED>(s_q, s_k, s_p, s_v, s_o, s_madd, r_lo, L, sc, &bars[1], ctx, out_row0, HD, h, q0);
    else attend<256, PACKED>(s_q, s_k, s_p, s_v, s_o, s_madd, r_lo, L, sc, &bars[1], ctx, out_row0, HD, h, q0);
  }
}

template <int NKMAX, bool PACKED>
int launch(const CUtensorMap& map, const int32_t* mask, void* ctx, int B, int L, int NH, float scale, float mask_add,
           const int32_t* cu_seqlens, cudaStream_t st) {
  auto kern = bert_attention_tc_kernel<NKMAX, PACKED>;
  const size_t smem = ACfg<NKMAX>::SMEM;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  dim3 grid((L + QT - 1) / QT, NH, B);
  e = ner_launch_pdl(kern, grid, dim3(THREADS), smem, st, map, mask, static_cast<__nv_bfloat16*>(ctx), L, NH, scale, mask_add,
                     cu_seqlens);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  return ner_launch_status();
}

}  // namespace

// wgmma path of ner_bert_attention (inference: no attention-probs dropout).  NER_ERR_UNSUPPORTED = not applicable
// (caller falls back to the mma.sync kernel): head_dim != 64, sequences longer than 256, misaligned QKV.
int ner_bert_attention_tc(const void* qkv_bf16, const int32_t* mask, void* ctx_bf16, int B, int L, int num_heads, int head_dim,
                          float scale, float mask_add, const int32_t* cu_seqlens, int n_rows, cudaStream_t st) {
  if (head_dim != D || L > 256 || n_rows < 1) return NER_ERR_UNSUPPORTED;
  const uint64_t cols = (uint64_t)3 * num_heads * D;
  if ((reinterpret_cast<uintptr_t>(qkv_bf16) & 15) != 0 || (cols * 2) % 16 != 0 ||
      (reinterpret_cast<uintptr_t>(ctx_bf16) & 15) != 0)
    return NER_ERR_UNSUPPORTED;
  tc::EncodeTiledFn fn = tc::tensor_map_encode_fn();
  if (fn == nullptr) return NER_ERR_UNSUPPORTED;
  CUtensorMap map;
  cuuint64_t dims[2] = {cols, (cuuint64_t)n_rows};
  cuuint64_t strides[1] = {cols * 2};
  cuuint32_t box[2] = {(cuuint32_t)D, (cuuint32_t)BOX_ROWS};
  cuuint32_t estr[2] = {1, 1};
  if (fn(&map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(qkv_bf16), dims, strides, box, estr,
         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return NER_ERR_UNSUPPORTED;
  if (L <= 128)
    return cu_seqlens ? launch<128, true>(map, mask, ctx_bf16, B, L, num_heads, scale, mask_add, cu_seqlens, st)
                      : launch<128, false>(map, mask, ctx_bf16, B, L, num_heads, scale, mask_add, cu_seqlens, st);
  return cu_seqlens ? launch<256, true>(map, mask, ctx_bf16, B, L, num_heads, scale, mask_add, cu_seqlens, st)
                    : launch<256, false>(map, mask, ctx_bf16, B, L, num_heads, scale, mask_add, cu_seqlens, st);
}
