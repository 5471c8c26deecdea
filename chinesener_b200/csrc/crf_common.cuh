// Shared pieces of the CRF dynamic-programming kernels (Viterbi, forward-alpha, backward).
//
// Work decomposition (all three kernels): ONE THREAD PER SEQUENCE, NT sequences per CTA.
// The K-wide DP state lives in registers; emission logits are streamed HBM -> smem with
// cp.async in chunks of T=8 time steps per sequence (coalesced 16-byte requests over the
// CTA's contiguous [NT, L*K] slab), then each thread reads its own row back with LDS.128.
// Row pitch P = 8K+4 floats makes P/4 odd, so the 8 threads of a quarter-warp hit 8
// distinct 16-byte bank groups (conflict-free).
#pragma once
#include "common.cuh"

namespace crf {

using namespace nerdev;

constexpr int T_CHUNK = 8;  // time steps staged per chunk
constexpr int NSTAGE = 2;   // cp.async ring depth

template <int K, int TT = T_CHUNK>
struct Geom {
  static constexpr int T = TT;
  static constexpr int G = (K % 4 == 0) ? 1 : ((K % 2 == 0) ? 2 : 4);  // steps per LDS.128 group
  static constexpr int CE = T * K;                                    // floats per row-chunk
  static constexpr int NQ = CE / 4;                                   // float4 per row-chunk
  static constexpr int P = 4 * (NQ | 1);                              // row pitch (floats)
  static constexpr int GQ = G * K / 4;                                // float4 per step group
  static constexpr bool UNROLL = (K <= 12);                           // registers vs local arrays
  static constexpr int KK4 = (K * K + 3) & ~3;
};

// Stage chunk `c` (time steps [t0, t0+T)) of the CTA's rows into dst[NT][P].
// s_len[r] = effective length of row r (>= 1); elements at t >= s_len[r] are not fetched.
template <int K, int NT, int TT = T_CHUNK>
__device__ __forceinline__ void stage_logits(float* dst, const float* __restrict__ gbase, int LK,
                                             int t0, int L, int nv, const int* s_len, int vec16) {
  using Gm = Geom<K, TT>;
  const int steps = min(Gm::T, L - t0);
  const int ne = steps * K;
  if (vec16) {
    if constexpr (Gm::NQ <= NT) {
      // Fixed (row-in-group, 16-byte column) per thread: every index below except t0 is loop-invariant,
      // so one request costs a length compare and a pointer add (the flat idx -> (row, column) split
      // this replaces cost more instructions per step than the DP itself).  NQ consecutive lanes
      // fetch one row's contiguous T*K*4-byte piece.
      constexpr int RPI = NT / Gm::NQ, NIT = (NT + RPI - 1) / RPI;
      const int rr = threadIdx.x / Gm::NQ, q = threadIdx.x - rr * Gm::NQ;
      if (rr < RPI) {
        const int e = t0 * K + 4 * q;           // element offset inside the row
        const int lim_c = (t0 + steps) * K;     // end of this chunk
        const float* g = gbase + (size_t)rr * LK + e;
        float* d = dst + rr * Gm::P + 4 * q;
#pragma unroll(NIT <= 16 ? NIT : 1)
        for (int it = 0; it < NIT; ++it) {
          const int r = rr + it * RPI;
          if (r < nv && e < min(lim_c, s_len[r] * K)) cp_async16(d + it * RPI * Gm::P, g + (size_t)it * RPI * LK);
        }
      }
    } else {
      for (int idx = threadIdx.x; idx < NT * Gm::NQ; idx += NT) {
        const int r = idx / Gm::NQ, q = idx - r * Gm::NQ;
        if (r < nv) {
          const int rem = min(ne, (s_len[r] - t0) * K);
          if (4 * q < rem)
            cp_async16(dst + r * Gm::P + 4 * q, gbase + (size_t)r * LK + (size_t)t0 * K + 4 * q);
        }
      }
    }
  } else {
    for (int idx = threadIdx.x; idx < NT * Gm::CE; idx += NT) {
      const int r = idx / Gm::CE, e = idx - r * Gm::CE;
      if (r < nv) {
        const int rem = min(ne, (s_len[r] - t0) * K);
        if (e < rem) cp_async4(dst + r * Gm::P + e, gbase + (size_t)r * LK + (size_t)t0 * K + e);
      }
    }
  }
}

// Block-wide max of per-thread ints through smem scratch (NT ints).
template <int NT>
__device__ __forceinline__ int block_max_int(int v, int* scratch) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  int m = scratch[0];
#pragma unroll
  for (int w = 1; w < NT / 32; ++w) m = max(m, scratch[w]);
  __syncthreads();
  return m;
}

// Load one step-group (G steps, G*K floats) of this thread's row into registers.
template <int K>
__device__ __forceinline__ void load_group(float* xs, const float* rowp, int g) {
  using Gm = Geom<K>;
  const float4* p4 = reinterpret_cast<const float4*>(rowp + g * Gm::G * K);
#pragma unroll
  for (int q = 0; q < Gm::GQ; ++q) {
    const float4 v = p4[q];
    xs[4 * q + 0] = v.x;
    xs[4 * q + 1] = v.y;
    xs[4 * q + 2] = v.z;
    xs[4 * q + 3] = v.w;
  }
}

// Effective length of a row: never past L, and len <= 0 decodes like 1 (tf.contrib.crf quirk).
__device__ __forceinline__ int clamp_len(const int32_t* __restrict__ seq_len, int row, int L) {
  return min(max(seq_len[row], 1), L);
}

// Index of the FIRST maximum of s[0..K) (strict '>': the lowest index wins a tie); its value goes to `best`.
template <int K, bool UNROLL = Geom<K>::UNROLL>
__device__ __forceinline__ int argmax_first(const float* s, float& best) {
  constexpr int UNR = UNROLL ? K : 1;
  best = s[0];
  int y = 0;
#pragma unroll UNR
  for (int j = 1; j < K; ++j)
    if (s[j] > best) {
      best = s[j];
      y = j;
    }
  return y;
}

// Coalesced [nv, L] int32 store of a CTA's decoded tags, zero beyond each row's length.  reader(r, p) returns the tag
// of row r at position p; (r, p) of the flat index is kept incrementally: no division.
template <int NT, typename Reader>
__device__ __forceinline__ void store_tags_coalesced(int32_t* obase, int nv, int L, const int* s_len, Reader reader) {
  int r = 0, p = threadIdx.x;
  while (p >= L) {
    p -= L;
    ++r;
  }
  const int total = nv * L;
  for (int idx = threadIdx.x; idx < total; idx += NT) {
    obase[idx] = (p < s_len[r]) ? reader(r, p) : 0;
    p += NT;
    while (p >= L) {
      p -= L;
      ++r;
    }
  }
}

// Lane-per-tag kernels (crf_small.cu): a group of GS lanes holds the K-wide state of one sequence.
template <int K>
struct Lanes {
  static constexpr int GS = K <= 8 ? 8 : (K <= 16 ? 16 : 32);
  static constexpr int SPW = 32 / GS;  // sequences per warp
};

// Shared memory of the lane-per-tag Viterbi kernel: backpointers [L][32] bytes + decoded tags [SPW][L] ints.
template <int K>
constexpr size_t viterbi_lanes_smem_bytes(int L) {
  return (((size_t)L * 32 + 15) & ~(size_t)15) + (size_t)Lanes<K>::SPW * L * 4;
}

constexpr size_t kMaxSmem = 227 * 1024;  // dynamic shared memory one CTA can opt in to on sm_90

}  // namespace crf

// Small-batch (lane-per-tag) variants, crf_small.cu.  Chosen by the C-ABI entry points when
// B <= NER_CRF_SMALL_B: few sequences -> optimise the per-step critical path, not HBM throughput.
#define NER_CRF_SMALL_B 4096
int ner_crf_viterbi_small(const float* logits, const int32_t* seq_len, const float* trans, int32_t* tags_out,
                          float* best_score, int B, int L, int K, cudaStream_t st);
int ner_crf_loglik_fwd_small(const float* logits, const int32_t* tags, const int32_t* seq_len, const float* trans,
                             float* ll, float* logz, float* alpha_ws, int B, int L, int K, cudaStream_t st);
int ner_crf_loglik_bwd_small(const float* logits, const int32_t* tags, const int32_t* seq_len, const float* trans,
                             const float* alpha_ws, const float* logz, const float* d_ll, float scale, float* d_logits,
                             float* d_trans, int B, int L, int K, cudaStream_t st);

// Dispatch a runtime K in [1,32] onto `template <int K> run<K>(args...)`.
#define NER_CRF_DISPATCH_K(K_, CALL)                                                     \
  switch (K_) {                                                                          \
    case 1: CALL(1); break;   case 2: CALL(2); break;   case 3: CALL(3); break;           \
    case 4: CALL(4); break;   case 5: CALL(5); break;   case 6: CALL(6); break;           \
    case 7: CALL(7); break;   case 8: CALL(8); break;   case 9: CALL(9); break;           \
    case 10: CALL(10); break; case 11: CALL(11); break; case 12: CALL(12); break;         \
    case 13: CALL(13); break; case 14: CALL(14); break; case 15: CALL(15); break;         \
    case 16: CALL(16); break; case 17: CALL(17); break; case 18: CALL(18); break;         \
    case 19: CALL(19); break; case 20: CALL(20); break; case 21: CALL(21); break;         \
    case 22: CALL(22); break; case 23: CALL(23); break; case 24: CALL(24); break;         \
    case 25: CALL(25); break; case 26: CALL(26); break; case 27: CALL(27); break;         \
    case 28: CALL(28); break; case 29: CALL(29); break; case 30: CALL(30); break;         \
    case 31: CALL(31); break; case 32: CALL(32); break;                                   \
    default: return NER_ERR_UNSUPPORTED;                                                  \
  }
