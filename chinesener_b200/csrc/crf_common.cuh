// Shared pieces of the CRF dynamic-programming kernels (Viterbi, forward-alpha, backward), and the device code of the
// two CRF losses: the ordinary one (crf_loglik.cu, crf_bwd.cu, the loss kernels of crf_small.cu) and the
// partial-annotation one (crf_partial.cu).  Each loss kernel keeps its own loop body; the staging, the recursion
// steps, the prologues, the stores and the shared-memory sizes below are the one implementation both use.
//
// Work decomposition of the throughput kernels: ONE THREAD PER SEQUENCE, NT sequences per CTA.
// The K-wide DP state lives in registers; emission logits are streamed HBM -> smem with
// cp.async in chunks of T=8 time steps per sequence (coalesced 16-byte requests over the
// CTA's contiguous [NT, L*K] slab), then each thread reads its own row back with LDS.128.
// Row pitch P = 8K+4 floats makes P/4 odd, so the 8 threads of a quarter-warp hit 8
// distinct 16-byte bank groups (conflict-free).
#pragma once
#include <cfloat>

#include "common.cuh"

namespace crf {

using namespace nerdev;

constexpr int T_CHUNK = 8;  // time steps staged per chunk
constexpr int NSTAGE = 2;   // cp.async ring depth
constexpr int LABP = 12;    // pitch (ints) of a row's staged labels: 3 x 16B, odd -> conflict-free LDS.128

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

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
  static constexpr bool ACC_REGS = (K <= 10);  // backward: the K*K pair-marginal accumulators fit in registers
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

// Stage chunk [t0, t0+TT) of the CTA's int32 label rows (gold tags, or allowed-tag masks) into dst[NT][LABP]; steps at
// t >= s_len[r] are not fetched.
template <int NT, int TT = T_CHUNK>
__device__ __forceinline__ void stage_labels(int* dst, const int32_t* __restrict__ gbase, int L, int t0, int nv,
                                             const int* s_len, int vec16) {
  const int steps = min(TT, L - t0);
  if (vec16) {
    for (int idx = threadIdx.x; idx < NT * (TT / 4); idx += NT) {
      const int r = idx / (TT / 4), q = idx - r * (TT / 4);
      if (r < nv && 4 * q < min(steps, s_len[r] - t0))
        cp_async16(dst + r * LABP + 4 * q, gbase + (size_t)r * L + t0 + 4 * q);
    }
  } else {
    for (int idx = threadIdx.x; idx < NT * TT; idx += NT) {
      const int r = idx / TT, e = idx - r * TT;
      if (r < nv && e < min(steps, s_len[r] - t0)) cp_async4(dst + r * LABP + e, gbase + (size_t)r * L + t0 + e);
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

// Can the scaled-probability (fast) path run on this transition matrix?  Only when its entries span < 30 nats and are
// finite (a NaN fails every test).  hi gets the largest entry.
__device__ __forceinline__ bool trans_is_narrow(const float* s_tr, int KK, float& hi) {
  float lo = INFINITY;
  hi = -INFINITY;
  for (int e = 0; e < KK; ++e) {
    lo = fminf(lo, s_tr[e]);
    hi = fmaxf(hi, s_tr[e]);
  }
  return (hi - lo < 30.f) && (fabsf(hi) < 1e30f) && (fabsf(lo) < 1e30f);
}

// ------------------------------------------------------------------------------- loss forward, thread per sequence
// State of one recursion: alpha_j = lacc + ln a[j] with a[] in the probability domain (fast path), or a[j] = alpha_j
// (exact path).  Fast path, per step:
//     a_t[j] = (sum_i a_{t-1}[i] * E[i][j]) * exp(x_t[j] - xm_t),   E = exp(trans - tmax),   lacc += xm_t + tmax
// i.e. K*K FFMA + K ex2 instead of K*K exp and K log; renormalising a to max 1 adds one rcp and one lg2.

// Shared memory of the thread-per-sequence forwards: trans, E, row lengths, and a ring of logit and label chunks.
template <int K, int NT, int TT>
constexpr size_t fwd_smem_bytes() {
  using Gm = Geom<K, TT>;
  return 4 * (2 * (size_t)Gm::KK4 + NT + (size_t)NSTAGE * NT * Gm::P + (size_t)NSTAGE * NT * LABP);
}

// max of x[0..K), in max3 steps
template <int K>
__device__ __forceinline__ float row_max(const float* x) {
  constexpr int UNR = Geom<K>::UNROLL ? K : 1;
  float m = x[0];
  if (K > 1) {
#pragma unroll UNR
    for (int j = 1; j + 1 < K; j += 2) m = max3(m, x[j], x[j + 1]);
    if (K % 2 == 0) m = fmaxf(m, x[K - 1]);
  }
  return m;
}

// E[i][2q], E[i][2q+1] (0 for the pad column of an odd K): from the packed registers E2[K][(K+1)/2], or from s_E.
template <int K, bool EREG>
__device__ __forceinline__ f32x2 e_pair(const f32x2* E2, const float* s_E, int i, int q) {
  if (EREG) return E2[i * ((K + 1) / 2) + q];
  return pk2(s_E[i * K + 2 * q], 2 * q + 1 < K ? s_E[i * K + 2 * q + 1] : 0.f);
}

// First step, fast path: a = exp(x - xm), lacc = xm.
template <int K>
__device__ __forceinline__ void fwd_fast_init(float* a, float& lacc, const float* x, float xm) {
  constexpr int UNR = Geom<K>::UNROLL ? K : 1;
#pragma unroll UNR
  for (int j = 0; j < K; ++j) a[j] = fast_ex2((x[j] - xm) * kLog2e);
  lacc = xm;
}

// a <- (a · E) * exp(x - xm);  lacc += xm + tmax;  with renorm, a is rescaled to max 1 (lacc += ln max a).  xm is the
// step's emission maximum (row_max).  Per step: K*K/2 FFMA2 (a_i broadcast x column pair) + K ex2.  The rescaling
// divides by max(max a, FLT_MIN): a row with no allowed path has a = 0, which stays 0 (alpha = -inf) instead of turning
// into NaN.  Any other row has max a >= (max of the previous a) * min E, since the tag holding xm contributes
// ex2(0) = 1: at least e^-60 when every second step renormalises.
template <int K, bool EREG>
__device__ __forceinline__ void fwd_fast_step(float* a, float& lacc, const float* x, float xm, float tmax,
                                              const f32x2* E2, const float* s_E, bool renorm) {
  constexpr int UNR = Geom<K>::UNROLL ? K : 1;
  constexpr int KP = (K + 1) / 2;
  const float nx2 = -xm * kLog2e;
  // K/2 independent packed accumulators, i-outer: K/2-way ILP in the FFMA2 block
  f32x2 ns[KP];
#pragma unroll UNR
  for (int q = 0; q < KP; ++q) ns[q] = mul2(pk2(a[0], a[0]), e_pair<K, EREG>(E2, s_E, 0, q));
#pragma unroll UNR
  for (int i = 1; i < K; ++i) {
#pragma unroll UNR
    for (int q = 0; q < KP; ++q) ns[q] = fma2(pk2(a[i], a[i]), e_pair<K, EREG>(E2, s_E, i, q), ns[q]);
  }
  lacc += xm + tmax;
  float n[2 * KP];
#pragma unroll UNR
  for (int q = 0; q < KP; ++q) {
    const f32x2 arg = fma2(pk2(x[2 * q], 2 * q + 1 < K ? x[2 * q + 1] : 0.f), pk2(kLog2e, kLog2e), pk2(nx2, nx2));
    float lo, hi;
    upk2(arg, lo, hi);
    ns[q] = mul2(ns[q], pk2(fast_ex2(lo), fast_ex2(hi)));
    if (renorm) upk2(ns[q], n[2 * q], n[2 * q + 1]);
  }
  if (renorm) {
    const float m = fmaxf(row_max<K>(n), FLT_MIN);
    const float r = __fdividef(1.f, m);
    lacc = fmaf(kLn2, fast_lg2(m), lacc);
#pragma unroll UNR
    for (int q = 0; q < KP; ++q) ns[q] = mul2(ns[q], pk2(r, r));
  }
#pragma unroll UNR
  for (int q = 0; q < KP; ++q) {
    float lo, hi;
    upk2(ns[q], lo, hi);
    a[2 * q] = lo;
    if (2 * q + 1 < K) a[2 * q + 1] = hi;
  }
}

// Exact path: a[j] <- x[j] + logsumexp_i(a[i] + trans[i][j]), each column with its own max (reduce_logsumexp, with
// its finite-max guard).
template <int K>
__device__ __forceinline__ void fwd_exact_step(float* a, const float* x, const float* s_tr) {
  constexpr int UNR = Geom<K>::UNROLL ? K : 1;
  float na[K];
#pragma unroll UNR
  for (int j = 0; j < K; ++j) {
    float m = -INFINITY;
#pragma unroll UNR
    for (int i = 0; i < K; ++i) m = fmaxf(m, a[i] + s_tr[i * K + j]);
    const float mm = (fabsf(m) <= 3.0e38f) ? m : 0.f;
    float sum = 0.f;
#pragma unroll UNR
    for (int i = 0; i < K; ++i) sum += expf(a[i] + s_tr[i * K + j] - mm);
    na[j] = x[j] + (logf(sum) + mm);
  }
#pragma unroll UNR
  for (int j = 0; j < K; ++j) a[j] = na[j];
}

// alpha_t into the workspace row dst[K].
template <int K>
__device__ __forceinline__ void store_alpha(float* dst, const float* a, float lacc, bool fast) {
  constexpr int UNR = Geom<K>::UNROLL ? K : 1;
#pragma unroll UNR
  for (int j = 0; j < K; ++j) dst[j] = fast ? fmaf(kLn2, fast_lg2(a[j]), lacc) : a[j];
}

// log Z = logsumexp_j alpha_j of the last step.
template <int K>
__device__ __forceinline__ float fwd_logz(const float* a, float lacc, bool fast) {
  constexpr int UNR = Geom<K>::UNROLL ? K : 1;
  if (fast) {
    float sum = 0.f;
#pragma unroll UNR
    for (int j = 0; j < K; ++j) sum += a[j];
    return lacc + logf(sum);
  }
  float m = a[0];
#pragma unroll UNR
  for (int j = 1; j < K; ++j) m = fmaxf(m, a[j]);
  const float mm = (fabsf(m) <= 3.0e38f) ? m : 0.f;
  float sum = 0.f;
#pragma unroll UNR
  for (int j = 0; j < K; ++j) sum += expf(a[j] - mm);
  return logf(sum) + mm;
}

// ------------------------------------------------------------------------------ loss backward, thread per sequence
// One thread walks t = len-1 .. 0 with beta[K] in registers; logits, the forward's alpha and the labels are streamed
// in reverse, and d_logits goes back through the logits' tile so the HBM store is coalesced.

// Shared memory of the thread-per-sequence backwards: trans, E, the CTA's d_trans, row maxima [32], row lengths, and a
// ring of NF staged float tensors (logits and the forward's alphas) plus the label chunks.
template <int K, int NT, int NF>
constexpr size_t bwd_smem_bytes() {
  using Gm = Geom<K>;
  return 4 * (3 * (size_t)Gm::KK4 + 32 + NT + (size_t)NF * NSTAGE * NT * Gm::P + (size_t)NSTAGE * NT * LABP);
}

// trans -> s_tr, s_dT = 0, row lengths -> s_len, E[i][j] = exp(trans[i][j] - rmax[i]) when the fast path applies.
// Returns whether it does; bmax gets the CTA's longest row.
template <int K, int NT>
__device__ __forceinline__ bool bwd_prologue(const float* __restrict__ trans, int mylen, float* s_tr, float* s_E,
                                             float* s_dT, float* s_rmax, int* s_len, int* scratch, int& bmax) {
  const int tid = threadIdx.x;
  for (int e = tid; e < K * K; e += NT) {
    s_tr[e] = trans[e];
    s_dT[e] = 0.f;
  }
  s_len[tid] = mylen;
  bmax = block_max_int<NT>(mylen, scratch);
  if (tid < K) {
    float rm = -INFINITY;
    for (int j = 0; j < K; ++j) rm = fmaxf(rm, s_tr[tid * K + j]);
    s_rmax[tid] = rm;
  }
  __syncthreads();
  float hi;
  const bool fast = trans_is_narrow(s_tr, K * K, hi);
  for (int e = tid; e < K * K; e += NT) s_E[e] = fast ? expf(s_tr[e] - s_rmax[e / K]) : 0.f;
  __syncthreads();
  return fast;
}

// d_logits of the chunks past the CTA's longest row (from chunk nchunk on) are zero.
template <int K, int NT>
__device__ __forceinline__ void zero_dlogits_tail(float* gd, int nv, int L, int nchunk) {
  using Gm = Geom<K>;
  const int LK = L * K;
  for (int c = nchunk; c < (L + Gm::T - 1) / Gm::T; ++c) {
    const int t0 = c * Gm::T;
    const int ne = min(Gm::T, L - t0) * K;
    for (int idx = threadIdx.x; idx < NT * Gm::CE; idx += NT) {
      const int r = idx / Gm::CE, e = idx - r * Gm::CE;
      if (r < nv && e < ne) gd[(size_t)r * LK + (size_t)t0 * K + e] = 0.f;
    }
  }
}

// beta[i] <- logsumexp_j(trans[i][j] + u[j]).  Fast path through E and the row maxima rmax, leaving q = exp(u - mq)
// and mq for the next pair marginal; exact path with each row's own max, leaving uk = u (q and uk may be one array).
template <int K>
__device__ __forceinline__ void beta_step(bool fast, float* beta, float* q, float& mq, float* uk, const float* u,
                                          const float* s_tr, const float* s_E, const float* rmax) {
  constexpr int UNR = Geom<K>::UNROLL ? K : 1;
  if (fast) {
    float m = u[0];
#pragma unroll UNR
    for (int j = 1; j < K; ++j) m = fmaxf(m, u[j]);
    mq = m;
#pragma unroll UNR
    for (int j = 0; j < K; ++j) q[j] = __expf(u[j] - m);
#pragma unroll UNR
    for (int i = 0; i < K; ++i) {
      float sum = 0.f;
#pragma unroll UNR
      for (int j = 0; j < K; ++j) sum = fmaf(s_E[i * K + j], q[j], sum);
      beta[i] = m + rmax[i] + __logf(sum);
    }
  } else {
    float nb[K];
#pragma unroll UNR
    for (int i = 0; i < K; ++i) {
      float m = -INFINITY;
#pragma unroll UNR
      for (int j = 0; j < K; ++j) m = fmaxf(m, s_tr[i * K + j] + u[j]);
      const float mm = (fabsf(m) <= 3.0e38f) ? m : 0.f;
      float sum = 0.f;
#pragma unroll UNR
      for (int j = 0; j < K; ++j) sum += expf(s_tr[i * K + j] + u[j] - mm);
      nb[i] = logf(sum) + mm;
    }
#pragma unroll UNR
    for (int i = 0; i < K; ++i) {
      beta[i] = nb[i];
      uk[i] = u[i];
    }
  }
}

// Coalesced store of chunk t0's d_logits from the staged tile sx[NT][P]; zero at t >= s_len[r].
template <int K, int NT>
__device__ __forceinline__ void store_dlogits_chunk(float* gd, const float* sx, const int* s_len, int nv, int L,
                                                    int t0, int vec) {
  using Gm = Geom<K>;
  const int LK = L * K;
  const int ne = min(Gm::T, L - t0) * K;
  if (vec) {
    for (int idx = threadIdx.x; idx < NT * Gm::NQ; idx += NT) {
      const int r = idx / Gm::NQ, qq = idx - r * Gm::NQ;
      if (r < nv && 4 * qq < ne) {
        const int valid = (s_len[r] - t0) * K;  // elements [0, valid) carry gradients
        float4 v = *reinterpret_cast<const float4*>(sx + r * Gm::P + 4 * qq);
        if (4 * qq + 0 >= valid) v.x = 0.f;
        if (4 * qq + 1 >= valid) v.y = 0.f;
        if (4 * qq + 2 >= valid) v.z = 0.f;
        if (4 * qq + 3 >= valid) v.w = 0.f;
        *reinterpret_cast<float4*>(gd + (size_t)r * LK + (size_t)t0 * K + 4 * qq) = v;
      }
    }
  } else {
    for (int idx = threadIdx.x; idx < NT * Gm::CE; idx += NT) {
      const int r = idx / Gm::CE, e = idx - r * Gm::CE;
      if (r < nv && e < ne) {
        const int valid = (s_len[r] - t0) * K;
        gd[(size_t)r * LK + (size_t)t0 * K + e] = (e < valid) ? sx[r * Gm::P + e] : 0.f;
      }
    }
  }
}

// d_trans += coef * acc * E (the per-thread register accumulators of the fast path, warp-reduced into s_dT) plus what
// the CTA gathered in s_dT.
template <int K, int NT>
__device__ __forceinline__ void flush_dtrans(const float* acc, float coef, bool active, float* s_dT, const float* s_E,
                                             float* d_trans) {
  if constexpr (Geom<K>::ACC_REGS) {
#pragma unroll
    for (int e = 0; e < K * K; ++e) {
      float v = active ? coef * acc[e] * s_E[e] : 0.f;
      v = warp_sum(v);
      if ((threadIdx.x & 31) == 0 && v != 0.f) atomicAdd(&s_dT[e], v);
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < K * K; e += NT) {
    const float v = s_dT[e];
    if (v != 0.f) atomicAdd(&d_trans[e], v);
  }
}

// The thread-per-sequence kernels run 64-thread CTAs above 128 rows per SM (a backward only where their shared memory
// fits), 32-thread CTAs otherwise.
inline bool use_cta64(int B) { return B > ner_num_sms() * 64 * 2; }

// ----------------------------------------------------------------------------------------------- lane per tag
// Lane-per-tag kernels (crf_small.cu, crf_partial.cu): a group of GS lanes holds the K-wide state of one sequence.
template <int K>
struct Lanes {
  static constexpr int GS = K <= 8 ? 8 : (K <= 16 ? 16 : 32);
  static constexpr int SPW = 32 / GS;  // sequences per warp
};

// The warp's longest row: the trip count of a lane-per-tag kernel's lock-step loop.
__device__ __forceinline__ int lanes_wmax(int len) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) len = max(len, __shfl_xor_sync(0xffffffffu, len, o));
  return len;
}

// x + logsumexp_i(a_i + trans[i][j]) over the group's lanes (tc[i] = trans[i][j] of this lane's tag j), exact with
// its own max.
template <int K>
__device__ __forceinline__ float lanes_alpha_step(float a, float x, const float* tc, int g) {
  constexpr int GS = Lanes<K>::GS;
  float v[K];
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < K; ++i) {
    v[i] = __shfl_sync(0xffffffffu, a, g * GS + i) + tc[i];
    m = fmaxf(m, v[i]);
  }
  const float mm = (fabsf(m) <= 3.0e38f) ? m : 0.f;
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < K; ++i) sum += __expf(v[i] - mm);
  return x + (__logf(sum) + mm);
}

// logsumexp_j a_j over the group's lanes (every lane of the group gets it).
template <int K>
__device__ __forceinline__ float lanes_logsumexp(float a, bool tag_ok) {
  constexpr int GS = Lanes<K>::GS;
  float m = a;
#pragma unroll
  for (int o = GS / 2; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o, GS));
  const float mm = (fabsf(m) <= 3.0e38f) ? m : 0.f;
  float e = tag_ok ? expf(a - mm) : 0.f;
#pragma unroll
  for (int o = GS / 2; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o, GS);
  return logf(e) + mm;
}

// Backward: v[j] = tr[j] + w_j, with w_j from lane j of the group (tr = row i of trans for this lane's tag i).
// Returns max_j v[j].
template <int K>
__device__ __forceinline__ float lanes_gather(float* v, float w, const float* tr, int g) {
  constexpr int GS = Lanes<K>::GS;
  float m = -INFINITY;
#pragma unroll
  for (int j = 0; j < K; ++j) {
    v[j] = tr[j] + __shfl_sync(0xffffffffu, w, g * GS + j);
    m = fmaxf(m, v[j]);
  }
  return m;
}

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
