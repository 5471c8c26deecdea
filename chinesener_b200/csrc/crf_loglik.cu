// CRF log-likelihood (gold-path score minus forward-alpha log-partition) for sm_90a —
// replaces tf.contrib.crf.crf_log_likelihood as called at reference tools/layer.py:122-127
// (crf_sequence_score / crf_log_norm semantics restated in SURVEY.md Appendix A.1).
//
// One thread per sequence; alpha[K] in registers.  Fast path (default, used when the
// transition matrix spans < 30 nats): the K*K logsumexp of one step is evaluated in the
// scaled-probability domain,
//     alpha_t[j] = lacc_t + ln p_t[j],   p_t[j] = (sum_i p_{t-1}[i] * E[i][j]) * exp(x_t[j] - max_j x_t[j]),
//     E = exp(trans - tmax),  lacc_t = lacc_{t-1} + max_j x_t[j] + tmax,   p renormalised to max 1
//     every other step (lacc += ln max p)
// i.e. K*K FFMA + K ex2 per step (+ one rcp / lg2 per two steps) instead of K*K exp and K log.  Chunks that lie completely inside a sequence (the common case) run a branch-free
// unrolled body; only the first and the ragged last chunk take the checked path.  The exact path (flags bit0, or
// chosen automatically for wide/inf transition matrices) evaluates every logsumexp with its
// own max, exactly as the reference's reduce_logsumexp does.
#include "crf_common.cuh"

namespace {

using namespace crf;

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
constexpr int TAGP = 12;  // tag-chunk pitch (ints): 3 x 16B, odd -> conflict-free LDS.128

template <int K, int NT, int TT>
size_t loglik_smem_bytes() {
  using Gm = Geom<K, TT>;
  size_t words = 2 * Gm::KK4 + 32 + NT + (size_t)NSTAGE * NT * Gm::P + (size_t)NSTAGE * NT * TAGP;
  return words * 4;
}

template <int NT, int TT>
__device__ __forceinline__ void stage_tags(int* dst, const int32_t* __restrict__ gbase, int L, int t0,
                                           int nv, const int* s_len, int vec16) {
  constexpr int T = TT;
  const int steps = min(T, L - t0);
  if (vec16) {
    for (int idx = threadIdx.x; idx < NT * (T / 4); idx += NT) {
      const int r = idx / (T / 4), q = idx - r * (T / 4);
      if (r < nv && 4 * q < min(steps, s_len[r] - t0))
        cp_async16(dst + r * TAGP + 4 * q, gbase + (size_t)r * L + t0 + 4 * q);
    }
  } else {
    for (int idx = threadIdx.x; idx < NT * T; idx += NT) {
      const int r = idx / T, e = idx - r * T;
      if (r < nv && e < min(steps, s_len[r] - t0))
        cp_async4(dst + r * TAGP + e, gbase + (size_t)r * L + t0 + e);
    }
  }
}

template <int K, int NT, int TT, bool EREG, int MINB>
__global__ void __launch_bounds__(NT, MINB)
crf_loglik_fwd_kernel(const float* __restrict__ logits, const int32_t* __restrict__ tags,
                      const int32_t* __restrict__ seq_len, const float* __restrict__ trans,
                      float* __restrict__ ll, float* __restrict__ logz_out,
                      float* __restrict__ alpha_ws, int B, int L, int vec_logits, int vec_tags,
                      int force_exact) {
  using Gm = Geom<K, TT>;
  constexpr int T = Gm::T, G = Gm::G, P = Gm::P;
  constexpr bool E_REGS = EREG;
  constexpr int UNR = Gm::UNROLL ? K : 1;

  extern __shared__ __align__(16) float smem[];
  float* s_tr = smem;                                   // raw trans [i][j]
  float* s_E = s_tr + Gm::KK4;                          // exp(trans - cmax[j]) stored [i][j]
  float* s_cmax = s_E + Gm::KK4;                        // [32]
  int* s_len = reinterpret_cast<int*>(s_cmax + 32);     // [NT]
  float* s_stage = reinterpret_cast<float*>(s_len + NT);
  int* s_tags = reinterpret_cast<int*>(s_stage + NSTAGE * NT * P);

  const int tid = threadIdx.x;
  const int row0 = blockIdx.x * NT;
  const int nv = min(NT, B - row0);
  const int LK = L * K;

  for (int e = tid; e < K * K; e += NT) s_tr[e] = trans[e];
  int rawlen = 0, mylen = 1;
  if (tid < nv) {
    rawlen = seq_len[row0 + tid];
    mylen = min(max(rawlen, 1), L);
  }
  s_len[tid] = mylen;
  const int bmax = block_max_int<NT>(tid < nv ? mylen : 1, reinterpret_cast<int*>(s_stage));

  // column maxima, range test, E matrix (tiny; every thread helps)
  if (tid < K) {
    float cm = -INFINITY;
    for (int i = 0; i < K; ++i) cm = fmaxf(cm, s_tr[i * K + tid]);
    s_cmax[tid] = cm;
  }
  __syncthreads();
  bool fast = !force_exact;
  float tmax = 0.f;
  {
    float lo = INFINITY, hi = -INFINITY;
    for (int e = 0; e < K * K; ++e) {
      const float v = s_tr[e];
      lo = fminf(lo, v);
      hi = fmaxf(hi, v);
    }
    if (!(hi - lo < 30.f) || !(fabsf(hi) < 1e30f) || !(fabsf(lo) < 1e30f)) fast = false;  // also NaN/inf
    tmax = fast ? hi : 0.f;
  }
  for (int e = tid; e < K * K; e += NT) s_E[e] = fast ? expf(s_tr[e] - tmax) : 0.f;
  __syncthreads();

  const float* gbase = logits + (size_t)row0 * LK;
  const int32_t* tbase = tags + (size_t)row0 * L;
  const int nchunk = (bmax + T - 1) / T;

#pragma unroll
  for (int s = 0; s < NSTAGE - 1; ++s) {
    if (s < nchunk) {
      stage_logits<K, NT, TT>(s_stage + s * NT * P, gbase, LK, s * T, L, nv, s_len, vec_logits);
      stage_tags<NT, TT>(s_tags + s * NT * TAGP, tbase, L, s * T, nv, s_len, vec_tags);
    }
    cp_async_commit();
  }

  // E as packed column pairs: E2[i][q] = (E[i][2q], E[i][2q+1]) (hi lane 0 for the pad column of an odd K)
  constexpr int KP = (K + 1) / 2;
  f32x2 E2[E_REGS ? K * KP : 1];
  if (E_REGS) {
#pragma unroll
    for (int i = 0; i < K; ++i)
#pragma unroll
      for (int q = 0; q < KP; ++q) E2[i * KP + q] = pk2(s_E[i * K + 2 * q], 2 * q + 1 < K ? s_E[i * K + 2 * q + 1] : 0.f);
  }
  auto e2 = [&](int i, int q) -> f32x2 {
    if (E_REGS) return E2[i * KP + q];
    return pk2(s_E[i * K + 2 * q], 2 * q + 1 < K ? s_E[i * K + 2 * q + 1] : 0.f);
  };
  // Fast path state: alpha_j = lacc + ln(a[j]) with a[] kept in the PROBABILITY domain and
  // renormalised (max -> 1) every other step; exact path state: a[j] = alpha_j.
  float a[K];
  float lacc = 0.f;
#pragma unroll UNR
  for (int j = 0; j < K; ++j) a[j] = 0.f;
  // a <- (a · E) * exp(x - max x);  lacc += max x + tmax   [+ renormalisation]
  // per step: K*K/2 FFMA2 (a_i broadcast x column pair) + K ex2 (+ 1 rcp + 1 lg2 when renormalising)
  auto fast_step = [&](const float* x, bool renorm) {
    float xm = x[0];
    if (K > 1) {
#pragma unroll UNR
      for (int j = 1; j + 1 < K; j += 2) xm = max3(xm, x[j], x[j + 1]);
      if (K % 2 == 0) xm = fmaxf(xm, x[K - 1]);
    }
    const float nx2 = -xm * kLog2e;
    // K/2 independent packed accumulators, i-outer: K/2-way ILP in the FFMA2 block
    f32x2 ns[KP];
#pragma unroll UNR
    for (int q = 0; q < KP; ++q) ns[q] = mul2(pk2(a[0], a[0]), e2(0, q));
#pragma unroll UNR
    for (int i = 1; i < K; ++i) {
#pragma unroll UNR
      for (int q = 0; q < KP; ++q) ns[q] = fma2(pk2(a[i], a[i]), e2(i, q), ns[q]);
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
      float m = n[0];
      if (K > 1) {
#pragma unroll UNR
        for (int j = 1; j + 1 < K; j += 2) m = max3(m, n[j], n[j + 1]);
        if (K % 2 == 0) m = fmaxf(m, n[K - 1]);
      }
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
  };
  auto fast_init = [&](const float* x) {
    float xm = x[0];
#pragma unroll UNR
    for (int j = 1; j < K; ++j) xm = fmaxf(xm, x[j]);
#pragma unroll UNR
    for (int j = 0; j < K; ++j) a[j] = fast_ex2((x[j] - xm) * kLog2e);
    lacc = xm;
  };
  auto store_alpha = [&](float* dst) {
#pragma unroll UNR
    for (int j = 0; j < K; ++j) dst[j] = fast ? fmaf(kLn2, fast_lg2(a[j]), lacc) : a[j];
  };

  float score = 0.f;
  int prev = 0;
  float* aws = (alpha_ws != nullptr && tid < nv) ? alpha_ws + (size_t)(row0 + tid) * LK : nullptr;

  for (int c = 0; c < nchunk; ++c) {
    const int cn = c + NSTAGE - 1;
    if (cn < nchunk) {
      stage_logits<K, NT, TT>(s_stage + (cn % NSTAGE) * NT * P, gbase, LK, cn * T, L, nv, s_len, vec_logits);
      stage_tags<NT, TT>(s_tags + (cn % NSTAGE) * NT * TAGP, tbase, L, cn * T, nv, s_len, vec_tags);
    }
    cp_async_commit();
    cp_async_wait<NSTAGE - 1>();
    __syncthreads();

    const int t0 = c * T;
    if (tid < nv && t0 < mylen) {
      const float* rowp = s_stage + (c % NSTAGE) * NT * P + tid * P;
      int tg[T];
      {
        const int4* tp = reinterpret_cast<const int4*>(s_tags + (c % NSTAGE) * NT * TAGP + tid * TAGP);
#pragma unroll
        for (int q = 0; q < T / 4; ++q) {
          const int4 v = tp[q];
          tg[4 * q + 0] = v.x;
          tg[4 * q + 1] = v.y;
          tg[4 * q + 2] = v.z;
          tg[4 * q + 3] = v.w;
        }
      }
      if (fast && t0 > 0 && t0 + T <= mylen) {
        // ---- whole chunk inside the sequence: branch-free body
#pragma unroll
        for (int g = 0; g < T / G; ++g) {
          float xs[G * K];
          load_group<K>(xs, rowp, g);
#pragma unroll
          for (int gg = 0; gg < G; ++gg) {
            const int tt = g * G + gg;
            const int tag = min(max(tg[tt], 0), K - 1);
            score += rowp[tt * K + tag] + s_tr[prev * K + tag];
            prev = tag;
            fast_step(xs + gg * K, (tt & 1) != 0 || T < 2);
            if (aws != nullptr) store_alpha(aws + (size_t)(t0 + tt) * K);
          }
        }
      } else
#pragma unroll
      for (int g = 0; g < T / G; ++g) {
        if (t0 + g * G < mylen) {
          float xs[G * K];
          load_group<K>(xs, rowp, g);
#pragma unroll
          for (int gg = 0; gg < G; ++gg) {
            const int tt = g * G + gg;
            const int t = t0 + tt;
            if (t < mylen) {
              // ---- gold path (crf_unary_score + crf_binary_score)
              const int tag = min(max(tg[tt], 0), K - 1);
              score += rowp[tt * K + tag];
              if (t > 0) score += s_tr[prev * K + tag];
              prev = tag;
              // ---- forward-alpha (crf_log_norm)
              if (t == 0) {
                if (fast) {
                  fast_init(xs + gg * K);
                } else {
#pragma unroll UNR
                  for (int j = 0; j < K; ++j) a[j] = xs[gg * K + j];
                }
              } else if (fast) {
                fast_step(xs + gg * K, true);
              } else {
                float na[K];
#pragma unroll UNR
                for (int j = 0; j < K; ++j) {
                  float m = -INFINITY;
#pragma unroll UNR
                  for (int i = 0; i < K; ++i) m = fmaxf(m, a[i] + s_tr[i * K + j]);
                  const float mm = (fabsf(m) <= 3.0e38f) ? m : 0.f;  // reduce_logsumexp's finite-max guard
                  float sum = 0.f;
#pragma unroll UNR
                  for (int i = 0; i < K; ++i) sum += expf(a[i] + s_tr[i * K + j] - mm);
                  na[j] = xs[gg * K + j] + (logf(sum) + mm);
                }
#pragma unroll UNR
                for (int j = 0; j < K; ++j) a[j] = na[j];
              }
              if (aws != nullptr) store_alpha(aws + (size_t)t * K);
            }
          }
        }
      }
    }
    __syncthreads();
  }

  if (tid < nv) {
    float logz;
    if (fast) {
      float sum = 0.f;
#pragma unroll UNR
      for (int j = 0; j < K; ++j) sum += a[j];
      logz = lacc + logf(sum);
    } else {
      float m = a[0];
#pragma unroll UNR
      for (int j = 1; j < K; ++j) m = fmaxf(m, a[j]);
      const float mm = (fabsf(m) <= 3.0e38f) ? m : 0.f;
      float sum = 0.f;
#pragma unroll UNR
      for (int j = 0; j < K; ++j) sum += expf(a[j] - mm);
      logz = logf(sum) + mm;
    }
    if (rawlen <= 0) {  // crf_log_norm / crf_sequence_score: zero for empty sequences
      logz = 0.f;
      score = 0.f;
    }
    ll[row0 + tid] = score - logz;
    if (logz_out != nullptr) logz_out[row0 + tid] = logz;
  }
}

template <int K, int NT, int TT, bool EREG, int MINB = 1>
int launch_fwd_nt(const float* logits, const int32_t* tags, const int32_t* seq_len,
                  const float* trans, float* ll, float* logz, float* alpha_ws, int B, int L,
                  int flags, cudaStream_t st) {
  const size_t smem = loglik_smem_bytes<K, NT, TT>();
  auto kern = crf_loglik_fwd_kernel<K, NT, TT, EREG, MINB>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  const int vl = ((L * K) % 4 == 0) && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0);
  const int vt = (L % 4 == 0) && ((reinterpret_cast<uintptr_t>(tags) & 15) == 0);
  const int grid = (B + NT - 1) / NT;
  kern<<<grid, NT, smem, st>>>(logits, tags, seq_len, trans, ll, logz, alpha_ws, B, L, vl, vt, flags & 1);
  return ner_launch_status();
}

template <int K>
int launch_fwd(const float* logits, const int32_t* tags, const int32_t* seq_len, const float* trans,
               float* ll, float* logz, float* alpha_ws, int B, int L, int flags, cudaStream_t st) {
  constexpr bool ER = (K <= 10);
  // big batches: 4-step chunks (30 KB smem / CTA) and <= 170 registers: 6 CTAs = 12 warps per SM
  if (B > ner_num_sms() * 64 * 2)
    return launch_fwd_nt<K, 64, 4, ER, 6>(logits, tags, seq_len, trans, ll, logz, alpha_ws, B, L, flags, st);
  return launch_fwd_nt<K, 32, T_CHUNK, ER>(logits, tags, seq_len, trans, ll, logz, alpha_ws, B, L, flags, st);
}

}  // namespace

extern "C" int ner_crf_loglik_fwd(const float* logits, const int32_t* tags, const int32_t* seq_len,
                                  const float* trans, float* ll, float* logz_out, float* alpha_ws,
                                  int B, int L, int K, int flags, ner_stream_t stream) {
  if (B < 0 || L < 1 || K < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!logits || !tags || !seq_len || !trans || !ll) return NER_ERR_INVALID_ARG;
  if (K > NER_MAX_TAGS) return NER_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (B <= NER_CRF_SMALL_B && !(flags & 2)) {  // flags bit1: force the throughput kernel (tests / benches)
    const int rc = ner_crf_loglik_fwd_small(logits, tags, seq_len, trans, ll, logz_out, alpha_ws, B, L, K, st);
    if (rc != NER_ERR_UNSUPPORTED) return rc;
  }
#define CALL(KK) return launch_fwd<KK>(logits, tags, seq_len, trans, ll, logz_out, alpha_ws, B, L, flags, st)
  NER_CRF_DISPATCH_K(K, CALL)
#undef CALL
  return NER_ERR_UNSUPPORTED;
}
