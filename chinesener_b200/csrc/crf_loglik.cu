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
// own max, exactly as the reference's reduce_logsumexp does.  The steps themselves are crf_common.cuh's, shared with
// the partial-annotation loss (crf_partial.cu).
#include "crf_common.cuh"

namespace {

using namespace crf;

template <int K, int NT, int TT, bool EREG, int MINB>
__global__ void __launch_bounds__(NT, MINB)
crf_loglik_fwd_kernel(const float* __restrict__ logits, const int32_t* __restrict__ tags,
                      const int32_t* __restrict__ seq_len, const float* __restrict__ trans,
                      float* __restrict__ ll, float* __restrict__ logz_out,
                      float* __restrict__ alpha_ws, int B, int L, int vec_logits, int vec_tags,
                      int force_exact) {
  using Gm = Geom<K, TT>;
  constexpr int T = Gm::T, G = Gm::G, P = Gm::P;
  constexpr int UNR = Gm::UNROLL ? K : 1;

  extern __shared__ __align__(16) float smem[];
  float* s_tr = smem;                                   // raw trans [i][j]
  float* s_E = s_tr + Gm::KK4;                          // exp(trans - tmax) [i][j]
  int* s_len = reinterpret_cast<int*>(s_E + Gm::KK4);   // [NT]
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
  float tmax;
  const bool fast = trans_is_narrow(s_tr, K * K, tmax) && !force_exact;
  if (!fast) tmax = 0.f;
  for (int e = tid; e < K * K; e += NT) s_E[e] = fast ? expf(s_tr[e] - tmax) : 0.f;
  __syncthreads();

  const float* gbase = logits + (size_t)row0 * LK;
  const int32_t* tbase = tags + (size_t)row0 * L;
  const int nchunk = (bmax + T - 1) / T;

#pragma unroll
  for (int s = 0; s < NSTAGE - 1; ++s) {
    if (s < nchunk) {
      stage_logits<K, NT, TT>(s_stage + s * NT * P, gbase, LK, s * T, L, nv, s_len, vec_logits);
      stage_labels<NT, TT>(s_tags + s * NT * LABP, tbase, L, s * T, nv, s_len, vec_tags);
    }
    cp_async_commit();
  }

  // E as packed column pairs: E2[i][q] = (E[i][2q], E[i][2q+1]) (hi lane 0 for the pad column of an odd K)
  constexpr int KP = (K + 1) / 2;
  f32x2 E2[EREG ? K * KP : 1];
  if (EREG) {
#pragma unroll
    for (int i = 0; i < K; ++i)
#pragma unroll
      for (int q = 0; q < KP; ++q) E2[i * KP + q] = pk2(s_E[i * K + 2 * q], 2 * q + 1 < K ? s_E[i * K + 2 * q + 1] : 0.f);
  }
  float a[K];
  float lacc = 0.f;
#pragma unroll UNR
  for (int j = 0; j < K; ++j) a[j] = 0.f;
  auto fast_step = [&](const float* x, bool renorm) {
    fwd_fast_step<K, EREG>(a, lacc, x, row_max<K>(x), tmax, E2, s_E, renorm);
  };

  float score = 0.f;
  int prev = 0;
  float* aws = (alpha_ws != nullptr && tid < nv) ? alpha_ws + (size_t)(row0 + tid) * LK : nullptr;

  for (int c = 0; c < nchunk; ++c) {
    const int cn = c + NSTAGE - 1;
    if (cn < nchunk) {
      stage_logits<K, NT, TT>(s_stage + (cn % NSTAGE) * NT * P, gbase, LK, cn * T, L, nv, s_len, vec_logits);
      stage_labels<NT, TT>(s_tags + (cn % NSTAGE) * NT * LABP, tbase, L, cn * T, nv, s_len, vec_tags);
    }
    cp_async_commit();
    cp_async_wait<NSTAGE - 1>();
    __syncthreads();

    const int t0 = c * T;
    if (tid < nv && t0 < mylen) {
      const float* rowp = s_stage + (c % NSTAGE) * NT * P + tid * P;
      int tg[T];
      {
        const int4* tp = reinterpret_cast<const int4*>(s_tags + (c % NSTAGE) * NT * LABP + tid * LABP);
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
            if (aws != nullptr) store_alpha<K>(aws + (size_t)(t0 + tt) * K, a, lacc, fast);
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
                  fwd_fast_init<K>(a, lacc, xs + gg * K, row_max<K>(xs + gg * K));
                } else {
#pragma unroll UNR
                  for (int j = 0; j < K; ++j) a[j] = xs[gg * K + j];
                }
              } else if (fast) {
                fast_step(xs + gg * K, true);
              } else {
                fwd_exact_step<K>(a, xs + gg * K, s_tr);
              }
              if (aws != nullptr) store_alpha<K>(aws + (size_t)t * K, a, lacc, fast);
            }
          }
        }
      }
    }
    __syncthreads();
  }

  if (tid < nv) {
    float logz = fwd_logz<K>(a, lacc, fast);
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
  const size_t smem = fwd_smem_bytes<K, NT, TT>();
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
  if (use_cta64(B))
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
  if (B <= NER_CRF_SMALL_B && !(flags & 2))  // flags bit1: force the throughput kernel (tests / benches)
    return ner_crf_loglik_fwd_small(logits, tags, seq_len, trans, ll, logz_out, alpha_ws, B, L, K, st);
#define CALL(KK) return launch_fwd<KK>(logits, tags, seq_len, trans, ll, logz_out, alpha_ws, B, L, flags, st)
  NER_CRF_DISPATCH_K(K, CALL)
#undef CALL
  return NER_ERR_UNSUPPORTED;
}
