// CRF-to-CRF knowledge distillation: the KL divergence between a teacher CRF's distribution over all tag paths and a
// student CRF's, and its gradient in the student's potentials, sm_90a.  Both CRFs share the tag space.  For row b of
// length n, with potentials x[t][j], transitions T[i][j] and p^tau(y) ~ exp(s(y) / tau):
//     KL_b = sum_t mu_T[t]·(x_T - x_S)[t] / tau + sum_{t>=1} xi_T[t]·(T_T - T_S) / tau - logZ_T + logZ_S
//     d KL_b / d x_S[t][j]  = (mu_S[t][j] - mu_T[t][j]) / tau
//     d KL_b / d T_S[i][j]  = sum_{t>=1} (xi_S[t][i][j] - xi_T[t][i][j]) / tau
// mu / xi are the unary / pairwise marginals of p^tau, logZ its partition (DESIGN.md §3.3).  A term whose teacher
// marginal is 0 adds 0 (a teacher transition of -inf), and a row with seq_len <= 0 has KL = 0 and no gradient.
//
// The forward runs the teacher's and the student's alpha recursion in one pass over both emission tensors; the
// backward runs both beta recursions in one reverse pass, and gets KL_b from the marginals it forms anyway.  1/tau is
// applied to every emission and transition as it is read: there are no scaled copies.  The two recursions run the same
// instructions on their own inputs, so a teacher equal to the student gives KL = 0.0 and d_s_logits = d_s_trans = 0
// exactly.  The fast scaled-probability step runs only when both scaled transition matrices pass trans_is_narrow;
// otherwise (or with flags bit0) both recursions take the exact per-column logsumexp.
//
// Route (a function of the call's shape only, as for the other CRF losses):
//   B <= NER_CRF_SMALL_B  lane per tag (as crf_small.cu), exact logsumexp, forward and backward.
//   forward   thread per sequence; 64-thread CTAs with 4-step chunks above 128 rows per SM, else 32-thread CTAs.
//   backward  thread per sequence on a four-tensor staging ring (both emissions, both alphas); 64-thread CTAs under
//             the same rule where the ring fits in shared memory, 32-thread CTAs where that fits (K <= 25), else the
//             lane-per-tag kernel at any B.
// Workspace: alpha_ws [2][B][L][K] = (alpha_T, alpha_S) in the log domain; logz [B][2] = (logZ_T, logZ_S).
#include "crf_common.cuh"

namespace {

using namespace crf;

constexpr int kMaxLen = 4095;  // document mode's longest row

template <int K>
struct Alpha {
  float a[K];
  float lacc;
};

// Both transition matrices scaled by inv_temp into shared memory; returns whether the fast path may run on both
// (hi_t / hi_s get their largest entries).
template <int K, int NT>
__device__ __forceinline__ bool load_trans_pair(const float* __restrict__ t_trans, const float* __restrict__ s_trans,
                                                float inv_temp, float* s_trt, float* s_trs, float& hi_t, float& hi_s) {
  for (int e = threadIdx.x; e < K * K; e += NT) {
    s_trt[e] = t_trans[e] * inv_temp;
    s_trs[e] = s_trans[e] * inv_temp;
  }
  __syncthreads();
  const bool nt = trans_is_narrow(s_trt, K * K, hi_t);
  const bool ns = trans_is_narrow(s_trs, K * K, hi_s);
  return nt && ns;
}

template <int K, int NT, int TT>
constexpr size_t distill_fwd_smem_bytes() {
  using Gm = Geom<K, TT>;
  return 4 * (4 * (size_t)Gm::KK4 + NT + 2 * (size_t)NSTAGE * NT * Gm::P);
}

template <int K, int NT, int TT, int MINB>
__global__ void __launch_bounds__(NT, MINB)
crf_distill_fwd_kernel(const float* __restrict__ t_logits, const float* __restrict__ t_trans,
                       const float* __restrict__ s_logits, const float* __restrict__ s_trans,
                       const int32_t* __restrict__ seq_len, float inv_temp, float* __restrict__ logz_out,
                       float* __restrict__ alpha_ws, int B, int L, int vec_logits, int force_exact) {
  using Gm = Geom<K, TT>;
  constexpr int T = Gm::T, G = Gm::G, P = Gm::P;
  constexpr int UNR = Gm::UNROLL ? K : 1;

  extern __shared__ __align__(16) float smem[];
  float* s_trt = smem;                      // teacher trans / tau [i][j]
  float* s_trs = s_trt + Gm::KK4;           // student trans / tau
  float* s_Et = s_trs + Gm::KK4;            // exp(trans_T / tau - tmax_T)
  float* s_Es = s_Et + Gm::KK4;             // exp(trans_S / tau - tmax_S)
  int* s_len = reinterpret_cast<int*>(s_Es + Gm::KK4);
  float* s_xt = reinterpret_cast<float*>(s_len + NT);
  float* s_xs = s_xt + NSTAGE * NT * P;

  const int tid = threadIdx.x;
  const int row0 = blockIdx.x * NT;
  const int nv = min(NT, B - row0);
  const int LK = L * K;

  int rawlen = 0, mylen = 1;
  if (tid < nv) {
    rawlen = seq_len[row0 + tid];
    mylen = min(max(rawlen, 1), L);
  }
  s_len[tid] = mylen;
  const int bmax = block_max_int<NT>(tid < nv ? mylen : 1, reinterpret_cast<int*>(s_xt));
  float tmax_t, tmax_s;
  const bool fast = load_trans_pair<K, NT>(t_trans, s_trans, inv_temp, s_trt, s_trs, tmax_t, tmax_s) && !force_exact;
  for (int e = tid; e < K * K; e += NT) {
    s_Et[e] = fast ? expf(s_trt[e] - tmax_t) : 0.f;
    s_Es[e] = fast ? expf(s_trs[e] - tmax_s) : 0.f;
  }
  __syncthreads();

  const float* gt = t_logits + (size_t)row0 * LK;
  const float* gs = s_logits + (size_t)row0 * LK;
  const int nchunk = (bmax + T - 1) / T;

#pragma unroll
  for (int s = 0; s < NSTAGE - 1; ++s) {
    if (s < nchunk) {
      stage_logits<K, NT, TT>(s_xt + s * NT * P, gt, LK, s * T, L, nv, s_len, vec_logits);
      stage_logits<K, NT, TT>(s_xs + s * NT * P, gs, LK, s * T, L, nv, s_len, vec_logits);
    }
    cp_async_commit();
  }

  // One step of either recursion on x (already scaled by 1/tau); the fast path renormalises every step.
  auto step = [&](Alpha<K>& s, const float* x, int t, float tmax, const float* s_tr, const float* s_E) {
    if (fast) {
      const float xm = row_max<K>(x);
      if (t == 0)
        fwd_fast_init<K>(s.a, s.lacc, x, xm);
      else
        fwd_fast_step<K, false>(s.a, s.lacc, x, xm, tmax, nullptr, s_E, true);
    } else if (t == 0) {
#pragma unroll UNR
      for (int j = 0; j < K; ++j) s.a[j] = x[j];
    } else {
      fwd_exact_step<K>(s.a, x, s_tr);
    }
  };

  Alpha<K> st, ss;  // teacher, student
#pragma unroll UNR
  for (int j = 0; j < K; ++j) st.a[j] = ss.a[j] = 0.f;
  st.lacc = ss.lacc = 0.f;
  float* aws_t = tid < nv ? alpha_ws + (size_t)(row0 + tid) * LK : nullptr;
  float* aws_s = aws_t != nullptr ? aws_t + (size_t)B * LK : nullptr;

  for (int c = 0; c < nchunk; ++c) {
    const int cn = c + NSTAGE - 1;
    if (cn < nchunk) {
      stage_logits<K, NT, TT>(s_xt + (cn % NSTAGE) * NT * P, gt, LK, cn * T, L, nv, s_len, vec_logits);
      stage_logits<K, NT, TT>(s_xs + (cn % NSTAGE) * NT * P, gs, LK, cn * T, L, nv, s_len, vec_logits);
    }
    cp_async_commit();
    cp_async_wait<NSTAGE - 1>();
    __syncthreads();

    const int t0 = c * T;
    if (tid < nv && t0 < mylen) {
      const float* rowt = s_xt + (c % NSTAGE) * NT * P + tid * P;
      const float* rows = s_xs + (c % NSTAGE) * NT * P + tid * P;
#pragma unroll
      for (int g = 0; g < T / G; ++g) {
        if (t0 + g * G < mylen) {
          float xts[G * K], xss[G * K];
          load_group<K>(xts, rowt, g);
          load_group<K>(xss, rows, g);
#pragma unroll
          for (int gg = 0; gg < G; ++gg) {
            const int t = t0 + g * G + gg;
            if (t < mylen) {
              float xt[K], xs[K];
#pragma unroll UNR
              for (int j = 0; j < K; ++j) {
                xt[j] = xts[gg * K + j] * inv_temp;
                xs[j] = xss[gg * K + j] * inv_temp;
              }
              step(st, xt, t, tmax_t, s_trt, s_Et);
              step(ss, xs, t, tmax_s, s_trs, s_Es);
              store_alpha<K>(aws_t + (size_t)t * K, st.a, st.lacc, fast);
              store_alpha<K>(aws_s + (size_t)t * K, ss.a, ss.lacc, fast);
            }
          }
        }
      }
    }
    __syncthreads();
  }

  if (tid < nv) {
    float lzt = fwd_logz<K>(st.a, st.lacc, fast), lzs = fwd_logz<K>(ss.a, ss.lacc, fast);
    if (rawlen <= 0) lzt = lzs = 0.f;  // empty sequence: KL = 0, nothing to differentiate
    logz_out[2 * (row0 + tid)] = lzt;
    logz_out[2 * (row0 + tid) + 1] = lzs;
  }
}

template <int K, int NT, int TT, int MINB = 1>
int launch_fwd_nt(const float* tl, const float* tt, const float* sl, const float* str, const int32_t* seq_len,
                  float inv_temp, float* logz, float* alpha_ws, int B, int L, int flags, cudaStream_t st) {
  const size_t smem = distill_fwd_smem_bytes<K, NT, TT>();
  auto kern = crf_distill_fwd_kernel<K, NT, TT, MINB>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  const int vl = ((L * K) % 4 == 0) && ((reinterpret_cast<uintptr_t>(tl) & 15) == 0) &&
                 ((reinterpret_cast<uintptr_t>(sl) & 15) == 0);
  kern<<<(B + NT - 1) / NT, NT, smem, st>>>(tl, tt, sl, str, seq_len, inv_temp, logz, alpha_ws, B, L, vl, flags & 1);
  return ner_launch_status();
}

// ---------------------------------------------------------------------------------------------------------- backward

template <int K, int NT>
constexpr size_t distill_bwd_smem_bytes() {
  using Gm = Geom<K>;
  return 4 * (6 * (size_t)Gm::KK4 + 64 + NT + 4 * (size_t)NSTAGE * NT * Gm::P);
}

// One reverse pass with beta_T and beta_S.  Fast path: with p[i] = exp(alpha_t[i] + rmax[i] + mq - logZ) and
// q[j] = exp(u_{t+1}[j] - mq), the pair marginal is xi[i][j] = p[i] E[i][j] q[j], each model with its own E and rmax.
// acc[i][j] sums xi_S - xi_T (registers for K <= 10, else shared-memory atomics); klp sums xi_T (T_T - T_S) / tau.
template <int K, int NT>
__global__ void __launch_bounds__(NT)
crf_distill_bwd_kernel(const float* __restrict__ t_logits, const float* __restrict__ t_trans,
                       const float* __restrict__ s_logits, const float* __restrict__ s_trans,
                       const int32_t* __restrict__ seq_len, float inv_temp, const float* __restrict__ alpha_ws,
                       const float* __restrict__ logz, const float* __restrict__ d_kl, float scale,
                       float* __restrict__ kl, float* __restrict__ d_s_logits, float* __restrict__ d_s_trans, int B,
                       int L, int vec_logits, int force_exact) {
  using Gm = Geom<K>;
  constexpr int T = Gm::T, G = Gm::G, P = Gm::P;
  constexpr int UNR = Gm::UNROLL ? K : 1;
  constexpr bool ACC_REGS = Gm::ACC_REGS;

  extern __shared__ __align__(16) float smem[];
  float* s_trt = smem;                                // teacher trans / tau [i][j]
  float* s_trs = s_trt + Gm::KK4;                     // student trans / tau
  float* s_Et = s_trs + Gm::KK4;                      // exp(trans_T / tau - rmax_T[i])
  float* s_Es = s_Et + Gm::KK4;                       // exp(trans_S / tau - rmax_S[i])
  float* s_dtr = s_Es + Gm::KK4;                      // (trans_T - trans_S) / tau
  float* s_dT = s_dtr + Gm::KK4;                      // CTA-level d_s_trans accumulator
  float* s_rmt = s_dT + Gm::KK4;                      // [32]
  float* s_rms = s_rmt + 32;                          // [32]
  int* s_len = reinterpret_cast<int*>(s_rms + 32);    // [NT]
  float* s_xt = reinterpret_cast<float*>(s_len + NT); // [NSTAGE][NT][P] teacher logits
  float* s_xs = s_xt + NSTAGE * NT * P;               // student logits, overwritten by d_s_logits
  float* s_at = s_xs + NSTAGE * NT * P;               // alpha_T
  float* s_as = s_at + NSTAGE * NT * P;               // alpha_S

  const int tid = threadIdx.x;
  const int row0 = blockIdx.x * NT;
  const int nv = min(NT, B - row0);
  const int LK = L * K;

  float lzt = 0.f, lzs = 0.f, gcoef = 0.f;
  int mylen = 0;
  if (tid < nv) {
    mylen = min(max(seq_len[row0 + tid], 0), L);
    lzt = logz[2 * (row0 + tid)];
    lzs = logz[2 * (row0 + tid) + 1];
    gcoef = (d_kl != nullptr ? d_kl[row0 + tid] : 1.f) * scale * inv_temp;
  }
  for (int e = tid; e < K * K; e += NT) s_dT[e] = 0.f;
  s_len[tid] = mylen;
  const int bmax = block_max_int<NT>(mylen, reinterpret_cast<int*>(s_xt));
  float hi_t, hi_s;
  const bool fast = load_trans_pair<K, NT>(t_trans, s_trans, inv_temp, s_trt, s_trs, hi_t, hi_s) && !force_exact;
  if (tid < K) {
    float rt = -INFINITY, rs = -INFINITY;
    for (int j = 0; j < K; ++j) {
      rt = fmaxf(rt, s_trt[tid * K + j]);
      rs = fmaxf(rs, s_trs[tid * K + j]);
    }
    s_rmt[tid] = rt;
    s_rms[tid] = rs;
  }
  __syncthreads();
  for (int e = tid; e < K * K; e += NT) {
    s_Et[e] = fast ? expf(s_trt[e] - s_rmt[e / K]) : 0.f;
    s_Es[e] = fast ? expf(s_trs[e] - s_rms[e / K]) : 0.f;
    s_dtr[e] = s_trt[e] - s_trs[e];
  }
  __syncthreads();

  const float* gxt = t_logits + (size_t)row0 * LK;
  const float* gxs = s_logits + (size_t)row0 * LK;
  const float* gat = alpha_ws + (size_t)row0 * LK;
  const float* gas = gat + (size_t)B * LK;
  float* gd = d_s_logits + (size_t)row0 * LK;
  const int nchunk = (bmax + T - 1) / T;
  zero_dlogits_tail<K, NT>(gd, nv, L, nchunk);

  auto stage = [&](int c, int buf) {
    stage_logits<K, NT>(s_xt + buf * NT * P, gxt, LK, c * T, L, nv, s_len, vec_logits);
    stage_logits<K, NT>(s_xs + buf * NT * P, gxs, LK, c * T, L, nv, s_len, vec_logits);
    stage_logits<K, NT>(s_at + buf * NT * P, gat, LK, c * T, L, nv, s_len, vec_logits);
    stage_logits<K, NT>(s_as + buf * NT * P, gas, LK, c * T, L, nv, s_len, vec_logits);
  };
#pragma unroll
  for (int s = 0; s < NSTAGE - 1; ++s) {
    if (s < nchunk) stage(nchunk - 1 - s, s % NSTAGE);
    cp_async_commit();
  }

  float bt[K], bs[K], qt[K], qs[K], acc[ACC_REGS ? K * K : 1];
  float mqt = 0.f, mqs = 0.f, klu = 0.f, klp = 0.f;
#pragma unroll UNR
  for (int j = 0; j < K; ++j) bt[j] = bs[j] = qt[j] = qs[j] = 0.f;
  if constexpr (ACC_REGS) {
#pragma unroll
    for (int e = 0; e < K * K; ++e) acc[e] = 0.f;
  }

  for (int it = 0; it < nchunk; ++it) {
    const int c = nchunk - 1 - it;
    const int itn = it + NSTAGE - 1;
    if (itn < nchunk) stage(nchunk - 1 - itn, itn % NSTAGE);
    cp_async_commit();
    cp_async_wait<NSTAGE - 1>();
    __syncthreads();

    const int buf = it % NSTAGE;
    const int t0 = c * T;
    if (tid < nv && t0 < mylen) {
      const float* rowxt = s_xt + buf * NT * P + tid * P;
      float* rowxs = s_xs + buf * NT * P + tid * P;
      const float* rowat = s_at + buf * NT * P + tid * P;
      const float* rowas = s_as + buf * NT * P + tid * P;
#pragma unroll
      for (int g = T / G - 1; g >= 0; --g) {
        if (t0 + g * G < mylen) {
          float xts[G * K], xss[G * K], ats[G * K], ass[G * K], dl[G * K];
          load_group<K>(xts, rowxt, g);
          load_group<K>(xss, rowxs, g);
          load_group<K>(ats, rowat, g);
          load_group<K>(ass, rowas, g);
#pragma unroll
          for (int gg = G - 1; gg >= 0; --gg) {
            const int t = t0 + g * G + gg;
            if (t < mylen) {
              const float* at = ats + gg * K;
              const float* as = ass + gg * K;
              // ---- pair marginals of (t, t+1) from step t+1's q / mq
              if (t < mylen - 1) {
                if (fast) {
                  float pt[K], ps[K];
#pragma unroll UNR
                  for (int i = 0; i < K; ++i) {
                    pt[i] = __expf(at[i] + s_rmt[i] + mqt - lzt);
                    ps[i] = __expf(as[i] + s_rms[i] + mqs - lzs);
                  }
#pragma unroll UNR
                  for (int i = 0; i < K; ++i)
#pragma unroll UNR
                    for (int j = 0; j < K; ++j) {
                      const float xit = __fmul_rn(__fmul_rn(pt[i], s_Et[i * K + j]), qt[j]);
                      const float d = __fmul_rn(__fmul_rn(ps[i], s_Es[i * K + j]), qs[j]) - xit;
                      klp = fmaf(xit, s_dtr[i * K + j], klp);
                      if constexpr (ACC_REGS) {
                        acc[i * K + j] += d;
                      } else {
                        if (d != 0.f) atomicAdd(&s_dT[i * K + j], gcoef * d);
                      }
                    }
                } else {
                  for (int i = 0; i < K; ++i)
                    for (int j = 0; j < K; ++j) {
                      const float xit = expf(at[i] + s_trt[i * K + j] + qt[j] - lzt);
                      const float d = expf(as[i] + s_trs[i * K + j] + qs[j] - lzs) - xit;
                      if (xit != 0.f) klp = fmaf(xit, s_dtr[i * K + j], klp);
                      if (d != 0.f) atomicAdd(&s_dT[i * K + j], gcoef * d);
                    }
                }
              }
              // ---- unary marginals: d_s_logits = g (mu_S - mu_T) / tau, an exact +0 where they agree
              const float* xt = xts + gg * K;
              const float* xs = xss + gg * K;
#pragma unroll UNR
              for (int j = 0; j < K; ++j) {
                const float mt = __expf(at[j] + bt[j] - lzt);
                const float d = __expf(as[j] + bs[j] - lzs) - mt;
                dl[gg * K + j] = fmaf(gcoef, d, 0.f);
                if (mt != 0.f) klu = fmaf(mt, __fmul_rn(xt[j], inv_temp) - __fmul_rn(xs[j], inv_temp), klu);
              }
              // ---- beta recursions to t-1
              if (t > 0) {
                float ut[K], us[K];
#pragma unroll UNR
                for (int j = 0; j < K; ++j) {
                  ut[j] = xt[j] * inv_temp + bt[j];
                  us[j] = xs[j] * inv_temp + bs[j];
                }
                beta_step<K>(fast, bt, qt, mqt, qt, ut, s_trt, s_Et, s_rmt);
                beta_step<K>(fast, bs, qs, mqs, qs, us, s_trs, s_Es, s_rms);
              }
            } else {
#pragma unroll UNR
              for (int j = 0; j < K; ++j) dl[gg * K + j] = 0.f;
            }
          }
          float4* o4 = reinterpret_cast<float4*>(rowxs + g * G * K);
#pragma unroll
          for (int qq = 0; qq < Gm::GQ; ++qq)
            o4[qq] = make_float4(dl[4 * qq], dl[4 * qq + 1], dl[4 * qq + 2], dl[4 * qq + 3]);
        }
      }
    }
    __syncthreads();
    store_dlogits_chunk<K, NT>(gd, s_xs + buf * NT * P, s_len, nv, L, t0, vec_logits);
    __syncthreads();
  }

  if (tid < nv) kl[row0 + tid] = (klu + klp) + (lzs - lzt);
  // d_s_trans += gcoef * acc (E is already inside acc), plus what the CTA gathered in s_dT
  if constexpr (ACC_REGS) {
#pragma unroll
    for (int e = 0; e < K * K; ++e) {
      float v = tid < nv ? gcoef * acc[e] : 0.f;
      v = warp_sum(v);
      if ((tid & 31) == 0 && v != 0.f) atomicAdd(&s_dT[e], v);
    }
  }
  __syncthreads();
  for (int e = tid; e < K * K; e += NT) {
    const float v = s_dT[e];
    if (v != 0.f) atomicAdd(&d_s_trans[e], v);
  }
}

template <int K, int NT>
int launch_bwd_nt(const float* tl, const float* tt, const float* sl, const float* str, const int32_t* seq_len,
                  float inv_temp, const float* alpha_ws, const float* logz, const float* d_kl, float scale, float* kl,
                  float* d_s_logits, float* d_s_trans, int B, int L, int flags, cudaStream_t st) {
  const size_t smem = distill_bwd_smem_bytes<K, NT>();
  auto kern = crf_distill_bwd_kernel<K, NT>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  const int vl = ((L * K) % 4 == 0) && ((reinterpret_cast<uintptr_t>(tl) & 15) == 0) &&
                 ((reinterpret_cast<uintptr_t>(sl) & 15) == 0) &&
                 ((reinterpret_cast<uintptr_t>(alpha_ws) & 15) == 0) &&
                 ((reinterpret_cast<uintptr_t>(d_s_logits) & 15) == 0);
  kern<<<(B + NT - 1) / NT, NT, smem, st>>>(tl, tt, sl, str, seq_len, inv_temp, alpha_ws, logz, d_kl, scale, kl,
                                            d_s_logits, d_s_trans, B, L, vl, flags & 1);
  return ner_launch_status();
}

// ------------------------------------------------------------------------------------- small batches: lane per tag
// A group of GS lanes holds one sequence, lane j owns tag j of both recursions, predecessors are exchanged with
// __shfl_sync, every logsumexp is exact with its own max.  The teacher and the student run the same instructions.

template <int K>
__global__ void __launch_bounds__(32)
crf_distill_fwd_lanes_kernel(const float* __restrict__ t_logits, const float* __restrict__ t_trans,
                             const float* __restrict__ s_logits, const float* __restrict__ s_trans,
                             const int32_t* __restrict__ seq_len, float inv_temp, float* __restrict__ logz_out,
                             float* __restrict__ alpha_ws, int B, int L) {
  constexpr int GS = Lanes<K>::GS, SPW = Lanes<K>::SPW, PF = 4;
  __shared__ float s_trt[K * K], s_trs[K * K];
  const int lane = threadIdx.x;
  const int g = lane / GS, j = lane % GS;
  const int b = blockIdx.x * SPW + g;
  const bool seq_ok = b < B;
  const bool tag_ok = j < K;
  for (int e = lane; e < K * K; e += 32) {
    s_trt[e] = t_trans[e] * inv_temp;
    s_trs[e] = s_trans[e] * inv_temp;
  }
  int rawlen = 0, len = 1;
  if (seq_ok) {
    rawlen = seq_len[b];
    len = min(max(rawlen, 1), L);
  }
  const int wmax = lanes_wmax(len);
  __syncwarp();
  float tct[K], tcs[K];
#pragma unroll
  for (int i = 0; i < K; ++i) {
    tct[i] = tag_ok ? s_trt[i * K + j] : 0.f;
    tcs[i] = tag_ok ? s_trs[i * K + j] : 0.f;
  }

  const size_t off = (size_t)(seq_ok ? b : 0) * L * K + (tag_ok ? j : 0);
  const float* xpt = t_logits + off;
  const float* xps = s_logits + off;
  float* wt = (seq_ok && tag_ok) ? alpha_ws + off : nullptr;
  float* ws = wt != nullptr ? wt + (size_t)B * L * K : nullptr;
  auto ld = [&](const float* p, int t) -> float {
    return (seq_ok && tag_ok && t < len) ? p[(size_t)t * K] * inv_temp : -INFINITY;
  };

  float at = ld(xpt, 0), as = ld(xps, 0);
  if (wt != nullptr) {
    wt[0] = at;
    ws[0] = as;
  }
  float xqt[PF], xqs[PF];
#pragma unroll
  for (int u = 0; u < PF; ++u) {
    xqt[u] = ld(xpt, 1 + u);
    xqs[u] = ld(xps, 1 + u);
  }
  for (int t0 = 1; t0 < wmax; t0 += PF) {
#pragma unroll
    for (int u = 0; u < PF; ++u) {
      const int t = t0 + u;
      const float xt = xqt[u], xs = xqs[u];
      xqt[u] = ld(xpt, t + PF);
      xqs[u] = ld(xps, t + PF);
      if (t < wmax) {
        const float nt = lanes_alpha_step<K>(at, xt, tct, g);
        const float ns = lanes_alpha_step<K>(as, xs, tcs, g);
        if (t < len) {
          at = tag_ok ? nt : -INFINITY;
          as = tag_ok ? ns : -INFINITY;
          if (wt != nullptr) {
            wt[(size_t)t * K] = at;
            ws[(size_t)t * K] = as;
          }
        }
      }
    }
  }
  float lzt = lanes_logsumexp<K>(at, tag_ok), lzs = lanes_logsumexp<K>(as, tag_ok);
  if (j == 0 && seq_ok) {
    if (rawlen <= 0) lzt = lzs = 0.f;
    logz_out[2 * b] = lzt;
    logz_out[2 * b + 1] = lzs;
  }
}

// Lane i = tag i walks t = len-1 .. 0 with beta_T[i] and beta_S[i]:
//   w_j = x_t[j] / tau + beta_t[j],  v_ij = trans[i][j] / tau + w_j,  beta_{t-1}[i] = logsumexp_j v_ij,
//   xi(t-1, t)[i][j] = exp(alpha_{t-1}[i] - logZ + v_ij),  mu_t[i] = exp(alpha_t[i] + beta_t[i] - logZ).
// Each lane sums its tag's share of KL; the group adds the shares.
template <int K>
__global__ void __launch_bounds__(32)
crf_distill_bwd_lanes_kernel(const float* __restrict__ t_logits, const float* __restrict__ t_trans,
                             const float* __restrict__ s_logits, const float* __restrict__ s_trans,
                             const int32_t* __restrict__ seq_len, float inv_temp, const float* __restrict__ alpha_ws,
                             const float* __restrict__ logz, const float* __restrict__ d_kl, float scale,
                             float* __restrict__ kl, float* __restrict__ d_s_logits, float* __restrict__ d_s_trans,
                             int B, int L) {
  constexpr int GS = Lanes<K>::GS, SPW = Lanes<K>::SPW, PF = 4;
  const int lane = threadIdx.x;
  const int g = lane / GS, i = lane % GS;
  const int b = blockIdx.x * SPW + g;
  const bool seq_ok = b < B;
  const bool tag_ok = i < K;
  int len = 0;
  float lzt = 0.f, lzs = 0.f, gco = 0.f;
  if (seq_ok) {
    len = min(max(seq_len[b], 0), L);
    lzt = logz[2 * b];
    lzs = logz[2 * b + 1];
    gco = (d_kl != nullptr ? d_kl[b] : 1.f) * scale * inv_temp;
  }
  const int wmax = lanes_wmax(len);

  float trt[K], trs[K], acc[K];
#pragma unroll
  for (int jj = 0; jj < K; ++jj) {
    trt[jj] = tag_ok ? t_trans[i * K + jj] * inv_temp : 0.f;
    trs[jj] = tag_ok ? s_trans[i * K + jj] * inv_temp : 0.f;
    acc[jj] = 0.f;
  }
  const bool io = seq_ok && tag_ok;
  const size_t off = (size_t)(seq_ok ? b : 0) * L * K + (tag_ok ? i : 0);
  const float* xpt = t_logits + off;
  const float* xps = s_logits + off;
  const float* pat = alpha_ws + off;
  const float* pas = pat + (size_t)B * L * K;
  float* dp = d_s_logits + off;
  if (io)
    for (int t = len; t < L; ++t) dp[(size_t)t * K] = 0.f;
  auto ldx = [&](const float* p, int t) -> float { return (io && t >= 0 && t < len) ? p[(size_t)t * K] * inv_temp : 0.f; };
  auto lda = [&](const float* p, int t) -> float { return (io && t >= 0 && t < len) ? p[(size_t)t * K] : 0.f; };

  float bt = 0.f, bs = 0.f, klu = 0.f, klp = 0.f;
  float xqt[PF], xqs[PF], aqt[PF], aqs[PF];
#pragma unroll
  for (int u = 0; u < PF; ++u) {
    xqt[u] = ldx(xpt, len - 1 - u);
    xqs[u] = ldx(xps, len - 1 - u);
    aqt[u] = lda(pat, len - 2 - u);
    aqs[u] = lda(pas, len - 2 - u);
  }
  float at_t = lda(pat, len - 1), as_t = lda(pas, len - 1);
  for (int s0 = 0; s0 < wmax; s0 += PF) {
#pragma unroll
    for (int u = 0; u < PF; ++u) {
      const int sidx = s0 + u;
      const int t = len - 1 - sidx;
      const float xt = xqt[u], xs = xqs[u], at_prev = aqt[u], as_prev = aqs[u];
      xqt[u] = ldx(xpt, t - PF);
      xqs[u] = ldx(xps, t - PF);
      aqt[u] = lda(pat, t - 1 - PF);
      aqs[u] = lda(pas, t - 1 - PF);
      if (sidx < wmax) {                    // warp-uniform: every lane takes part in the shuffles
        const bool live = t >= 0;
        if (io && live) {
          const float mt = __expf(at_t + bt - lzt);
          dp[(size_t)t * K] = fmaf(gco, __expf(as_t + bs - lzs) - mt, 0.f);
          if (mt != 0.f) klu = fmaf(mt, xt - xs, klu);
        }
        const float wt_ = (tag_ok && live) ? xt + bt : -INFINITY;
        const float ws_ = (tag_ok && live) ? xs + bs : -INFINITY;
        float vt[K], vs[K];
        const float mt = lanes_gather<K>(vt, wt_, trt, g);
        const float ms = lanes_gather<K>(vs, ws_, trs, g);
        if (live && t >= 1) {
          const float mmt = (fabsf(mt) <= 3.0e38f) ? mt : 0.f;
          const float mms = (fabsf(ms) <= 3.0e38f) ? ms : 0.f;
          const float amt = at_prev - lzt, ams = as_prev - lzs;
          float sumt = 0.f, sums = 0.f;
#pragma unroll
          for (int jj = 0; jj < K; ++jj) {
            sumt += __expf(vt[jj] - mmt);
            sums += __expf(vs[jj] - mms);
            const float xit = __expf(amt + vt[jj]);
            acc[jj] += __expf(ams + vs[jj]) - xit;
            if (io && xit != 0.f) klp = fmaf(xit, trt[jj] - trs[jj], klp);
          }
          bt = __logf(sumt) + mmt;
          bs = __logf(sums) + mms;
          at_t = at_prev;
          as_t = as_prev;
        }
      }
    }
  }
  float share = klu + klp;
#pragma unroll
  for (int o = GS / 2; o > 0; o >>= 1) share += __shfl_xor_sync(0xffffffffu, share, o, GS);
  if (i == 0 && seq_ok) kl[b] = share + (lzs - lzt);
  if (io && len > 0) {
#pragma unroll
    for (int jj = 0; jj < K; ++jj)
      if (acc[jj] != 0.f) atomicAdd(d_s_trans + i * K + jj, gco * acc[jj]);
  }
}

template <int K>
int launch_fwd(const float* tl, const float* tt, const float* sl, const float* str, const int32_t* seq_len,
               float inv_temp, float* logz, float* alpha_ws, int B, int L, int flags, cudaStream_t st) {
  if (B <= NER_CRF_SMALL_B) {
    constexpr int SPW = Lanes<K>::SPW;
    crf_distill_fwd_lanes_kernel<K><<<(B + SPW - 1) / SPW, 32, 0, st>>>(tl, tt, sl, str, seq_len, inv_temp, logz,
                                                                        alpha_ws, B, L);
    return ner_launch_status();
  }
  if (use_cta64(B))
    return launch_fwd_nt<K, 64, 4, 4>(tl, tt, sl, str, seq_len, inv_temp, logz, alpha_ws, B, L, flags, st);
  return launch_fwd_nt<K, 32, T_CHUNK>(tl, tt, sl, str, seq_len, inv_temp, logz, alpha_ws, B, L, flags, st);
}

template <int K>
int launch_bwd(const float* tl, const float* tt, const float* sl, const float* str, const int32_t* seq_len,
               float inv_temp, const float* alpha_ws, const float* logz, const float* d_kl, float scale, float* kl,
               float* d_s_logits, float* d_s_trans, int B, int L, int flags, cudaStream_t st) {
  if (B > NER_CRF_SMALL_B) {
    if constexpr (distill_bwd_smem_bytes<K, 64>() <= kMaxSmem) {
      if (use_cta64(B))
        return launch_bwd_nt<K, 64>(tl, tt, sl, str, seq_len, inv_temp, alpha_ws, logz, d_kl, scale, kl, d_s_logits,
                                    d_s_trans, B, L, flags, st);
    }
    if constexpr (distill_bwd_smem_bytes<K, 32>() <= kMaxSmem)
      return launch_bwd_nt<K, 32>(tl, tt, sl, str, seq_len, inv_temp, alpha_ws, logz, d_kl, scale, kl, d_s_logits,
                                  d_s_trans, B, L, flags, st);
  }
  constexpr int SPW = Lanes<K>::SPW;
  crf_distill_bwd_lanes_kernel<K><<<(B + SPW - 1) / SPW, 32, 0, st>>>(tl, tt, sl, str, seq_len, inv_temp, alpha_ws,
                                                                      logz, d_kl, scale, kl, d_s_logits, d_s_trans, B,
                                                                      L);
  return ner_launch_status();
}

// 1/tau must be a positive finite number; L at most document mode's 4095.
int check_common(int B, int L, int K, float inv_temp) {
  if (B < 0 || L < 1 || K < 1 || !(inv_temp > 0.f) || !(inv_temp <= FLT_MAX)) return NER_ERR_INVALID_ARG;
  if (K > NER_MAX_TAGS || L > kMaxLen) return NER_ERR_UNSUPPORTED;
  return NER_OK;
}

}  // namespace

extern "C" int ner_crf_distill_fwd(const float* t_logits, const float* t_trans, const float* s_logits,
                                   const float* s_trans, const int32_t* seq_len, float inv_temp, float* logz,
                                   float* alpha_ws, int B, int L, int K, int flags, ner_stream_t stream) {
  const int rc = check_common(B, L, K, inv_temp);
  if (rc != NER_OK || B == 0) return rc;
  if (!t_logits || !t_trans || !s_logits || !s_trans || !seq_len || !logz || !alpha_ws) return NER_ERR_INVALID_ARG;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define CALL(KK) \
  return launch_fwd<KK>(t_logits, t_trans, s_logits, s_trans, seq_len, inv_temp, logz, alpha_ws, B, L, flags, st)
  NER_CRF_DISPATCH_K(K, CALL)
#undef CALL
  return NER_ERR_UNSUPPORTED;
}

extern "C" int ner_crf_distill_bwd(const float* t_logits, const float* t_trans, const float* s_logits,
                                   const float* s_trans, const int32_t* seq_len, float inv_temp,
                                   const float* alpha_ws, const float* logz, const float* d_kl, float scale, float* kl,
                                   float* d_s_logits, float* d_s_trans, int B, int L, int K, int flags,
                                   ner_stream_t stream) {
  const int rc = check_common(B, L, K, inv_temp);
  if (rc != NER_OK || B == 0) return rc;
  if (!t_logits || !t_trans || !s_logits || !s_trans || !seq_len || !alpha_ws || !logz || !kl || !d_s_logits ||
      !d_s_trans)
    return NER_ERR_INVALID_ARG;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define CALL(KK)                                                                                                  \
  return launch_bwd<KK>(t_logits, t_trans, s_logits, s_trans, seq_len, inv_temp, alpha_ws, logz, d_kl, scale, kl, \
                        d_s_logits, d_s_trans, B, L, flags, st)
  NER_CRF_DISPATCH_K(K, CALL)
#undef CALL
  return NER_ERR_UNSUPPORTED;
}
