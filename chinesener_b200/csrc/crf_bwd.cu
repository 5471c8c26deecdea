// Gradient of the CRF log-likelihood w.r.t. emission logits and the transition matrix,
// sm_90a.  The reference obtains it by tf.gradients through the crf_log_norm while-loop
// (reference tools/train_utils.py:314 over tools/layer.py:122-127); here it is the closed
// form forward-backward:
//     d ll / d x[t][j]      = 1[y_t = j]              - P(y_t = j | x)
//     d ll / d trans[i][j]  = sum_t 1[y_{t-1}=i,y_t=j] - sum_t P(y_{t-1}=i, y_t=j | x)
// One thread per sequence walks t = len-1 .. 0 with beta[K] in registers; alpha_t comes
// from the forward kernel's workspace.  Logits / alpha / tags are streamed (in reverse) by
// cp.async like the forward kernels; d_logits is written back through the same smem tile so
// the HBM store is coalesced.  Pair marginals are accumulated per thread as
// acc[i][j] += pa[i]*q[j] (rank-1 update) and scaled by exp(trans - rowmax) once at the end.
#include "crf_common.cuh"

namespace {

using namespace crf;

template <int K, int NT>
__global__ void __launch_bounds__(NT)
crf_loglik_bwd_kernel(const float* __restrict__ logits, const int32_t* __restrict__ tags,
                      const int32_t* __restrict__ seq_len, const float* __restrict__ trans,
                      const float* __restrict__ alpha_ws, const float* __restrict__ logz,
                      const float* __restrict__ d_ll, float scale, float* __restrict__ d_logits,
                      float* __restrict__ d_trans, int B, int L, int vec_logits, int vec_tags) {
  using Gm = Geom<K>;
  constexpr int T = Gm::T, G = Gm::G, P = Gm::P;
  constexpr int UNR = Gm::UNROLL ? K : 1;
  constexpr bool ACC_REGS = Gm::ACC_REGS;  // K*K rank-1 accumulators in registers

  extern __shared__ __align__(16) float smem[];
  float* s_tr = smem;                                // raw trans [i][j]
  float* s_E = s_tr + Gm::KK4;                       // exp(trans[i][j] - rmax[i])
  float* s_dT = s_E + Gm::KK4;                       // CTA-level d_trans accumulator
  float* s_rmax = s_dT + Gm::KK4;                    // [32]
  int* s_len = reinterpret_cast<int*>(s_rmax + 32);  // [NT]
  float* s_x = reinterpret_cast<float*>(s_len + NT); // [NSTAGE][NT][P] logits, overwritten by d_logits
  float* s_a = s_x + NSTAGE * NT * P;                // [NSTAGE][NT][P] alpha
  int* s_tags = reinterpret_cast<int*>(s_a + NSTAGE * NT * P);

  const int tid = threadIdx.x;
  const int row0 = blockIdx.x * NT;
  const int nv = min(NT, B - row0);
  const int LK = L * K;

  const int mylen = tid < nv ? min(max(seq_len[row0 + tid], 0), L) : 0;
  int bmax;
  const bool fast = bwd_prologue<K, NT>(trans, mylen, s_tr, s_E, s_dT, s_rmax, s_len, reinterpret_cast<int*>(s_x), bmax);

  const float* gx = logits + (size_t)row0 * LK;
  const float* ga = alpha_ws + (size_t)row0 * LK;
  const int32_t* gt = tags + (size_t)row0 * L;
  float* gd = d_logits + (size_t)row0 * LK;
  const int nchunk = (bmax + T - 1) / T;
  zero_dlogits_tail<K, NT>(gd, nv, L, nchunk);

  auto stage = [&](int c, int buf) {
    stage_logits<K, NT>(s_x + buf * NT * P, gx, LK, c * T, L, nv, s_len, vec_logits);
    stage_logits<K, NT>(s_a + buf * NT * P, ga, LK, c * T, L, nv, s_len, vec_logits);
    stage_labels<NT>(s_tags + buf * NT * LABP, gt, L, c * T, nv, s_len, vec_tags);
  };

  // reverse streaming: iteration it handles chunk c = nchunk-1-it
#pragma unroll
  for (int s = 0; s < NSTAGE - 1; ++s) {
    if (s < nchunk) stage(nchunk - 1 - s, s % NSTAGE);
    cp_async_commit();
  }

  float beta[K], q[K], acc[ACC_REGS ? K * K : 1], rmx[K];
#pragma unroll UNR
  for (int j = 0; j < K; ++j) {
    beta[j] = 0.f;
    q[j] = 0.f;
    rmx[j] = s_rmax[j];
  }
  if constexpr (ACC_REGS) {
#pragma unroll
    for (int e = 0; e < K * K; ++e) acc[e] = 0.f;
  }
  float mq = 0.f;
  float u_keep[K];  // exact path: u[j] = x_{t+1}[j] + beta_{t+1}[j]
#pragma unroll UNR
  for (int j = 0; j < K; ++j) u_keep[j] = 0.f;
  int next_tag = 0;
  float lz = 0.f, gcoef = 0.f;
  if (tid < nv) {
    lz = logz[row0 + tid];
    gcoef = (d_ll != nullptr ? d_ll[row0 + tid] : 1.f) * scale;
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
      float* rowx = s_x + buf * NT * P + tid * P;
      const float* rowa = s_a + buf * NT * P + tid * P;
      int tg[T];
      {
        const int4* tp = reinterpret_cast<const int4*>(s_tags + buf * NT * LABP + tid * LABP);
#pragma unroll
        for (int qq = 0; qq < T / 4; ++qq) {
          const int4 v = tp[qq];
          tg[4 * qq + 0] = v.x;
          tg[4 * qq + 1] = v.y;
          tg[4 * qq + 2] = v.z;
          tg[4 * qq + 3] = v.w;
        }
      }
#pragma unroll
      for (int g = T / G - 1; g >= 0; --g) {
        if (t0 + g * G < mylen) {
          float xs[G * K], as[G * K], dl[G * K];
          load_group<K>(xs, rowx, g);
          load_group<K>(as, rowa, g);
#pragma unroll
          for (int gg = G - 1; gg >= 0; --gg) {
            const int tt = g * G + gg;
            const int t = t0 + tt;
            if (t < mylen) {
              const int tag = min(max(tg[tt], 0), K - 1);
              // ---- pair marginals for (t, t+1), using q/mq (fast) or u_keep (exact) of step t+1
              if (t < mylen - 1) {
                if (fast) {
                  float pa[K];
#pragma unroll UNR
                  for (int i = 0; i < K; ++i) pa[i] = __expf(as[gg * K + i] + rmx[i] + mq - lz);
                  if constexpr (ACC_REGS) {
#pragma unroll
                    for (int i = 0; i < K; ++i)
#pragma unroll
                      for (int j = 0; j < K; ++j) acc[i * K + j] = fmaf(pa[i], q[j], acc[i * K + j]);
                  } else {
                    for (int i = 0; i < K; ++i)
                      for (int j = 0; j < K; ++j)
                        atomicAdd(&s_dT[i * K + j], -gcoef * pa[i] * q[j] * s_E[i * K + j]);
                  }
                } else {
                  for (int i = 0; i < K; ++i)
                    for (int j = 0; j < K; ++j) {
                      const float pr = expf(as[gg * K + i] + s_tr[i * K + j] + u_keep[j] - lz);
                      atomicAdd(&s_dT[i * K + j], -gcoef * pr);
                    }
                }
                atomicAdd(&s_dT[tag * K + next_tag], gcoef);
              }
              next_tag = tag;
              // ---- unary marginal + d_logits
#pragma unroll UNR
              for (int j = 0; j < K; ++j) {
                const float p = __expf(as[gg * K + j] + beta[j] - lz);
                dl[gg * K + j] = gcoef * ((j == tag ? 1.f : 0.f) - p);
              }
              // ---- beta recursion to t-1
              if (t > 0) {
                float u[K];
#pragma unroll UNR
                for (int j = 0; j < K; ++j) u[j] = xs[gg * K + j] + beta[j];
                beta_step<K>(fast, beta, q, mq, u_keep, u, s_tr, s_E, rmx);
              }
            } else {
#pragma unroll UNR
              for (int j = 0; j < K; ++j) dl[gg * K + j] = 0.f;
            }
          }
          // write the G steps of d_logits back over the staged logits (STS.128)
          float4* o4 = reinterpret_cast<float4*>(rowx + g * G * K);
#pragma unroll
          for (int qq = 0; qq < Gm::GQ; ++qq)
            o4[qq] = make_float4(dl[4 * qq], dl[4 * qq + 1], dl[4 * qq + 2], dl[4 * qq + 3]);
        }
      }
    }
    __syncthreads();
    store_dlogits_chunk<K, NT>(gd, s_x + buf * NT * P, s_len, nv, L, t0, vec_logits);
    __syncthreads();
  }

  flush_dtrans<K, NT>(acc, -gcoef, tid < nv, s_dT, s_E, d_trans);
}

template <int K, int NT>
int launch_bwd_nt(const float* logits, const int32_t* tags, const int32_t* seq_len, const float* trans,
                  const float* alpha_ws, const float* logz, const float* d_ll, float scale, float* d_logits,
                  float* d_trans, int B, int L, cudaStream_t st) {
  const size_t smem = bwd_smem_bytes<K, NT, 2>();
  auto kern = crf_loglik_bwd_kernel<K, NT>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  const int vl = ((L * K) % 4 == 0) && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0) &&
                 ((reinterpret_cast<uintptr_t>(alpha_ws) & 15) == 0) && ((reinterpret_cast<uintptr_t>(d_logits) & 15) == 0);
  const int vt = (L % 4 == 0) && ((reinterpret_cast<uintptr_t>(tags) & 15) == 0);
  const int grid = (B + NT - 1) / NT;
  kern<<<grid, NT, smem, st>>>(logits, tags, seq_len, trans, alpha_ws, logz, d_ll, scale, d_logits, d_trans, B, L, vl, vt);
  return ner_launch_status();
}

template <int K>
int launch_bwd(const float* logits, const int32_t* tags, const int32_t* seq_len, const float* trans,
               const float* alpha_ws, const float* logz, const float* d_ll, float scale, float* d_logits,
               float* d_trans, int B, int L, cudaStream_t st) {
  // 64-thread CTAs need twice the staging ring of 32-thread ones: past K = 26 that is more shared memory than a CTA
  // can have, so those K stay on 32-thread CTAs at every B
  if constexpr (bwd_smem_bytes<K, 64, 2>() <= kMaxSmem) {
    if (use_cta64(B))
      return launch_bwd_nt<K, 64>(logits, tags, seq_len, trans, alpha_ws, logz, d_ll, scale, d_logits, d_trans, B, L,
                                  st);
  }
  return launch_bwd_nt<K, 32>(logits, tags, seq_len, trans, alpha_ws, logz, d_ll, scale, d_logits, d_trans, B, L, st);
}

}  // namespace

extern "C" int ner_crf_loglik_bwd(const float* logits, const int32_t* tags, const int32_t* seq_len,
                                  const float* trans, const float* alpha_ws, const float* logz,
                                  const float* d_ll, float scale, float* d_logits, float* d_trans, int B, int L,
                                  int K, ner_stream_t stream) {
  if (B < 0 || L < 1 || K < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!logits || !tags || !seq_len || !trans || !alpha_ws || !logz || !d_logits || !d_trans) return NER_ERR_INVALID_ARG;
  if (K > NER_MAX_TAGS) return NER_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (B <= NER_CRF_SMALL_B)  // few sequences: the lane-per-tag kernel (crf_small.cu) walks a much shorter chain
    return ner_crf_loglik_bwd_small(logits, tags, seq_len, trans, alpha_ws, logz, d_ll, scale, d_logits, d_trans, B, L, K,
                                    st);
#define CALL(KK) \
  return launch_bwd<KK>(logits, tags, seq_len, trans, alpha_ws, logz, d_ll, scale, d_logits, d_trans, B, L, st)
  NER_CRF_DISPATCH_K(K, CALL)
#undef CALL
  return NER_ERR_UNSUPPORTED;
}
