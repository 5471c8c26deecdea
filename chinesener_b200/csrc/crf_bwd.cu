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

constexpr int TAGP = 12;

template <int K, int NT>
constexpr size_t bwd_smem_bytes() {
  using Gm = Geom<K>;
  size_t words = 3 * Gm::KK4 + 32 + NT + 2 * (size_t)NSTAGE * NT * Gm::P + (size_t)NSTAGE * NT * TAGP;
  return words * 4;
}

template <int NT>
__device__ __forceinline__ void stage_tags_b(int* dst, const int32_t* __restrict__ gbase, int L, int t0, int nv,
                                             const int* s_len, int vec16) {
  constexpr int T = T_CHUNK;
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
      if (r < nv && e < min(steps, s_len[r] - t0)) cp_async4(dst + r * TAGP + e, gbase + (size_t)r * L + t0 + e);
    }
  }
}

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
  constexpr bool ACC_REGS = (K <= 10);  // K*K rank-1 accumulators in registers

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

  for (int e = tid; e < K * K; e += NT) {
    s_tr[e] = trans[e];
    s_dT[e] = 0.f;
  }
  int mylen = 0;
  if (tid < nv) mylen = min(max(seq_len[row0 + tid], 0), L);
  s_len[tid] = mylen;
  const int bmax = block_max_int<NT>(mylen, reinterpret_cast<int*>(s_x));
  if (tid < K) {
    float rm = -INFINITY;
    for (int j = 0; j < K; ++j) rm = fmaxf(rm, s_tr[tid * K + j]);
    s_rmax[tid] = rm;
  }
  __syncthreads();
  bool fast = true;
  {
    float lo = INFINITY, hi = -INFINITY;
    for (int e = 0; e < K * K; ++e) {
      lo = fminf(lo, s_tr[e]);
      hi = fmaxf(hi, s_tr[e]);
    }
    if (!(hi - lo < 30.f) || !(fabsf(hi) < 1e30f) || !(fabsf(lo) < 1e30f)) fast = false;
  }
  for (int e = tid; e < K * K; e += NT) s_E[e] = fast ? expf(s_tr[e] - s_rmax[e / K]) : 0.f;
  __syncthreads();

  const float* gx = logits + (size_t)row0 * LK;
  const float* ga = alpha_ws + (size_t)row0 * LK;
  const int32_t* gt = tags + (size_t)row0 * L;
  float* gd = d_logits + (size_t)row0 * LK;
  const int nchunk = (bmax + T - 1) / T;
  const int nchunk_all = (L + T - 1) / T;

  // chunks past the longest row of this CTA: pure zero fill
  for (int c = nchunk; c < nchunk_all; ++c) {
    const int t0 = c * T;
    const int ne = min(T, L - t0) * K;
    for (int idx = tid; idx < NT * Gm::CE; idx += NT) {
      const int r = idx / Gm::CE, e = idx - r * Gm::CE;
      if (r < nv && e < ne) gd[(size_t)r * LK + (size_t)t0 * K + e] = 0.f;
    }
  }

  auto stage = [&](int c, int buf) {
    stage_logits<K, NT>(s_x + buf * NT * P, gx, LK, c * T, L, nv, s_len, vec_logits);
    stage_logits<K, NT>(s_a + buf * NT * P, ga, LK, c * T, L, nv, s_len, vec_logits);
    stage_tags_b<NT>(s_tags + buf * NT * TAGP, gt, L, c * T, nv, s_len, vec_tags);
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
        const int4* tp = reinterpret_cast<const int4*>(s_tags + buf * NT * TAGP + tid * TAGP);
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
                if (fast) {
                  mq = u[0];
#pragma unroll UNR
                  for (int j = 1; j < K; ++j) mq = fmaxf(mq, u[j]);
#pragma unroll UNR
                  for (int j = 0; j < K; ++j) q[j] = __expf(u[j] - mq);
#pragma unroll UNR
                  for (int i = 0; i < K; ++i) {
                    float sum = 0.f;
#pragma unroll UNR
                    for (int j = 0; j < K; ++j) sum = fmaf(s_E[i * K + j], q[j], sum);
                    beta[i] = mq + rmx[i] + __logf(sum);
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
                    u_keep[i] = u[i];
                  }
                }
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
    // coalesced store of this chunk's d_logits (zeros at t >= len)
    {
      const float* sx = s_x + buf * NT * P;
      const int ne = min(T, L - t0) * K;
      if (vec_logits) {
        for (int idx = tid; idx < NT * Gm::NQ; idx += NT) {
          const int r = idx / Gm::NQ, qq = idx - r * Gm::NQ;
          if (r < nv && 4 * qq < ne) {
            const int valid = (s_len[r] - t0) * K;  // elements [0, valid) carry gradients
            float4 v = *reinterpret_cast<const float4*>(sx + r * P + 4 * qq);
            if (4 * qq + 0 >= valid) v.x = 0.f;
            if (4 * qq + 1 >= valid) v.y = 0.f;
            if (4 * qq + 2 >= valid) v.z = 0.f;
            if (4 * qq + 3 >= valid) v.w = 0.f;
            *reinterpret_cast<float4*>(gd + (size_t)r * LK + (size_t)t0 * K + 4 * qq) = v;
          }
        }
      } else {
        for (int idx = tid; idx < NT * Gm::CE; idx += NT) {
          const int r = idx / Gm::CE, e = idx - r * Gm::CE;
          if (r < nv && e < ne) {
            const int valid = (s_len[r] - t0) * K;
            gd[(size_t)r * LK + (size_t)t0 * K + e] = (e < valid) ? sx[r * P + e] : 0.f;
          }
        }
      }
    }
    __syncthreads();
  }

  // ---- reduce the per-thread pair accumulators into d_trans
  if constexpr (ACC_REGS) {
#pragma unroll
    for (int e = 0; e < K * K; ++e) {
      float v = (tid < nv) ? -gcoef * acc[e] * s_E[e] : 0.f;
      v = warp_sum(v);
      if ((tid & 31) == 0 && v != 0.f) atomicAdd(&s_dT[e], v);
    }
  }
  __syncthreads();
  for (int e = tid; e < K * K; e += NT) {
    const float v = s_dT[e];
    if (v != 0.f) atomicAdd(&d_trans[e], v);
  }
}

template <int K, int NT>
int launch_bwd_nt(const float* logits, const int32_t* tags, const int32_t* seq_len, const float* trans,
                  const float* alpha_ws, const float* logz, const float* d_ll, float scale, float* d_logits,
                  float* d_trans, int B, int L, cudaStream_t st) {
  const size_t smem = bwd_smem_bytes<K, NT>();
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
  if (bwd_smem_bytes<K, 64>() <= kMaxSmem && B > ner_num_sms() * 64 * 2)
    return launch_bwd_nt<K, 64>(logits, tags, seq_len, trans, alpha_ws, logz, d_ll, scale, d_logits, d_trans, B, L, st);
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
  if (B <= NER_CRF_SMALL_B) {   // few sequences: the lane-per-tag kernel (crf_small.cu) walks a much shorter chain
    const int rc = ner_crf_loglik_bwd_small(logits, tags, seq_len, trans, alpha_ws, logz, d_ll, scale, d_logits, d_trans, B, L,
                                            K, st);
    if (rc != NER_ERR_UNSUPPORTED) return rc;
  }
#define CALL(KK) \
  return launch_bwd<KK>(logits, tags, seq_len, trans, alpha_ws, logz, d_ll, scale, d_logits, d_trans, B, L, st)
  NER_CRF_DISPATCH_K(K, CALL)
#undef CALL
  return NER_ERR_UNSUPPORTED;
}
