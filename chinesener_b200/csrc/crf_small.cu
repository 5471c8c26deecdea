// Latency-oriented CRF kernels for small batches (B below a few thousand sequences), sm_90a.
//
// The thread-per-sequence kernels (crf_viterbi.cu / crf_loglik.cu) are built for HBM throughput at
// very large B; at the model's real batch (B = 64) they leave one warp walking a 128-step
// dependent chain of ~400 instructions per step.  Here ONE LANE OWNS ONE TAG: a group of
// GS = 8/16/32 lanes holds the K-wide DP state of one sequence (32/GS sequences per warp, one warp
// per CTA so the few sequences spread over many SMs), the K predecessors are exchanged with
// __shfl_sync, and the per-step critical path drops to ~K shuffle+add+compare.
// Arithmetic (fp32 association order, strict '>' first-max ties, exact per-column logsumexp) is
// identical to the throughput kernels, so Viterbi stays bit-exact (reference semantics:
// tf.contrib.crf as called at tools/layer.py:122,140; SURVEY.md Appendix A.1).
#include "crf_common.cuh"

namespace {

using namespace nerdev;
using namespace crf;

constexpr int PF = 4;  // emission prefetch depth (time steps)

template <int K>
__global__ void __launch_bounds__(32)
crf_viterbi_lanes_kernel(const float* __restrict__ logits, const int32_t* __restrict__ seq_len,
                         const float* __restrict__ trans, int32_t* __restrict__ tags_out,
                         float* __restrict__ best_score, int B, int L) {
  constexpr int GS = Lanes<K>::GS, SPW = Lanes<K>::SPW;
  extern __shared__ uint8_t sm_raw[];
  uint8_t* s_bp = sm_raw;                                            // [L][32]
  int32_t* s_tags = reinterpret_cast<int32_t*>(sm_raw + (((size_t)L * 32 + 15) & ~(size_t)15));  // [SPW][L]

  const int lane = threadIdx.x;
  const int g = lane / GS, j = lane % GS;
  const int b = blockIdx.x * SPW + g;
  const bool seq_ok = b < B;
  const bool tag_ok = j < K;
  int len = 1;
  if (seq_ok) len = min(max(seq_len[b], 1), L);  // len <= 0 decodes like len 1 (TF quirk)
  int wmax = len;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));

  float tc[K];  // trans[i][j] for this lane's tag j
#pragma unroll
  for (int i = 0; i < K; ++i) tc[i] = tag_ok ? trans[i * K + j] : 0.f;

  const float* xp = logits + (size_t)(seq_ok ? b : 0) * L * K + (tag_ok ? j : 0);
  auto ld = [&](int t) -> float { return (seq_ok && tag_ok && t < len) ? xp[(size_t)t * K] : -INFINITY; };
  float s = ld(0);
  float xq[PF];
#pragma unroll
  for (int i = 0; i < PF; ++i) xq[i] = ld(1 + i);

  for (int t0 = 1; t0 < wmax; t0 += PF) {
#pragma unroll
    for (int u = 0; u < PF; ++u) {
      const int t = t0 + u;
      const float x = xq[u];
      xq[u] = ld(t + PF);
      if (t < wmax) {
        float best = __shfl_sync(0xffffffffu, s, g * GS) + tc[0];
        int arg = 0;
#pragma unroll
        for (int i = 1; i < K; ++i) {
          const float v = __shfl_sync(0xffffffffu, s, g * GS + i) + tc[i];
          if (v > best) {
            best = v;
            arg = i;
          }
        }
        if (t < len) {
          s = tag_ok ? x + best : -INFINITY;
          s_bp[t * 32 + lane] = (uint8_t)arg;
        }
      }
    }
  }
  // first-max argmax over the group's tags
  float bv = s;
  int bi = j;
#pragma unroll
  for (int o = GS / 2; o > 0; o >>= 1) {
    const float ov = __shfl_down_sync(0xffffffffu, bv, o, GS);
    const int oi = __shfl_down_sync(0xffffffffu, bi, o, GS);
    if (ov > bv || (ov == bv && oi < bi)) {
      bv = ov;
      bi = oi;
    }
  }
  __syncwarp();
  if (j == 0 && seq_ok) {
    if (best_score != nullptr) best_score[b] = bv;
    int y = bi;
    for (int t = len - 1; t >= 1; --t) {
      s_tags[g * L + t] = y;
      y = s_bp[t * 32 + g * GS + y];
    }
    s_tags[g * L] = y;
  }
  __syncwarp();
  if (seq_ok)
    for (int t = j; t < L; t += GS) tags_out[(size_t)b * L + t] = (t < len) ? s_tags[g * L + t] : 0;
}

template <int K>
__global__ void __launch_bounds__(32)
crf_loglik_lanes_kernel(const float* __restrict__ logits, const int32_t* __restrict__ tags,
                        const int32_t* __restrict__ seq_len, const float* __restrict__ trans,
                        float* __restrict__ ll, float* __restrict__ logz_out, float* __restrict__ alpha_ws, int B,
                        int L) {
  constexpr int GS = Lanes<K>::GS, SPW = Lanes<K>::SPW;
  __shared__ float s_tr[K * K];
  const int lane = threadIdx.x;
  const int g = lane / GS, j = lane % GS;
  const int b = blockIdx.x * SPW + g;
  const bool seq_ok = b < B;
  const bool tag_ok = j < K;
  for (int e = lane; e < K * K; e += 32) s_tr[e] = trans[e];
  int rawlen = 0, len = 1;
  if (seq_ok) {
    rawlen = seq_len[b];
    len = min(max(rawlen, 1), L);
  }
  const int wmax = lanes_wmax(len);
  __syncwarp();

  float tc[K];
#pragma unroll
  for (int i = 0; i < K; ++i) tc[i] = tag_ok ? s_tr[i * K + j] : 0.f;

  const size_t base = (size_t)(seq_ok ? b : 0) * L;
  const float* xp = logits + base * K + (tag_ok ? j : 0);
  const int32_t* tp = tags + base;
  auto ld = [&](int t) -> float { return (seq_ok && tag_ok && t < len) ? xp[(size_t)t * K] : -INFINITY; };
  auto ldtag = [&](int t) -> int { return (seq_ok && t < len) ? min(max(tp[t], 0), K - 1) : 0; };

  float a = ld(0);
  int prev = ldtag(0);
  float score = __shfl_sync(0xffffffffu, a, g * GS + prev);  // x[0][tag_0] (all lanes of the group hold it)
  if (alpha_ws != nullptr && seq_ok && tag_ok) alpha_ws[base * K + j] = a;
  float xq[PF];
  int tq[PF];
#pragma unroll
  for (int i = 0; i < PF; ++i) {
    xq[i] = ld(1 + i);
    tq[i] = ldtag(1 + i);
  }

  for (int t0 = 1; t0 < wmax; t0 += PF) {
#pragma unroll
    for (int u = 0; u < PF; ++u) {
      const int t = t0 + u;
      const float x = xq[u];
      const int tag = tq[u];
      xq[u] = ld(t + PF);
      tq[u] = ldtag(t + PF);
      if (t < wmax) {
        // exact logsumexp_i(alpha_i + trans[i][j]) with its own max (tf.reduce_logsumexp)
        const float na = lanes_alpha_step<K>(a, x, tc, g);
        const float xtag = __shfl_sync(0xffffffffu, x, g * GS + tag);
        if (t < len) {
          a = tag_ok ? na : -INFINITY;
          score += xtag + s_tr[prev * K + tag];
          prev = tag;
          if (alpha_ws != nullptr && seq_ok && tag_ok) alpha_ws[(base + t) * K + j] = a;
        }
      }
    }
  }
  float logz = lanes_logsumexp<K>(a, tag_ok);
  if (j == 0 && seq_ok) {
    if (rawlen <= 0) {
      logz = 0.f;
      score = 0.f;
    }
    ll[b] = score - logz;
    if (logz_out != nullptr) logz_out[b] = logz;
  }
}

// Backward of the log-likelihood for small batches, lane i = tag i (see crf_bwd.cu for the closed form):
//   w_j          = x_t[j] + beta_t[j]                                   (lane j; broadcast by shuffles)
//   v_ij         = trans[i][j] + w_j                                    (lane i, all j)
//   beta_{t-1}[i] = logsumexp_j v_ij                                    (own max, as reduce_logsumexp)
//   M_t[i][j]    = exp(alpha_{t-1}[i] - logZ + v_ij)                    pair marginal, accumulated in registers
//   d_x[t][i]    = g * (1[y_t = i] - exp(alpha_t[i] + beta_t[i] - logZ))
// g = d_ll[b] * scale.  d_trans gets one atomic per (sequence, i, j) at the end.
template <int K>
__global__ void __launch_bounds__(32)
crf_loglik_bwd_lanes_kernel(const float* __restrict__ logits, const int32_t* __restrict__ tags,
                            const int32_t* __restrict__ seq_len, const float* __restrict__ trans,
                            const float* __restrict__ alpha_ws, const float* __restrict__ logz,
                            const float* __restrict__ d_ll, float scale, float* __restrict__ d_logits,
                            float* __restrict__ d_trans, int B, int L) {
  constexpr int GS = Lanes<K>::GS, SPW = Lanes<K>::SPW;
  const int lane = threadIdx.x;
  const int g = lane / GS, i = lane % GS;
  const int b = blockIdx.x * SPW + g;
  const bool seq_ok = b < B;
  const bool tag_ok = i < K;
  const int len = seq_ok ? min(max(seq_len[b], 0), L) : 0;
  const int wmax = lanes_wmax(len);

  float tr[K];   // row i of the transition matrix
#pragma unroll
  for (int jj = 0; jj < K; ++jj) tr[jj] = tag_ok ? trans[i * K + jj] : 0.f;
  float acc[K];  // sum_t (M_t[i][j] - 1[y_{t-1}=i, y_t=j])
#pragma unroll
  for (int jj = 0; jj < K; ++jj) acc[jj] = 0.f;

  const size_t base = (size_t)(seq_ok ? b : 0) * L;
  const float lz = seq_ok ? logz[b] : 0.f;
  const float gco = seq_ok ? (d_ll != nullptr ? d_ll[b] : 1.f) * scale : 0.f;
  const float* xp = logits + base * K + (tag_ok ? i : 0);
  const float* ap = alpha_ws + base * K + (tag_ok ? i : 0);
  const int32_t* tp = tags + base;
  float* dp = d_logits + base * K + (tag_ok ? i : 0);
  const bool io = seq_ok && tag_ok;
  // zero fill past the sequence end
  if (io)
    for (int t = len; t < L; ++t) dp[(size_t)t * K] = 0.f;

  auto ldx = [&](int t) -> float { return (io && t >= 0 && t < len) ? xp[(size_t)t * K] : 0.f; };
  auto lda = [&](int t) -> float { return (io && t >= 0 && t < len) ? ap[(size_t)t * K] : 0.f; };
  auto ldtag = [&](int t) -> int { return (seq_ok && t >= 0 && t < len) ? min(max(tp[t], 0), K - 1) : 0; };

  // iteration s handles position t = len-1-s of its own sequence (the sequences of a warp may differ in
  // length: the shorter one simply runs out of live steps first); operands are fetched PF iterations ahead
  float beta = 0.f;
  float xq[PF], aq[PF];
  int tq[PF];
#pragma unroll
  for (int u = 0; u < PF; ++u) {
    xq[u] = ldx(len - 1 - u);
    aq[u] = lda(len - 2 - u);
    tq[u] = ldtag(len - 2 - u);
  }
  float a_t = lda(len - 1);     // alpha_t[i] of the current position
  int tag_t = ldtag(len - 1);   // y_t
  for (int s0 = 0; s0 < wmax; s0 += PF) {
#pragma unroll
    for (int u = 0; u < PF; ++u) {
      const int sidx = s0 + u;
      const int t = len - 1 - sidx;
      const float x = xq[u], a_prev = aq[u];
      const int tag_prev = tq[u];
      xq[u] = ldx(t - PF);
      aq[u] = lda(t - 1 - PF);
      tq[u] = ldtag(t - 1 - PF);
      if (sidx < wmax) {                    // warp-uniform: every lane takes part in the shuffles
        const bool live = t >= 0;           // uniform over the lanes of one sequence
        if (io && live) {
          const float p = __expf(a_t + beta - lz);
          dp[(size_t)t * K] = gco * ((i == tag_t ? 1.f : 0.f) - p);
        }
        float v[K];
        const float m = lanes_gather<K>(v, (tag_ok && live) ? x + beta : -INFINITY, tr, g);
        if (live && t >= 1) {
          const float mm = (fabsf(m) <= 3.0e38f) ? m : 0.f;
          const float am = a_prev - lz;
          float sum = 0.f;
#pragma unroll
          for (int jj = 0; jj < K; ++jj) {
            sum += __expf(v[jj] - mm);
            acc[jj] += __expf(am + v[jj]) - ((i == tag_prev && jj == tag_t) ? 1.f : 0.f);
          }
          beta = __logf(sum) + mm;
          a_t = a_prev;
          tag_t = tag_prev;
        }
      }
    }
  }
  if (io && len > 0) {
#pragma unroll
    for (int jj = 0; jj < K; ++jj) atomicAdd(d_trans + i * K + jj, -gco * acc[jj]);
  }
}

template <int K>
int launch_loglik_bwd_lanes(const float* logits, const int32_t* tags, const int32_t* seq_len, const float* trans,
                            const float* alpha_ws, const float* logz, const float* d_ll, float scale, float* d_logits,
                            float* d_trans, int B, int L, cudaStream_t st) {
  constexpr int SPW = Lanes<K>::SPW;
  crf_loglik_bwd_lanes_kernel<K><<<(B + SPW - 1) / SPW, 32, 0, st>>>(logits, tags, seq_len, trans, alpha_ws, logz, d_ll, scale,
                                                                 d_logits, d_trans, B, L);
  return ner_launch_status();
}

template <int K>
int launch_viterbi_lanes(const float* logits, const int32_t* seq_len, const float* trans, int32_t* tags_out,
                         float* best_score, int B, int L, cudaStream_t st) {
  constexpr int SPW = Lanes<K>::SPW;
  const size_t smem = crf::viterbi_lanes_smem_bytes<K>(L);
  if (smem > crf::kMaxSmem) return NER_ERR_UNSUPPORTED;
  auto kern = crf_viterbi_lanes_kernel<K>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  }
  kern<<<(B + SPW - 1) / SPW, 32, smem, st>>>(logits, seq_len, trans, tags_out, best_score, B, L);
  return ner_launch_status();
}

template <int K>
int launch_loglik_lanes(const float* logits, const int32_t* tags, const int32_t* seq_len, const float* trans, float* ll,
                        float* logz, float* alpha_ws, int B, int L, cudaStream_t st) {
  constexpr int SPW = Lanes<K>::SPW;
  crf_loglik_lanes_kernel<K><<<(B + SPW - 1) / SPW, 32, 0, st>>>(logits, tags, seq_len, trans, ll, logz, alpha_ws, B, L);
  return ner_launch_status();
}

}  // namespace

// Internal entry points used by ner_crf_viterbi / ner_crf_loglik_fwd for small batches.
int ner_crf_viterbi_small(const float* logits, const int32_t* seq_len, const float* trans, int32_t* tags_out,
                          float* best_score, int B, int L, int K, cudaStream_t st) {
#define CALL(KK) return launch_viterbi_lanes<KK>(logits, seq_len, trans, tags_out, best_score, B, L, st)
  NER_CRF_DISPATCH_K(K, CALL)
#undef CALL
  return NER_ERR_UNSUPPORTED;
}

int ner_crf_loglik_bwd_small(const float* logits, const int32_t* tags, const int32_t* seq_len, const float* trans,
                             const float* alpha_ws, const float* logz, const float* d_ll, float scale, float* d_logits,
                             float* d_trans, int B, int L, int K, cudaStream_t st) {
#define CALL(KK) \
  return launch_loglik_bwd_lanes<KK>(logits, tags, seq_len, trans, alpha_ws, logz, d_ll, scale, d_logits, d_trans, B, L, st)
  NER_CRF_DISPATCH_K(K, CALL)
#undef CALL
  return NER_ERR_UNSUPPORTED;
}

int ner_crf_loglik_fwd_small(const float* logits, const int32_t* tags, const int32_t* seq_len, const float* trans,
                             float* ll, float* logz, float* alpha_ws, int B, int L, int K, cudaStream_t st) {
#define CALL(KK) return launch_loglik_lanes<KK>(logits, tags, seq_len, trans, ll, logz, alpha_ws, B, L, st)
  NER_CRF_DISPATCH_K(K, CALL)
#undef CALL
  return NER_ERR_UNSUPPORTED;
}
