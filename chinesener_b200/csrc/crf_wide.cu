// Wide-tag-set CRF kernels, sm_90a: Viterbi, log-likelihood forward and its gradient for 1 <= K <= 128 tags
// (NER_MAX_TAGS_WIDE).  They serve tag sets past the 32 of the K-specialised kernels (crf_viterbi.cu, crf_loglik.cu,
// crf_bwd.cu, crf_small.cu); they accept K <= 32 too, so the tests can pin them to those kernels on the same inputs.
//
// Work decomposition: a CTA of W = 64 or 128 threads (K padded up to W) serves G = 1 or 4 sequences.  Thread j owns
// tag j of each of its G sequences.  The K x K transition matrix (or its exp-space copy E = exp(T - max T)) sits in
// shared memory as [i][W + j], so the K reads of one step by thread j are conflict-free, and each read serves all G
// sequences.  The previous step's K-wide state is in shared memory as [i][g] and is read as broadcasts.  Each step is
// one (or, on the fast paths, two) __syncthreads; nothing of size K x K leaves the chip.
//
//  - Viterbi: thread j takes the first maximum over i (strict '>', ascending i) of s[i] + T[i][j], then adds x[t][j]:
//    the association order of ner_crf_viterbi, so tags and best_score are bit-exact.  The byte-wide backpointers of a
//    row are L*K bytes (512 KB at L = 4095, K = 128), so they go to a caller workspace, one coalesced byte per thread
//    and step.  The backtrace stages kBtChunk steps of them in shared memory at a time and walks those there.
//  - Forward: the exact path (flags bit0, or a transition matrix spanning >= 30 nats or not finite, crf_common.cuh's
//    rule) is a per-column logsumexp with its own max.  The fast path keeps alpha = lacc + a with a per-row offset lacc
//    and runs
//        p_i = exp(a_i - m),  a'_j = x_j + log(sum_i p_i E[i][j]),  lacc' = lacc + m + tmax,   m = max_i a_i
//    i.e. K exps, K logs and K*K FMAs per step.  Since E >= e^-30 and max p = 1, the sum never underflows, and a stays
//    within a few nats of 0, so its rounding does not grow with the row's length.
//  - Backward: the marginals recursion, with thread i owning source tag i: beta_{t-1}[i] = logsumexp_j(T[i][j] + u_j),
//    u_j = x_t[j] + beta_t[j], and the pair marginals xi_t(i,j) = exp(alpha_{t-1}[i] + T[i][j] + u_j - logZ) summed into
//    a per-CTA K x K shared slab whose column i belongs only to thread i (no atomics in the CTA).  The fast path sums
//    pa_i * q_j with q_j = exp(u_j - max u) and scales by E once at the end.  The gold-path counts go to a second slab.
//    One global atomic add per (CTA, i, j) flushes both into d_trans.
#include "crf_common.cuh"

namespace {

using namespace nerdev;

constexpr int kBtChunk = 64;  // Viterbi backtrace: steps of backpointers staged per pass

// Per-sequence reduction over the CTA's W threads of v[g]; every thread gets the result.  red holds [G][W/32] floats
// and must not be written again until every thread has read it (the callers alternate two buffers).
template <int W, int G, bool MAX>
__device__ __forceinline__ void block_reduce(float (&v)[G], float* red) {
  constexpr int NW = W / 32;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    v[g] = MAX ? warp_max(v[g]) : warp_sum(v[g]);
    if (lane == 0) red[g * NW + w] = v[g];
  }
  __syncthreads();
#pragma unroll
  for (int g = 0; g < G; ++g) {
    float r = red[g * NW];
#pragma unroll
    for (int q = 1; q < NW; ++q) r = MAX ? fmaxf(r, red[g * NW + q]) : r + red[g * NW + q];
    v[g] = r;
  }
}

__device__ __forceinline__ float finite_or_zero(float m) { return (fabsf(m) <= 3.0e38f) ? m : 0.f; }

// trans -> s_m[i][W + j] (zero in the pad columns), and crf_common.cuh's trans_is_narrow over the K x K entries as a
// CTA reduction.  Returns whether the fast path applies; tmax gets the largest entry.
template <int W>
__device__ __forceinline__ bool stage_trans(const float* __restrict__ trans, int K, float* s_m, float* red,
                                            float& tmax) {
  float lo = INFINITY, hi = -INFINITY;
  for (int e = threadIdx.x; e < K * W; e += W) {
    const int i = e / W, j = e - i * W;
    const float v = j < K ? trans[i * K + j] : 0.f;
    s_m[e] = v;
    if (j < K) {
      lo = fminf(lo, v);
      hi = fmaxf(hi, v);
    }
  }
  float r[2] = {hi, -lo};
  block_reduce<W, 2, true>(r, red);
  __syncthreads();
  tmax = r[0];
  return (r[0] + r[1] < 30.f) && (fabsf(r[0]) < 1e30f) && (fabsf(r[1]) < 1e30f);
}

// ---------------------------------------------------------------------------------------------------------- Viterbi
template <int W, int G>
constexpr size_t viterbi_smem_bytes(int K) {
  return 4 * ((size_t)K * W + 2 * (size_t)G * W) + (size_t)G * kBtChunk * W;
}

template <int W, int G>
__global__ void __launch_bounds__(W)
crf_wide_viterbi_kernel(const float* __restrict__ logits, const int32_t* __restrict__ seq_len,
                        const float* __restrict__ trans, int32_t* __restrict__ tags_out,
                        float* __restrict__ best_score, uint8_t* bp, int B, int L, int K) {
  extern __shared__ __align__(16) float smem[];
  float* s_tr = smem;                                           // [K][W]
  float* s_s = s_tr + K * W;                                    // [2][W][G] scores of the previous step
  uint8_t* s_bp = reinterpret_cast<uint8_t*>(s_s + 2 * G * W);  // [G][kBtChunk][W] backpointers being walked
  __shared__ int s_y[G];

  const int j = threadIdx.x;
  const bool tag_ok = j < K;
  const int b0 = blockIdx.x * G;
  for (int e = j; e < K * W; e += W) {
    const int i = e / W, jj = e - i * W;
    s_tr[e] = jj < K ? trans[i * K + jj] : 0.f;
  }
  int len[G];
  int lmax = 1;
  const float* xp[G];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const int b = b0 + g;
    len[g] = b < B ? min(max(seq_len[b], 1), L) : 0;  // seq_len <= 0 decodes one position, as ner_crf_viterbi
    lmax = max(lmax, len[g]);
    xp[g] = logits + (size_t)min(b, B - 1) * L * K + (tag_ok ? j : 0);
  }
  auto ld = [&](int g, int t) -> float { return (tag_ok && t < len[g]) ? xp[g][(size_t)t * K] : -INFINITY; };

  float s[G], xn[G];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    s[g] = ld(g, 0);
    s_s[j * G + g] = s[g];
    xn[g] = ld(g, 1);
  }
  __syncthreads();

  for (int t = 1; t < lmax; ++t) {
    const float* cur = s_s + ((t - 1) & 1) * G * W;
    float* nxt = s_s + (t & 1) * G * W;
    float x[G];
#pragma unroll
    for (int g = 0; g < G; ++g) {
      x[g] = xn[g];
      xn[g] = ld(g, t + 1);
    }
    float best[G];
    int arg[G];
    {
      const float t0 = s_tr[j];
#pragma unroll
      for (int g = 0; g < G; ++g) {
        best[g] = cur[g] + t0;
        arg[g] = 0;
      }
    }
#pragma unroll 4
    for (int i = 1; i < K; ++i) {
      const float tij = s_tr[i * W + j];
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const float v = cur[i * G + g] + tij;
        if (v > best[g]) {
          best[g] = v;
          arg[g] = i;
        }
      }
    }
#pragma unroll
    for (int g = 0; g < G; ++g) {
      if (t < len[g]) {
        s[g] = tag_ok ? best[g] + x[g] : -INFINITY;
        if (tag_ok) bp[((size_t)(b0 + g) * L + t) * K + j] = (uint8_t)arg[g];
      }
      nxt[j * G + g] = s[g];
    }
    __syncthreads();
  }

  // first maximum of the last step's scores (lowest tag on a tie), then the tags past each row's end
  const float* fin = s_s + ((lmax - 1) & 1) * G * W;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    if (j == g && len[g] > 0) {
      float bv = fin[g];
      int bi = 0;
      for (int k = 1; k < K; ++k) {
        const float v = fin[k * G + g];
        if (v > bv) {
          bv = v;
          bi = k;
        }
      }
      s_y[g] = bi;
      if (best_score != nullptr) best_score[b0 + g] = bv;
    }
  }
#pragma unroll
  for (int g = 0; g < G; ++g)
    if (len[g] > 0)
      for (int t = len[g] + j; t < L; t += W) tags_out[(size_t)(b0 + g) * L + t] = 0;
  __syncthreads();

  // backtrace, kBtChunk steps at a time: stage bp[lo, hi) of every row, then thread g walks row g through them
  int y = j < G ? s_y[j] : 0;
  int mylen = 0;  // len[j] for the walking threads j < G
#pragma unroll
  for (int g = 0; g < G; ++g)
    if (j == g) mylen = len[g];
  for (int hi = lmax; hi > 1; hi -= kBtChunk) {
    const int lo = max(hi - kBtChunk, 1);
#pragma unroll
    for (int g = 0; g < G; ++g)
      if (tag_ok)
        for (int t = lo; t < min(hi, len[g]); ++t)
          s_bp[(g * kBtChunk + (t - lo)) * W + j] = bp[((size_t)(b0 + g) * L + t) * K + j];
    __syncthreads();
    if (mylen > 0) {
      int32_t* out = tags_out + (size_t)(b0 + j) * L;
      for (int t = min(hi, mylen) - 1; t >= lo; --t) {
        out[t] = y;
        y = s_bp[(j * kBtChunk + (t - lo)) * W + y];
      }
    }
    __syncthreads();
  }
  if (mylen > 0) tags_out[(size_t)(b0 + j) * L] = y;
}

// --------------------------------------------------------------------------------------------------------- forward
template <int W, int G>
constexpr size_t fwd_smem_bytes(int K) {
  return 4 * ((size_t)K * W + 2 * (size_t)G * W + 2 * (size_t)G * (W / 32) + 2 * (W / 32));
}

template <int W, int G>
__global__ void __launch_bounds__(W)
crf_wide_fwd_kernel(const float* __restrict__ logits, const int32_t* __restrict__ tags,
                    const int32_t* __restrict__ seq_len, const float* __restrict__ trans, float* __restrict__ ll,
                    float* __restrict__ logz_out, float* __restrict__ alpha_ws, int B, int L, int K, int force_exact) {
  constexpr int NW = W / 32;
  extern __shared__ __align__(16) float smem[];
  float* s_m = smem;                   // [K][W]: trans (exact path) or E = exp(trans - tmax) (fast path)
  float* s_a = s_m + K * W;            // [2][W][G]: alpha (exact) or p = exp(alpha - m) (fast) of the previous step
  float* s_red = s_a + 2 * G * W;      // [2][G][NW]
  float* s_red2 = s_red + 2 * G * NW;  // [2][NW], the trans range

  const int j = threadIdx.x;
  const bool tag_ok = j < K;
  const int b0 = blockIdx.x * G;
  float tmax;
  const bool fast = stage_trans<W>(trans, K, s_m, s_red2, tmax) && !force_exact;
  if (fast) {
    for (int e = j; e < K * W; e += W) s_m[e] = (e % W) < K ? expf(s_m[e] - tmax) : 0.f;
  }

  int rawlen[G], len[G];
  int lmax = 1;
  const float* xp[G];
  const int32_t* tp[G];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const int b = b0 + g;
    rawlen[g] = b < B ? seq_len[b] : 0;
    len[g] = b < B ? min(max(rawlen[g], 1), L) : 0;
    lmax = max(lmax, len[g]);
    xp[g] = logits + (size_t)min(b, B - 1) * L * K + (tag_ok ? j : 0);
    tp[g] = tags + (size_t)min(b, B - 1) * L;
  }
  auto ld = [&](int g, int t) -> float { return (tag_ok && t < len[g]) ? xp[g][(size_t)t * K] : -INFINITY; };
  auto ldtag = [&](int g, int t) -> int { return t < len[g] ? min(max(tp[g][t], 0), K - 1) : 0; };
  auto store = [&](int g, int t, float v) {
    if (alpha_ws != nullptr && tag_ok && t < len[g]) alpha_ws[((size_t)(b0 + g) * L + t) * K + j] = v;
  };

  // alpha_j = lacc + a[j]: the fast path moves each step's common offset (max a + max T) into the per-row scalar lacc, so
  // a[] stays within a few nats of 0 and its fp32 rounding does not grow with the row's length (lacc is one rounding
  // per step, as the K-specialised kernels' scaled-probability state has).  The exact path keeps lacc = 0.
  float a[G], lacc[G], xn[G], score[G];
  int prev[G], yn[G];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    a[g] = ld(g, 0);
    lacc[g] = 0.f;
    store(g, 0, a[g]);
    prev[g] = ldtag(g, 0);
    score[g] = (len[g] > 0 && j == prev[g]) ? a[g] : 0.f;
    xn[g] = ld(g, 1);
    yn[g] = ldtag(g, 1);
  }
  __syncthreads();  // s_m complete

  for (int t = 1; t < lmax; ++t) {
    const int par = t & 1;
    float* sa = s_a + par * G * W;
    float x[G];
    int y[G];
#pragma unroll
    for (int g = 0; g < G; ++g) {
      x[g] = xn[g];
      y[g] = yn[g];
      xn[g] = ld(g, t + 1);
      yn[g] = ldtag(g, t + 1);
    }
    float na[G], off[G];
#pragma unroll
    for (int g = 0; g < G; ++g) off[g] = 0.f;
    if (fast) {
      float m[G];
#pragma unroll
      for (int g = 0; g < G; ++g) m[g] = a[g];
      block_reduce<W, G, true>(m, s_red + par * G * NW);
#pragma unroll
      for (int g = 0; g < G; ++g) {
        m[g] = finite_or_zero(m[g]);
        sa[j * G + g] = expf(a[g] - m[g]);
      }
      __syncthreads();
      float acc[G];
#pragma unroll
      for (int g = 0; g < G; ++g) acc[g] = 0.f;
#pragma unroll 4
      for (int i = 0; i < K; ++i) {
        const float e = s_m[i * W + j];
#pragma unroll
        for (int g = 0; g < G; ++g) acc[g] = fmaf(sa[i * G + g], e, acc[g]);
      }
#pragma unroll
      for (int g = 0; g < G; ++g) {
        na[g] = x[g] + logf(acc[g]);
        off[g] = m[g] + tmax;
      }
    } else {
#pragma unroll
      for (int g = 0; g < G; ++g) sa[j * G + g] = a[g];
      __syncthreads();
      float m[G], sum[G];
#pragma unroll
      for (int g = 0; g < G; ++g) {
        m[g] = -INFINITY;
        sum[g] = 0.f;
      }
#pragma unroll 4
      for (int i = 0; i < K; ++i) {
        const float tr = s_m[i * W + j];
#pragma unroll
        for (int g = 0; g < G; ++g) m[g] = fmaxf(m[g], sa[i * G + g] + tr);
      }
#pragma unroll
      for (int g = 0; g < G; ++g) m[g] = finite_or_zero(m[g]);
#pragma unroll 4
      for (int i = 0; i < K; ++i) {
        const float tr = s_m[i * W + j];
#pragma unroll
        for (int g = 0; g < G; ++g) sum[g] += expf(sa[i * G + g] + tr - m[g]);
      }
#pragma unroll
      for (int g = 0; g < G; ++g) na[g] = x[g] + (logf(sum[g]) + m[g]);
    }
#pragma unroll
    for (int g = 0; g < G; ++g) {
      if (t < len[g]) {
        a[g] = tag_ok ? na[g] : -INFINITY;
        lacc[g] += off[g];
        store(g, t, lacc[g] + a[g]);
        if (j == y[g]) score[g] += x[g] + trans[prev[g] * K + j];
        prev[g] = y[g];
      }
    }
  }

  // log Z = logsumexp_j alpha_j (with its own max), the gold score summed over the CTA
  float m[G], e[G];
#pragma unroll
  for (int g = 0; g < G; ++g) m[g] = a[g];
  block_reduce<W, G, true>(m, s_red);
#pragma unroll
  for (int g = 0; g < G; ++g) {
    m[g] = finite_or_zero(m[g]);
    e[g] = tag_ok ? expf(a[g] - m[g]) : 0.f;
  }
  block_reduce<W, G, false>(e, s_red + G * NW);
  block_reduce<W, G, false>(score, s_red);
#pragma unroll
  for (int g = 0; g < G; ++g) {
    if (j == g && len[g] > 0) {
      float logz = lacc[g] + (logf(e[g]) + m[g]);
      float sc = score[g];
      if (rawlen[g] <= 0) {  // crf_log_norm / crf_sequence_score: zero for empty sequences
        logz = 0.f;
        sc = 0.f;
      }
      ll[b0 + g] = sc - logz;
      if (logz_out != nullptr) logz_out[b0 + g] = logz;
    }
  }
}

// -------------------------------------------------------------------------------------------------------- backward
template <int W, int G>
constexpr size_t bwd_smem_bytes(int K) {
  return 4 * (3 * (size_t)K * W + 2 * (size_t)G * W + 2 * (size_t)G * (W / 32) + 2 * (W / 32));
}

template <int W, int G>
__global__ void __launch_bounds__(W)
crf_wide_bwd_kernel(const float* __restrict__ logits, const int32_t* __restrict__ tags,
                    const int32_t* __restrict__ seq_len, const float* __restrict__ trans,
                    const float* __restrict__ alpha_ws, const float* __restrict__ logz, const float* __restrict__ d_ll,
                    float scale, float* __restrict__ d_logits, float* __restrict__ d_trans, int B, int L, int K) {
  constexpr int NW = W / 32;
  extern __shared__ __align__(16) float smem[];
  float* s_mt = smem;                  // [K][W]: s_mt[j][i] = trans[i][j] (exact) or E[i][j] (fast)
  float* s_acc = s_mt + K * W;         // [K][W]: sum of pair marginals, column i of the matrix at [.][i] (thread i)
  float* s_cnt = s_acc + K * W;        // [K][W]: gold-path transition counts, the same layout
  float* s_u = s_cnt + K * W;          // [2][W][G]: u (exact) or q = exp(u - max u) (fast) of the step
  float* s_red = s_u + 2 * G * W;      // [2][G][NW]
  float* s_red2 = s_red + 2 * G * NW;  // [2][NW]

  const int i = threadIdx.x;  // this thread's tag: destination for the unary terms, source for the pairs
  const bool tag_ok = i < K;
  const int b0 = blockIdx.x * G;

  // transposed trans / E and the zeroed slabs
  float lo = INFINITY, hi = -INFINITY;
  for (int e = i; e < K * W; e += W) {
    const int r = e / W, c = e - r * W;  // s_mt[r][c] = trans[c][r]
    const float v = c < K ? trans[c * K + r] : 0.f;
    s_mt[e] = v;
    s_acc[e] = 0.f;
    s_cnt[e] = 0.f;
    if (c < K) {
      lo = fminf(lo, v);
      hi = fmaxf(hi, v);
    }
  }
  float rng[2] = {hi, -lo};
  block_reduce<W, 2, true>(rng, s_red2);
  const float tmax = rng[0];
  const bool fast = (rng[0] + rng[1] < 30.f) && (fabsf(rng[0]) < 1e30f) && (fabsf(rng[1]) < 1e30f);
  __syncthreads();
  if (fast) {
    for (int e = i; e < K * W; e += W) s_mt[e] = (e % W) < K ? expf(s_mt[e] - tmax) : 0.f;
  }

  int len[G];
  int lmax = 0;
  float lz[G], gco[G];
  size_t base[G];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const int b = b0 + g;
    const bool ok = b < B;
    len[g] = ok ? min(max(seq_len[b], 0), L) : 0;
    lmax = max(lmax, len[g]);
    lz[g] = ok ? logz[b] : 0.f;
    gco[g] = ok ? (d_ll != nullptr ? d_ll[b] : 1.f) * scale : 0.f;
    base[g] = (size_t)min(b, B - 1) * L;
    if (ok && tag_ok)
      for (int t = len[g]; t < L; ++t) d_logits[(base[g] + t) * K + i] = 0.f;
  }
  auto ldx = [&](int g, int t) -> float { return (tag_ok && t >= 0 && t < len[g]) ? logits[(base[g] + t) * K + i] : 0.f; };
  auto lda = [&](int g, int t) -> float {
    return (tag_ok && t >= 0 && t < len[g]) ? alpha_ws[(base[g] + t) * K + i] : -INFINITY;
  };
  auto ldtag = [&](int g, int t) -> int { return (t >= 0 && t < len[g]) ? min(max(tags[base[g] + t], 0), K - 1) : 0; };

  // beta_t[i] = boff + beta[i]: as in the forward, the fast path moves each step's common offset (max u + max T) into
  // the per-row scalar boff, so beta[] stays near 0 and its rounding does not grow with the row's length.
  float beta[G], boff[G], xc[G], ac[G];
  int yc[G];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    beta[g] = 0.f;
    boff[g] = 0.f;
    xc[g] = ldx(g, len[g] - 1);
    ac[g] = lda(g, len[g] - 1);
    yc[g] = ldtag(g, len[g] - 1);
  }
  __syncthreads();  // s_mt complete

  for (int s = 0; s < lmax; ++s) {
    const int par = s & 1;
    float* su = s_u + par * G * W;
    int t[G], yp[G];
    float xp[G], ap[G], u[G];
#pragma unroll
    for (int g = 0; g < G; ++g) {
      t[g] = len[g] - 1 - s;
      xp[g] = ldx(g, t[g] - 1);
      ap[g] = lda(g, t[g] - 1);
      yp[g] = ldtag(g, t[g] - 1);
      if (tag_ok && t[g] >= 0) {
        const float p = expf(ac[g] + (boff[g] - lz[g]) + beta[g]);
        d_logits[(base[g] + t[g]) * K + i] = gco[g] * ((i == yc[g] ? 1.f : 0.f) - p);
      }
      u[g] = (tag_ok && t[g] >= 1) ? xc[g] + beta[g] : -INFINITY;
    }
    float mu[G];
    if (fast) {
#pragma unroll
      for (int g = 0; g < G; ++g) mu[g] = u[g];
      block_reduce<W, G, true>(mu, s_red + par * G * NW);
#pragma unroll
      for (int g = 0; g < G; ++g) {
        mu[g] = finite_or_zero(mu[g]);
        su[i * G + g] = expf(u[g] - mu[g]);
      }
    } else {
#pragma unroll
      for (int g = 0; g < G; ++g) su[i * G + g] = u[g];
    }
    __syncthreads();

    float nb[G], off[G];
#pragma unroll
    for (int g = 0; g < G; ++g) off[g] = 0.f;
    if (fast) {
      // beta_{t-1}[i] = max u + tmax + log sum_j E[i][j] q_j;  xi(i,j) = pa_i E[i][j] q_j
      float pa[G], sum[G];
#pragma unroll
      for (int g = 0; g < G; ++g) {
        pa[g] = t[g] >= 1 ? gco[g] * expf(ap[g] + (boff[g] - lz[g]) + mu[g] + tmax) : 0.f;
        sum[g] = 0.f;
      }
#pragma unroll 4
      for (int jj = 0; jj < K; ++jj) {
        const float e = s_mt[jj * W + i];
        float acc = s_acc[jj * W + i];
#pragma unroll
        for (int g = 0; g < G; ++g) {
          const float q = su[jj * G + g];
          sum[g] = fmaf(e, q, sum[g]);
          acc = fmaf(pa[g], q, acc);
        }
        s_acc[jj * W + i] = acc;
      }
#pragma unroll
      for (int g = 0; g < G; ++g) {
        nb[g] = logf(sum[g]);
        off[g] = mu[g] + tmax;
      }
    } else {
      // beta_{t-1}[i] = logsumexp_j (trans[i][j] + u_j) with its own max m_i;  xi(i,j) = pa_i exp(trans + u - m_i)
      float m[G], pa[G], sum[G];
#pragma unroll
      for (int g = 0; g < G; ++g) {
        m[g] = -INFINITY;
        sum[g] = 0.f;
      }
#pragma unroll 4
      for (int jj = 0; jj < K; ++jj) {
        const float tr = s_mt[jj * W + i];
#pragma unroll
        for (int g = 0; g < G; ++g) m[g] = fmaxf(m[g], tr + su[jj * G + g]);
      }
#pragma unroll
      for (int g = 0; g < G; ++g) {
        m[g] = finite_or_zero(m[g]);
        pa[g] = t[g] >= 1 ? gco[g] * expf(ap[g] + (boff[g] - lz[g]) + m[g]) : 0.f;
      }
#pragma unroll 4
      for (int jj = 0; jj < K; ++jj) {
        const float tr = s_mt[jj * W + i];
        float acc = s_acc[jj * W + i];
#pragma unroll
        for (int g = 0; g < G; ++g) {
          const float e = expf(tr + su[jj * G + g] - m[g]);
          sum[g] += e;
          acc = fmaf(pa[g], e, acc);
        }
        s_acc[jj * W + i] = acc;
      }
#pragma unroll
      for (int g = 0; g < G; ++g) nb[g] = logf(sum[g]) + m[g];
    }
#pragma unroll
    for (int g = 0; g < G; ++g) {
      if (t[g] >= 1) {
        if (i == yp[g]) s_cnt[yc[g] * W + i] += gco[g];
        beta[g] = nb[g];
        boff[g] += off[g];
        xc[g] = xp[g];
        ac[g] = ap[g];
        yc[g] = yp[g];
      }
    }
  }
  __syncthreads();

  // d_trans[r][c] += cnt - sum xi, one global add per (CTA, r, c)
  for (int e = i; e < K * K; e += W) {
    const int c = e / K, r = e - c * K;  // slab entry [c][r] holds matrix entry (r, c)
    const float acc = s_acc[c * W + r];
    const float v = s_cnt[c * W + r] - (fast ? acc * s_mt[c * W + r] : acc);
    if (v != 0.f) atomicAdd(&d_trans[r * K + c], v);
  }
}

// ------------------------------------------------------------------------------------------------------- launches
// Every configuration ner_crf_wide_plan can pick fits one CTA's shared memory at its largest K (K = W), so the plan
// never has to look at shared memory.
template <int W, int G>
constexpr bool fits_at_full_width() {
  return viterbi_smem_bytes<W, G>(W) <= crf::kMaxSmem && fwd_smem_bytes<W, G>(W) <= crf::kMaxSmem &&
         bwd_smem_bytes<W, G>(W) <= crf::kMaxSmem;
}
static_assert(fits_at_full_width<64, 1>() && fits_at_full_width<64, 4>() && fits_at_full_width<128, 1>() &&
                  fits_at_full_width<128, 4>(),
              "a wide CRF configuration exceeds one CTA's shared memory");

#define NER_WIDE_DISPATCH(PLAN, CALL)              \
  switch (PLAN) {                                  \
    case NER_CRF_WIDE_64_G1: CALL(64, 1); break;   \
    case NER_CRF_WIDE_64_G4: CALL(64, 4); break;   \
    case NER_CRF_WIDE_128_G1: CALL(128, 1); break; \
    case NER_CRF_WIDE_128_G4: CALL(128, 4); break; \
    default: return NER_ERR_UNSUPPORTED;           \
  }

template <int W, int G, typename Kern, typename... Args>
int run(Kern kern, size_t smem, int B, cudaStream_t st, Args... args) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  kern<<<(B + G - 1) / G, W, smem, st>>>(args...);
  return ner_launch_status();
}

}  // namespace

extern "C" int ner_crf_wide_plan(int B, int L, int K, int num_sms) {
  if (B < 1 || L < 1 || K < 1 || K > NER_MAX_TAGS_WIDE || num_sms < 1) return NER_CRF_WIDE_NONE;
  // four sequences per CTA once the batch fills every SM with at least two such CTAs: the transition reads are
  // then shared by four rows; below that, one row per CTA spreads the batch over more SMs
  const bool g4 = B >= 8 * num_sms;
  if (K <= 64) return g4 ? NER_CRF_WIDE_64_G4 : NER_CRF_WIDE_64_G1;
  return g4 ? NER_CRF_WIDE_128_G4 : NER_CRF_WIDE_128_G1;
}

extern "C" size_t ner_crf_wide_viterbi_workspace_bytes(int B, int L, int K) {
  if (B < 1 || L < 1 || K < 1 || K > NER_MAX_TAGS_WIDE) return 0;
  return (size_t)B * L * K;
}

extern "C" int ner_crf_wide_viterbi(const float* logits, const int32_t* seq_len, const float* trans, int32_t* tags_out,
                                    float* best_score, void* workspace, size_t workspace_bytes, int B, int L, int K,
                                    ner_stream_t stream) {
  if (B < 0 || L < 1) return NER_ERR_INVALID_ARG;
  if (K < 1 || K > NER_MAX_TAGS_WIDE) return NER_ERR_UNSUPPORTED;
  if (B == 0) return NER_OK;
  if (!logits || !seq_len || !trans || !tags_out) return NER_ERR_INVALID_ARG;
  if (!workspace || workspace_bytes < ner_crf_wide_viterbi_workspace_bytes(B, L, K)) return NER_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* bp = static_cast<uint8_t*>(workspace);
#define CALL(W, G)                                                                                                  \
  return run<W, G>(crf_wide_viterbi_kernel<W, G>, viterbi_smem_bytes<W, G>(K), B, st, logits, seq_len, trans, tags_out, \
                   best_score, bp, B, L, K)
  NER_WIDE_DISPATCH(ner_crf_wide_plan(B, L, K, ner_num_sms()), CALL)
#undef CALL
  return NER_ERR_UNSUPPORTED;
}

extern "C" int ner_crf_wide_loglik_fwd(const float* logits, const int32_t* tags, const int32_t* seq_len,
                                       const float* trans, float* ll, float* logz_out, float* alpha_ws, int B, int L,
                                       int K, int flags, ner_stream_t stream) {
  if (B < 0 || L < 1) return NER_ERR_INVALID_ARG;
  if (K < 1 || K > NER_MAX_TAGS_WIDE) return NER_ERR_UNSUPPORTED;
  if (B == 0) return NER_OK;
  if (!logits || !tags || !seq_len || !trans || !ll) return NER_ERR_INVALID_ARG;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define CALL(W, G)                                                                                                   \
  return run<W, G>(crf_wide_fwd_kernel<W, G>, fwd_smem_bytes<W, G>(K), B, st, logits, tags, seq_len, trans, ll, logz_out, \
                   alpha_ws, B, L, K, flags & 1)
  NER_WIDE_DISPATCH(ner_crf_wide_plan(B, L, K, ner_num_sms()), CALL)
#undef CALL
  return NER_ERR_UNSUPPORTED;
}

extern "C" int ner_crf_wide_loglik_bwd(const float* logits, const int32_t* tags, const int32_t* seq_len,
                                       const float* trans, const float* alpha_ws, const float* logz, const float* d_ll,
                                       float scale, float* d_logits, float* d_trans, int B, int L, int K,
                                       ner_stream_t stream) {
  if (B < 0 || L < 1) return NER_ERR_INVALID_ARG;
  if (K < 1 || K > NER_MAX_TAGS_WIDE) return NER_ERR_UNSUPPORTED;
  if (B == 0) return NER_OK;
  if (!logits || !tags || !seq_len || !trans || !alpha_ws || !logz || !d_logits || !d_trans) return NER_ERR_INVALID_ARG;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define CALL(W, G)                                                                                                    \
  return run<W, G>(crf_wide_bwd_kernel<W, G>, bwd_smem_bytes<W, G>(K), B, st, logits, tags, seq_len, trans, alpha_ws, \
                   logz, d_ll, scale, d_logits, d_trans, B, L, K)
  NER_WIDE_DISPATCH(ner_crf_wide_plan(B, L, K, ner_num_sms()), CALL)
#undef CALL
  return NER_ERR_UNSUPPORTED;
}
