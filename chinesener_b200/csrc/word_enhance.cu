// Small-table word-enhance embeddings (sm_90a): the ExSoftword multi-hot projection and a deterministic gradient for
// the trainable [V <= 8, E <= 128] tables of the Softword / ExSoftword plugins (model/bilstm_crf_softword.py,
// model/bilstm_crf_ex_softword.py).
//
//   ner_multihot_embed_fwd:  out[t, 0:E] = sum_v weights[t, v] * table[v, :]     (v ascending, zero weights skipped)
//   ner_small_table_grad:    d_table[v, :] += sum_t c(t, v) * d_out[t, :]         c one-hot (ids) or multi-hot (weights)
//
// The gradient lands on at most 8 * 128 addresses, so a float-atomic scatter (ner_softlexicon_pool_bwd) serialises on
// them and sums in arrival order.  Here every CTA owns a fixed token range and writes one [V, E] partial; a second kernel
// adds the partials in CTA order.  The grid is a function of n_tok and the SM count only, so one device gives a
// bit-identical gradient on every call (the scheme of sumsq_partial_kernel / sumsq_final_kernel in train_ops.cu).
#include "common.cuh"

namespace {

using namespace nerdev;

constexpr int kMaxV = 8;
constexpr int kMaxE = 128;
constexpr int kThreads = 256;
constexpr int kGradCtasPerSm = 4;    // 4 x 256 threads x 4 loads in flight per SM: enough bytes in flight for HBM
constexpr int kGradMinTokPerCta = 64;
constexpr int kGradUnroll = 4;

int grad_grid(int n_tok) {
  long g = ((long)n_tok + kGradMinTokPerCta - 1) / kGradMinTokPerCta;
  const long cap = (long)ner_num_sms() * kGradCtasPerSm;
  return (int)(g < cap ? g : cap);
}

// One thread per output element (t, e); the table sits in shared memory.  (t, e) advance by the grid stride without a
// 64-bit division per element.
__global__ void __launch_bounds__(kThreads)
multihot_embed_fwd_kernel(const float* __restrict__ table, const float* __restrict__ weights, float* __restrict__ out,
                          int n_tok, int V, int E, int ld_out) {
  __shared__ float tab[kMaxV * kMaxE];
  for (int i = threadIdx.x; i < V * E; i += kThreads) tab[i] = table[i];
  __syncthreads();
  const size_t i0 = (size_t)blockIdx.x * kThreads + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * kThreads;
  size_t t = i0 / E;
  int e = (int)(i0 - t * E);
  const size_t st = stride / E;
  const int se = (int)(stride - st * E);
  while (t < (size_t)n_tok) {
    const float* w = weights + t * V;
    float acc = 0.f;
#pragma unroll
    for (int v = 0; v < kMaxV; ++v) {
      if (v < V) {
        const float c = __ldg(w + v);
        if (c != 0.f) acc = fmaf(c, tab[v * E + e], acc);
      }
    }
    out[t * ld_out + e] = acc;
    t += st;
    e += se;
    if (e >= E) {
      e -= E;
      ++t;
    }
  }
}

// Coefficients c(t, 0:kMaxV) of one token: one-hot of the clamped id, or its weight row (zero past V).
__device__ __forceinline__ void load_coef(float (&c)[kMaxV], const int32_t* __restrict__ ids,
                                          const float* __restrict__ weights, long t, int V) {
  if (ids) {
    const int id = min(max(__ldg(ids + t), 0), V - 1);
#pragma unroll
    for (int v = 0; v < kMaxV; ++v) c[v] = (v == id) ? 1.f : 0.f;
  } else {
#pragma unroll
    for (int v = 0; v < kMaxV; ++v) c[v] = (v < V) ? __ldg(weights + (size_t)t * V + v) : 0.f;
  }
}

// acc[v] += c[v] * d for the non-zero coefficients (fmaf(1, d, acc) == acc + d: the one-hot sum is exact per add).
__device__ __forceinline__ void grad_accum(float (&acc)[kMaxV], const float (&c)[kMaxV], float d) {
#pragma unroll
  for (int v = 0; v < kMaxV; ++v)
    if (c[v] != 0.f) acc[v] = fmaf(c[v], d, acc[v]);
}

// CTA b owns tokens [b * chunk, min((b + 1) * chunk, n_tok)).  Thread (r, e) = (tid / E, tid % E) sums column e of the
// tokens b * chunk + r + k * R (R = 256 / E rows) in token order; the R row sums are added in row order and the CTA's
// [V, E] partial goes to partials[b].  Fixed maps and orders throughout: no float atomics.
__global__ void __launch_bounds__(kThreads, kGradCtasPerSm)
small_table_grad_partial_kernel(const int32_t* __restrict__ ids, const float* __restrict__ weights,
                                const float* __restrict__ d_out, int n_tok, int V, int E, int ld_dout,
                                float* __restrict__ partials) {
  __shared__ float red[kThreads * kMaxV];     // [R][V * E], R * E <= 256
  const int R = kThreads / E;
  const int r = threadIdx.x / E;
  const int e = threadIdx.x - r * E;
  const int VE = V * E;
  const long chunk = ((long)n_tok + gridDim.x - 1) / gridDim.x;
  const long t0 = (long)blockIdx.x * chunk;
  const long t1 = min(t0 + chunk, (long)n_tok);
  float acc[kMaxV];
#pragma unroll
  for (int v = 0; v < kMaxV; ++v) acc[v] = 0.f;
  if (r < R) {
    long t = t0 + r;
    // kGradUnroll tokens per trip: their loads are issued together, then accumulated in token order
    for (; t + (kGradUnroll - 1) * (long)R < t1; t += kGradUnroll * (long)R) {
      float d[kGradUnroll];
      float c[kGradUnroll][kMaxV];
#pragma unroll
      for (int k = 0; k < kGradUnroll; ++k) {
        const long tk = t + k * (long)R;
        d[k] = __ldg(d_out + (size_t)tk * ld_dout + e);
        load_coef(c[k], ids, weights, tk, V);
      }
#pragma unroll
      for (int k = 0; k < kGradUnroll; ++k) grad_accum(acc, c[k], d[k]);
    }
    for (; t < t1; t += R) {
      float c[kMaxV];
      load_coef(c, ids, weights, t, V);
      grad_accum(acc, c, __ldg(d_out + (size_t)t * ld_dout + e));
    }
#pragma unroll
    for (int v = 0; v < kMaxV; ++v)
      if (v < V) red[r * VE + v * E + e] = acc[v];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < VE; i += kThreads) {
    float s = 0.f;
    for (int q = 0; q < R; ++q) s += red[q * VE + i];
    partials[(size_t)blockIdx.x * VE + i] = s;
  }
}

// One warp per table element i: lane l sums partials l, l + 32, ... in order, then a fixed shuffle tree; the result is
// added into d_table[i].
__global__ void __launch_bounds__(kThreads)
small_table_grad_final_kernel(const float* __restrict__ partials, int n_part, int VE, float* __restrict__ d_table) {
  const int i = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= VE) return;
  float s = 0.f;
  for (int b = lane; b < n_part; b += 32) s += partials[(size_t)b * VE + i];
  s = warp_sum(s);
  if (lane == 0) d_table[i] += s;
}

}  // namespace

extern "C" int ner_multihot_embed_fwd(const float* table, const float* weights, float* out, int n_tok, int V, int E,
                                      int ld_out, ner_stream_t stream) {
  if (n_tok < 0 || V < 1 || E < 1 || ld_out < E) return NER_ERR_INVALID_ARG;
  if (V > kMaxV || E > kMaxE) return NER_ERR_UNSUPPORTED;
  if (n_tok == 0) return NER_OK;
  if (!table || !weights || !out) return NER_ERR_INVALID_ARG;
  long grid = (long)(((size_t)n_tok * E + kThreads - 1) / kThreads);
  if (grid > (long)ner_num_sms() * 8) grid = (long)ner_num_sms() * 8;
  multihot_embed_fwd_kernel<<<(int)grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(table, weights, out, n_tok, V,
                                                                                           E, ld_out);
  return ner_launch_status();
}

extern "C" size_t ner_small_table_grad_scratch_floats(int V, int E) {
  if (V < 1 || E < 1 || V > kMaxV || E > kMaxE) return 0;
  return (size_t)ner_num_sms() * kGradCtasPerSm * V * E;
}

extern "C" int ner_small_table_grad(float* d_table, const int32_t* ids, const float* weights, const float* d_out,
                                    int n_tok, int V, int E, int ld_dout, float* scratch, ner_stream_t stream) {
  if (n_tok < 0 || V < 1 || E < 1 || ld_dout < E) return NER_ERR_INVALID_ARG;
  if (V > kMaxV || E > kMaxE) return NER_ERR_UNSUPPORTED;
  if (ids && weights) return NER_ERR_INVALID_ARG;
  if (n_tok == 0) return NER_OK;
  if (!ids && !weights) return NER_ERR_INVALID_ARG;
  if (!d_table || !d_out || !scratch) return NER_ERR_INVALID_ARG;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int grid = grad_grid(n_tok);
  small_table_grad_partial_kernel<<<grid, kThreads, 0, st>>>(ids, weights, d_out, n_tok, V, E, ld_dout, scratch);
  const int VE = V * E;
  small_table_grad_final_kernel<<<(VE + kThreads / 32 - 1) / (kThreads / 32), kThreads, 0, st>>>(scratch, grid, VE,
                                                                                               d_table);
  return ner_launch_status();
}
