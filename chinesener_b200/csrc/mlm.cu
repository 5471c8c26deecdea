// Masked-LM pretraining kernels (sm_90a): dynamic whole-word masking (ner_mlm_mask) and the vocabulary-wide cross-entropy of
// the masked positions with its gradient and argmax (ner_vocab_xent).  Definitions in ner_b200.h.
//
// ner_mlm_mask: one CTA of 512 threads per row, one thread per position (L <= 512).  Word starts are numbered by a block
// scan, the words are sorted by (hash key, first position) with a bitonic sort in shared memory, and one thread walks them
// in that order taking every word that still fits the row's budget (google-research/bert create_pretraining_data.py,
// create_masked_lm_predictions).  A second scan orders the chosen positions.
//
// ner_vocab_xent: HBM-bound.  One CTA per row stages the row's V logits in shared memory (84.5 KB at V = 21 128) with
// 16-byte streaming loads, keeping each thread's first maximum on the way; the sum of exponentials and the bf16 gradient
// then work from shared memory, so every logit is read from HBM once and every gradient element written once.  Per-row
// losses go to the scratch and a one-CTA finaliser adds them in index order: identical inputs give a bit-identical loss.
#include <cmath>

#include "common.cuh"

namespace {

using namespace nerdev;

constexpr int kMaskThreads = 512;     // = the largest L
constexpr int kXentThreads = 512;
constexpr int kScratchHead = 16;      // scratch[0] = d_loss / count, scratch[1] = count (int bits); rows from kScratchHead

// Stream k of the masking hash at (row b, position t).  k = 0: word keys, 1: the 80 / 10 / 10 draw, 2: the random id.
__device__ __forceinline__ uint32_t mask_hash(uint64_t seed, uint32_t k, int b, int t) {
  return hash3((uint32_t)seed + k * 0x9E3779B9u, (uint32_t)(seed >> 32) ^ (uint32_t)b, (uint32_t)t);
}

// Exclusive prefix sum of v over the CTA (kMaskThreads threads); *total = the sum.  Ends with a barrier.
__device__ __forceinline__ int block_excl_scan(int v, int* warp_tot, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_tot[w] = x;
  __syncthreads();
  int before = 0, all = 0;
  for (int i = 0; i < kMaskThreads / 32; ++i) {
    const int s = warp_tot[i];
    before += i < w ? s : 0;
    all += s;
  }
  *total = all;
  __syncthreads();
  return before + x - v;
}

__global__ void __launch_bounds__(kMaskThreads)
mlm_mask_kernel(const int32_t* __restrict__ token_ids, const int32_t* __restrict__ seq_len,
                const uint8_t* __restrict__ word_start, const int32_t* __restrict__ pred_offsets, int L, uint64_t seed, int V,
                int mask_id, int32_t* __restrict__ masked_ids, int32_t* __restrict__ positions,
                int32_t* __restrict__ labels) {
  __shared__ uint64_t keys[kMaskThreads];       // (key << 32 | first position) of each word, then sorted
  __shared__ int16_t wstart[kMaskThreads];      // first position of word w
  __shared__ int16_t wlen_at[kMaskThreads];     // length of the word starting at position t
  __shared__ uint8_t chosen_at[kMaskThreads];   // 1 at the first position of every chosen word
  __shared__ int warp_tot[kMaskThreads / 32];
  const int b = blockIdx.x, t = threadIdx.x;
  const int n = min(max(__ldg(seq_len + b), 0), L);
  const int off = __ldg(pred_offsets + b);
  const int k = max(__ldg(pred_offsets + b + 1) - off, 0);
  const bool cand = t >= 1 && t <= n - 2;
  const bool start = cand && (t == 1 || word_start == nullptr || word_start[(size_t)b * L + t] != 0);
  chosen_at[t] = 0;
  int nw;
  const int wid = block_excl_scan(start ? 1 : 0, warp_tot, &nw);   // word index of a start; words before t otherwise
  if (start) {
    wstart[wid] = (int16_t)t;
    keys[wid] = (uint64_t)mask_hash(seed, 0, b, t) << 32 | (uint32_t)t;
  }
  int P = 1;
  while (P < nw) P <<= 1;
  if (t >= nw && t < P) keys[t] = ~0ull;
  __syncthreads();
  const int my_word = cand ? (start ? wid : wid - 1) : -1;
  if (start) wlen_at[t] = (int16_t)((wid + 1 < nw ? wstart[wid + 1] : n - 1) - t);
  __syncthreads();
  // bitonic sort of keys[0, P) (P <= 512 = one element per thread)
  for (int size = 2; size <= P; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      const int j = t ^ stride;
      if (t < P && j > t) {
        const uint64_t a = keys[t], c = keys[j];
        if ((a > c) == ((t & size) == 0)) {
          keys[t] = c;
          keys[j] = a;
        }
      }
      __syncthreads();
    }
  }
  if (t == 0) {           // the greedy walk: a word that no longer fits is skipped, later (shorter) words may still fit
    int taken = 0;
    for (int i = 0; i < nw && taken < k; ++i) {
      const int s = (int)(uint32_t)keys[i];
      const int len = wlen_at[s];
      if (taken + len <= k) {
        taken += len;
        chosen_at[s] = 1;
      }
    }
  }
  __syncthreads();
  const bool sel = my_word >= 0 && chosen_at[wstart[my_word]];
  int taken;
  const int idx = block_excl_scan(sel ? 1 : 0, warp_tot, &taken);
  if (t < L) {
    const size_t at = (size_t)b * L + t;
    const int tok = __ldg(token_ids + at);
    int out = tok;
    if (sel) {
      const uint32_t u = mask_hash(seed, 1, b, t) >> 8;            // u / 2^24 in [0, 1)
      if (u * 5u < (4u << 24)) out = mask_id;                      // u < 0.8
      else if (u * 10u < (9u << 24)) out = (int)__umulhi(mask_hash(seed, 2, b, t), (uint32_t)V);   // u < 0.9
      positions[off + idx] = b * L + t;
      labels[off + idx] = tok;
    }
    masked_ids[at] = out;
  }
  for (int i = taken + t; i < k; i += kMaskThreads) {
    positions[off + i] = b * L;
    labels[off + i] = -1;
  }
}

// count = #labels in [0, V); scratch[0] = d_loss / count (0 when count = 0).
__global__ void __launch_bounds__(1024)
vocab_count_kernel(const int32_t* __restrict__ labels, int M, int V, float d_loss, float* __restrict__ scratch) {
  int acc = 0;
  for (int r = threadIdx.x; r < M; r += blockDim.x) {
    const int y = __ldg(labels + r);
    acc += (y >= 0 && y < V) ? 1 : 0;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ int part[32];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    int n = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) n += part[w];
    reinterpret_cast<int*>(scratch)[1] = n;
    scratch[0] = n > 0 ? (float)((double)d_loss / (double)n) : 0.f;
  }
}

__device__ __forceinline__ void take_first_max(float& m, int& a, float om, int oa) {
  if (om > m || (om == m && oa < a)) {
    m = om;
    a = oa;
  }
}

// Sum over the CTA in a fixed order (butterfly in each warp, then the warps in index order); every thread gets the sum.
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  for (int w = 0; w < kXentThreads / 32; ++w) s += red[w];
  return s;
}

__device__ __forceinline__ uint2 pack_bf16x4(float a, float b, float c, float d) {
  __nv_bfloat162 lo = __floats2bfloat162_rn(a, b), hi = __floats2bfloat162_rn(c, d);
  return make_uint2(*reinterpret_cast<uint32_t*>(&lo), *reinterpret_cast<uint32_t*>(&hi));
}

template <bool GRAD>
__global__ void __launch_bounds__(kXentThreads)
vocab_xent_kernel(const float* __restrict__ logits, int ld, const int32_t* __restrict__ labels, int M, int V,
                  int32_t* __restrict__ pred, __nv_bfloat16* __restrict__ d_logits, float* __restrict__ scratch) {
  extern __shared__ float4 z4[];
  float* z = reinterpret_cast<float*>(z4);
  __shared__ float red_m[kXentThreads / 32];
  __shared__ int red_a[kXentThreads / 32];
  __shared__ float red_s[kXentThreads / 32];
  const int r = blockIdx.x, tid = threadIdx.x;
  const float4* src = reinterpret_cast<const float4*>(logits + (size_t)r * ld);
  const int nv4 = (V + 3) >> 2;
  float m = -INFINITY;
  int arg = 0x7fffffff;
  constexpr int U = 4;                  // float4 loads in flight per thread
  for (int i0 = tid; i0 < nv4; i0 += U * kXentThreads) {
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * kXentThreads;
      if (i < nv4) v[u] = __ldcs(src + i);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * kXentThreads;
      if (i < nv4) {
        z4[i] = v[u];
        const float e[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (4 * i + c < V && e[c] > m) {            // strict: this thread's first maximum (its indices ascend)
            m = e[c];
            arg = 4 * i + c;
          }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) take_first_max(m, arg, __shfl_xor_sync(0xffffffffu, m, o),
                                                  __shfl_xor_sync(0xffffffffu, arg, o));
  if ((tid & 31) == 0) {
    red_m[tid >> 5] = m;
    red_a[tid >> 5] = arg;
  }
  __syncthreads();
  m = red_m[0];
  arg = red_a[0];
  for (int w = 1; w < kXentThreads / 32; ++w) take_first_max(m, arg, red_m[w], red_a[w]);
  if (arg == 0x7fffffff) arg = 0;        // no element above -inf (all -inf or NaN): index 0, as np.argmax of -inf rows
  const int y = __ldg(labels + r);
  const bool counted = y >= 0 && y < V;
  float s = 0.f, zy = 0.f;
  if (counted) {                          // block-uniform
    if (tid == 0) zy = __ldg(logits + (size_t)r * ld + y);     // not z[y]: the pass below overwrites z with e
    float acc = 0.f;
    for (int j = tid; j < V; j += kXentThreads) {
      const float e = expf(z[j] - m);
      acc += e;
      if (GRAD) z[j] = e;
    }
    s = block_sum(acc, red_s);
  }
  if (GRAD) {
    const float scale = scratch[0];
    const float inv = counted ? scale / s : 0.f;
    const int yy = counted ? y : -1;
    uint2* dst = reinterpret_cast<uint2*>(d_logits + (size_t)r * ld);
    for (int i = tid; i < (ld >> 2); i += kXentThreads) {
      float g[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int j = 4 * i + c;
        g[c] = (counted && j < V) ? z[j] * inv - (j == yy ? scale : 0.f) : 0.f;
      }
      __stcs(dst + i, pack_bf16x4(g[0], g[1], g[2], g[3]));
    }
  }
  if (tid == 0) {
    if (pred != nullptr) pred[r] = arg;
    scratch[kScratchHead + r] = counted ? (m - zy) + logf(s) : 0.f;
    reinterpret_cast<int*>(scratch)[kScratchHead + M + r] = counted && arg == y ? 1 : 0;
  }
}

// loss = (row losses summed in index order) / count, 0 when count = 0; count and correct.
__global__ void __launch_bounds__(256)
vocab_final_kernel(const float* __restrict__ scratch, int M, float* __restrict__ loss, int32_t* __restrict__ count,
                   int32_t* __restrict__ correct) {
  __shared__ double part[256];
  __shared__ int cpart[256];
  double acc = 0.0;
  int c = 0;
  const int* rc = reinterpret_cast<const int*>(scratch) + kScratchHead + M;
  for (int i = threadIdx.x; i < M; i += 256) {
    acc += (double)scratch[kScratchHead + i];
    c += rc[i];
  }
  part[threadIdx.x] = acc;
  cpart[threadIdx.x] = c;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      part[threadIdx.x] += part[threadIdx.x + o];
      cpart[threadIdx.x] += cpart[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const int n = reinterpret_cast<const int*>(scratch)[1];
    loss[0] = n > 0 ? (float)(part[0] / (double)n) : 0.f;
    count[0] = n;
    correct[0] = cpart[0];
  }
}

}  // namespace

extern "C" int ner_mlm_mask(const int32_t* token_ids, const int32_t* seq_len, const uint8_t* word_start,
                            const int32_t* pred_offsets, int B, int L, uint64_t seed, int V, int mask_id,
                            int32_t* masked_ids, int32_t* positions, int32_t* labels, ner_stream_t stream) {
  if (B < 0 || L < 1 || V < 1) return NER_ERR_INVALID_ARG;
  if (L > NER_MLM_MAX_LEN || V > NER_MLM_MAX_VOCAB) return NER_ERR_UNSUPPORTED;
  if (mask_id < 0 || mask_id >= V) return NER_ERR_INVALID_ARG;
  if ((long long)B * L > 0x7fffffffLL) return NER_ERR_UNSUPPORTED;
  if (B == 0) return NER_OK;
  if (!token_ids || !seq_len || !pred_offsets || !masked_ids || !positions || !labels) return NER_ERR_INVALID_ARG;
  mlm_mask_kernel<<<B, kMaskThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      token_ids, seq_len, word_start, pred_offsets, L, seed, V, mask_id, masked_ids, positions, labels);
  return ner_launch_status();
}

extern "C" size_t ner_vocab_xent_scratch_floats(int M) { return (size_t)kScratchHead + 2 * (size_t)(M > 0 ? M : 0); }

extern "C" int ner_vocab_xent(const float* logits, int ld, const int32_t* labels, int M, int V, float d_loss, float* loss,
                              int32_t* count, int32_t* correct, int32_t* pred, void* d_logits, float* scratch,
                              ner_stream_t stream) {
  if (M < 0 || V < 1 || ld < V) return NER_ERR_INVALID_ARG;
  if (V > NER_MLM_MAX_VOCAB) return NER_ERR_UNSUPPORTED;
  if (ld % 4 != 0) return NER_ERR_INVALID_ARG;
  if (M == 0) return NER_OK;
  if (!logits || !labels || !loss || !count || !correct || !scratch) return NER_ERR_INVALID_ARG;
  if (reinterpret_cast<uintptr_t>(logits) % 16 || reinterpret_cast<uintptr_t>(d_logits) % 8) return NER_ERR_INVALID_ARG;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t smem = (size_t)((V + 3) / 4) * sizeof(float4);
  vocab_count_kernel<<<1, 1024, 0, st>>>(labels, M, V, d_loss, scratch);
  if (d_logits != nullptr) {
    cudaFuncSetAttribute(vocab_xent_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    vocab_xent_kernel<true><<<M, kXentThreads, smem, st>>>(logits, ld, labels, M, V, pred,
                                                           static_cast<__nv_bfloat16*>(d_logits), scratch);
  } else {
    cudaFuncSetAttribute(vocab_xent_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    vocab_xent_kernel<false><<<M, kXentThreads, smem, st>>>(logits, ld, labels, M, V, pred, nullptr, scratch);
  }
  vocab_final_kernel<<<1, 256, 0, st>>>(scratch, M, loss, count, correct);
  return ner_launch_status();
}
