// Training-data augmentation kernels (sm_90a): mention replacement, label-wise token replacement, shuffle within segments
// and the [MASK]ing of masked-LM replacement on a device batch (ner_augment_rows), and the Gumbel-max draw of the
// replacement ids from the masked-LM logits (ner_vocab_sample).  The rules are stated in ner_b200.h; chinesener_b200/
// augment.py drives both and tests/_augment_oracle.py restates them.
//
// ner_augment_rows: one CTA of 256 threads per row, the row in dynamic shared memory (16 L + 8 P bytes, P = the power of
// two >= L).  The two passes whose outcome depends on everything to their left (mention replacement with its running
// length, and the segmentation of the shuffled row) are one thread's walks over shared memory; token replacement, the
// sort of the shuffle keys (bitonic, as ner_mlm_mask sorts its words), the [MASK] choice and the stores are CTA-wide.
//
// ner_vocab_sample: HBM-bound like ner_vocab_xent.  One CTA per slot streams the row's logits once with 16-byte loads;
// a thread computes a Gumbel draw only when the logit could still beat its running best (every draw is < kGumbelMax).
#include <cmath>

#include "common.cuh"

namespace {

using namespace nerdev;

constexpr int kRowThreads = 256;
constexpr int kSampleThreads = 512;
constexpr float kGumbelMax = 17.f;    // > -log(-log(1 - 2^-24)) = 16.64, the largest draw

// hash streams (the k of aug_hash)
enum : uint32_t { kRow = 0, kMrPick, kMrDraw, kLwPick, kLwDraw, kSisPick, kSisKey, kMlmPick, kGumbel };

__device__ __forceinline__ uint32_t aug_hash(uint64_t seed, uint32_t k, uint32_t b, uint32_t t) {
  return hash3((uint32_t)seed + k * 0x9E3779B9u, (uint32_t)(seed >> 32) ^ b, t);
}
__host__ __device__ inline uint32_t threshold(float p) { return (uint32_t)(p * 16777216.f); }   // p * 2^24, exact
__device__ __forceinline__ bool drawn(uint32_t h, uint32_t thr) { return (h >> 8) < thr; }
__device__ __forceinline__ int pick(uint32_t h, int n) { return (int)__umulhi(h, (uint32_t)n); }

struct RowArgs {
  const int32_t *token_ids, *label_ids, *seq_len, *mask, *segment_ids;
  int B, L, K, T;
  const int32_t *tag_class, *type_tag;
  const int32_t *mention_type_off, *mention_tok_off, *mention_tokens;
  int n_mentions, n_mention_tokens;
  const int32_t *tag_tok_off, *tag_tokens;
  int n_tag_tokens;
  uint32_t thr_row, thr_mr, thr_lwtr, thr_sis, thr_mlm;
  uint64_t seed;
  int pad_id, pad_tag, mask_id;
  int32_t *token_out, *label_out, *seq_len_out, *mask_out, *segment_out, *mlm_ids, *mlm_positions;
};

// [lo, hi) of entry i of an offsets array with n_off + 1 entries into a pool of `size` elements; empty when malformed
__device__ __forceinline__ int2 csr_range(const int32_t* off, int i, int size) {
  const int lo = __ldg(off + i), hi = __ldg(off + i + 1);
  return (lo < 0 || hi < lo || hi > size) ? make_int2(0, 0) : make_int2(lo, hi);
}

// Exclusive prefix sum of v over the CTA; *total = the sum.  Ends with a barrier.
__device__ __forceinline__ int row_excl_scan(int v, int* warp_tot, int* total) {
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
  for (int i = 0; i < kRowThreads / 32; ++i) {
    const int s = warp_tot[i];
    before += i < w ? s : 0;
    all += s;
  }
  *total = all;
  __syncthreads();
  return before + x - v;
}

__global__ void __launch_bounds__(kRowThreads) augment_rows_kernel(const RowArgs a) {
  extern __shared__ int4 smem4[];
  const int L = a.L, b = blockIdx.x, tid = threadIdx.x;
  int32_t* in_tok = reinterpret_cast<int32_t*>(smem4);   // the input row; later the segment starts, then scratch
  int32_t* in_tag = in_tok + L;                          // the input tags; later per-position flags
  int32_t* tok = in_tag + L;                             // the row being built
  int32_t* tag = tok + L;
  uint64_t* keys = reinterpret_cast<uint64_t*>(tag + L);           // byte offset 16 L: 8-byte aligned
  __shared__ int32_t cls_of[NER_MAX_TAGS_WIDE];
  __shared__ int s_n, s_shuffle;
  __shared__ int warp_tot[kRowThreads / 32];
  const size_t base = (size_t)b * L;
  const bool mlm = a.mlm_ids != nullptr;
  if (!drawn(aug_hash(a.seed, kRow, b, 0), a.thr_row)) {          // not chosen: the row passes through byte for byte
    for (int t = tid; t < L; t += kRowThreads) {
      const int x = __ldg(a.token_ids + base + t);
      a.token_out[base + t] = x;
      a.label_out[base + t] = __ldg(a.label_ids + base + t);
      a.mask_out[base + t] = __ldg(a.mask + base + t);
      a.segment_out[base + t] = __ldg(a.segment_ids + base + t);
      if (mlm) a.mlm_ids[base + t] = x;
    }
    if (mlm && tid < NER_AUGMENT_MLM_BUDGET) a.mlm_positions[b * NER_AUGMENT_MLM_BUDGET + tid] = -1;
    if (tid == 0) a.seq_len_out[b] = __ldg(a.seq_len + b);
    return;
  }
  const int n0 = min(max(__ldg(a.seq_len + b), 0), L);
  for (int k = tid; k < a.K; k += kRowThreads) cls_of[k] = __ldg(a.tag_class + k);
  for (int t = tid; t < n0; t += kRowThreads) {
    in_tok[t] = __ldg(a.token_ids + base + t);
    in_tag[t] = __ldg(a.label_ids + base + t);
  }
  __syncthreads();
  auto cls = [&](int y) { return (y >= 0 && y < a.K) ? cls_of[y] : 0; };
  auto tag_id = [&](int x, int inside) { return __ldg(a.type_tag + 2 * x + inside); };

  // mention replacement: mentions left to right, a replacement kept only while the row stays within L
  if (a.thr_mr == 0) {
    for (int t = tid; t < n0; t += kRowThreads) {
      tok[t] = in_tok[t];
      tag[t] = in_tag[t];
    }
    if (tid == 0) s_n = n0;
  } else if (tid == 0) {
    int m = 0, cur = n0;
    for (int s = 0; s < n0;) {
      const int y = in_tag[s], c = cls(y);
      if (c < 2 || (c & 1)) {
        tok[m] = in_tok[s];
        tag[m++] = y;
        ++s;
        continue;
      }
      const int x = (c - 2) >> 1, inside = tag_id(x, 1);
      int e = s;
      while (e + 1 < n0 && in_tag[e + 1] == inside) ++e;         // span::run_end
      const int len = e - s + 1;
      bool replaced = false;
      if (drawn(aug_hash(a.seed, kMrPick, b, s), a.thr_mr)) {
        const int2 r = csr_range(a.mention_type_off, x, a.n_mentions);
        if (r.y > r.x) {
          const int j = r.x + pick(aug_hash(a.seed, kMrDraw, b, s), r.y - r.x);
          const int2 q = csr_range(a.mention_tok_off, j, a.n_mention_tokens);
          const int nl = q.y - q.x;
          if (nl >= 1 && (nl == 1 || inside >= 0) && cur - len + nl <= L) {
            for (int i = 0; i < nl; ++i) {
              tok[m + i] = __ldg(a.mention_tokens + q.x + i);
              tag[m + i] = i == 0 ? y : inside;
            }
            m += nl;
            cur += nl - len;
            replaced = true;
          }
        }
      }
      if (!replaced)
        for (int i = s; i <= e; ++i) {
          tok[m] = in_tok[i];
          tag[m++] = in_tag[i];
        }
      s = e + 1;
    }
    s_n = m;
  }
  __syncthreads();
  const int n = s_n;

  // label-wise token replacement
  if (a.thr_lwtr != 0)
    for (int t = tid; t < n; t += kRowThreads) {
      const int y = tag[t];
      if (cls(y) >= 1 && drawn(aug_hash(a.seed, kLwPick, b, t), a.thr_lwtr)) {
        const int2 r = csr_range(a.tag_tok_off, y, a.n_tag_tokens);
        if (r.y > r.x) tok[t] = __ldg(a.tag_tokens + r.x + pick(aug_hash(a.seed, kLwDraw, b, t), r.y - r.x));
      }
    }

  // shuffle within segments: in_tok[t] = first position of t's segment, in_tag[s] = 1 where segment s is shuffled
  if (a.thr_sis != 0) {
    __syncthreads();
    if (tid == 0) {
      int st = 0, mention = -1, prev = -1, any = 0;
      for (int t = 0; t <= n; ++t) {
        bool cont = false;
        int c = 0, x = -1;
        if (t < n) {
          c = cls(tag[t]);
          x = c >= 2 ? (c - 2) >> 1 : -1;
          cont = t > 0 && ((c == 1 && prev == 1) || (c >= 2 && (c & 1) && mention == x));
        }
        if (!cont) {
          if (t > 0) {                                    // close the segment [st, t)
            const bool sh = t - st >= 2 && drawn(aug_hash(a.seed, kSisPick, b, st), a.thr_sis);
            in_tag[st] = sh ? 1 : 0;
            any |= sh;
          }
          st = t;
        }
        if (t < n) {
          in_tok[t] = st;
          mention = (c >= 2 && (!(c & 1) || cont)) ? x : -1;
          prev = c;
        }
      }
      s_shuffle = any;
    }
    __syncthreads();
    if (s_shuffle) {
      int P = 1;
      while (P < n) P <<= 1;
      for (int t = tid; t < P; t += kRowThreads) {
        if (t < n) {
          const int st = in_tok[t];
          const uint32_t h = in_tag[st] ? aug_hash(a.seed, kSisKey, b, t) : 0u;
          keys[t] = (uint64_t)st << 44 | (uint64_t)h << 12 | (uint32_t)t;
        } else {
          keys[t] = ~0ull;
        }
      }
      __syncthreads();
      for (int size = 2; size <= P; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
          for (int i = tid; i < P; i += kRowThreads) {
            const int j = i ^ stride;
            if (j > i) {
              const uint64_t u = keys[i], v = keys[j];
              if ((u > v) == ((i & size) == 0)) {
                keys[i] = v;
                keys[j] = u;
              }
            }
          }
          __syncthreads();
        }
      for (int t = tid; t < n; t += kRowThreads) in_tok[t] = tok[(int)(keys[t] & 0xFFF)];
      __syncthreads();
      for (int t = tid; t < n; t += kRowThreads) tok[t] = in_tok[t];
    }
  }
  __syncthreads();

  // masked-LM replacement: O tokens drawn with p, the first NER_AUGMENT_MLM_BUDGET of them in position order
  if (mlm) {
    int carried = 0;
    for (int t0 = 0; t0 < n; t0 += kRowThreads) {
      const int t = t0 + tid;
      const bool f = t < n && a.thr_mlm != 0 && cls(tag[t]) == 1 && drawn(aug_hash(a.seed, kMlmPick, b, t), a.thr_mlm);
      int tot;
      const int rank = carried + row_excl_scan(f ? 1 : 0, warp_tot, &tot);
      const bool take = f && rank < NER_AUGMENT_MLM_BUDGET;
      if (t < n) in_tag[t] = take ? 1 : 0;
      if (take) a.mlm_positions[b * NER_AUGMENT_MLM_BUDGET + rank] = (int)(base + t);
      carried += tot;
    }
    for (int i = min(carried, NER_AUGMENT_MLM_BUDGET) + tid; i < NER_AUGMENT_MLM_BUDGET; i += kRowThreads)
      a.mlm_positions[b * NER_AUGMENT_MLM_BUDGET + i] = -1;
    __syncthreads();
  }
  for (int t = tid; t < L; t += kRowThreads) {
    const bool in = t < n;
    const int x = in ? tok[t] : a.pad_id;
    a.token_out[base + t] = x;
    a.label_out[base + t] = in ? tag[t] : a.pad_tag;
    a.mask_out[base + t] = in ? 1 : 0;
    a.segment_out[base + t] = 0;
    if (mlm) a.mlm_ids[base + t] = (in && in_tag[t]) ? a.mask_id : x;
  }
  if (tid == 0) a.seq_len_out[b] = n;
}

__device__ __forceinline__ void take_first_max(float& m, int& a, float om, int oa) {
  if (om > m || (om == m && oa < a)) {
    m = om;
    a = oa;
  }
}

__global__ void __launch_bounds__(kSampleThreads)
vocab_sample_kernel(const float* __restrict__ logits, int ld, int V, const uint8_t* __restrict__ eligible,
                    const int32_t* __restrict__ positions, long long n_tokens, float inv_temp, uint64_t seed,
                    int32_t* __restrict__ token_ids) {
  __shared__ float red_m[kSampleThreads / 32];
  __shared__ int red_a[kSampleThreads / 32];
  const int r = blockIdx.x, tid = threadIdx.x;
  const int pos = __ldg(positions + r);
  if (pos < 0 || pos >= n_tokens) return;                  // block-uniform
  const int orig = token_ids[pos];
  const float4* src = reinterpret_cast<const float4*>(logits + (size_t)r * ld);
  const int nv4 = (V + 3) >> 2;
  float m = -INFINITY;
  int arg = 0x7fffffff;
  constexpr int U = 4;
  for (int i0 = tid; i0 < nv4; i0 += U * kSampleThreads) {
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * kSampleThreads;
      if (i < nv4) v[u] = __ldcs(src + i);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * kSampleThreads;
      if (i >= nv4) continue;
      const float e[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int j = 4 * i + c;
        if (j >= V || j == orig || !__ldg(eligible + j)) continue;
        const float s0 = e[c] * inv_temp;
        if (!(s0 + kGumbelMax > m)) continue;              // cannot win (or NaN)
        const float uu = ((float)(aug_hash(seed, kGumbel, (uint32_t)pos, (uint32_t)j) >> 9) + 0.5f) * 0x1p-23f;
        const float s = s0 - logf(-logf(uu));
        if (s > m) {                                      // strict: this thread's indices ascend
          m = s;
          arg = j;
        }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    take_first_max(m, arg, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, arg, o));
  if ((tid & 31) == 0) {
    red_m[tid >> 5] = m;
    red_a[tid >> 5] = arg;
  }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < kSampleThreads / 32; ++w) take_first_max(m, arg, red_m[w], red_a[w]);
    if (arg != 0x7fffffff) token_ids[pos] = arg;           // no eligible id: the token stays
  }
}

bool prob_ok(float p) { return p >= 0.f && p <= 1.f; }   // false for NaN

}  // namespace

extern "C" size_t ner_augment_rows_smem_bytes(int L) {
  if (L < 1 || L > NER_AUGMENT_MAX_LEN) return 0;
  int P = 1;
  while (P < L) P <<= 1;
  return (size_t)4 * L * sizeof(int32_t) + (size_t)P * sizeof(uint64_t);
}

extern "C" int ner_augment_rows(const int32_t* token_ids, const int32_t* label_ids, const int32_t* seq_len,
                                const int32_t* mask, const int32_t* segment_ids, int B, int L, const int32_t* tag_class,
                                int K, const int32_t* type_tag, int T, const int32_t* mention_type_off,
                                const int32_t* mention_tok_off, const int32_t* mention_tokens, int n_mentions,
                                int n_mention_tokens, const int32_t* tag_tok_off, const int32_t* tag_tokens,
                                int n_tag_tokens, float p_row, float p_mr, float p_lwtr, float p_sis, float p_mlm,
                                uint64_t seed, int pad_id, int pad_tag, int mask_id, int32_t* token_out,
                                int32_t* label_out, int32_t* seq_len_out, int32_t* mask_out, int32_t* segment_out,
                                int32_t* mlm_ids, int32_t* mlm_positions, ner_stream_t stream) {
  if (B < 0 || L < 1 || K < 1 || T < 0) return NER_ERR_INVALID_ARG;
  if (L > NER_AUGMENT_MAX_LEN || K > NER_MAX_TAGS_WIDE) return NER_ERR_UNSUPPORTED;
  if ((long long)B * L > 0x7fffffffLL) return NER_ERR_UNSUPPORTED;
  if (!prob_ok(p_row) || !prob_ok(p_mr) || !prob_ok(p_lwtr) || !prob_ok(p_sis) || !prob_ok(p_mlm))
    return NER_ERR_INVALID_ARG;
  if (n_mentions < 0 || n_mention_tokens < 0 || n_tag_tokens < 0) return NER_ERR_INVALID_ARG;
  if ((mlm_ids == nullptr) != (mlm_positions == nullptr)) return NER_ERR_INVALID_ARG;
  if (mlm_ids == nullptr && p_mlm > 0.f) return NER_ERR_INVALID_ARG;
  if (mlm_ids != nullptr && mask_id < 0) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!token_ids || !label_ids || !seq_len || !mask || !segment_ids || !tag_class || !token_out || !label_out ||
      !seq_len_out || !mask_out || !segment_out)
    return NER_ERR_INVALID_ARG;
  if (p_mr > 0.f && (T < 1 || !type_tag || !mention_type_off || !mention_tok_off || (n_mention_tokens > 0 && !mention_tokens)))
    return NER_ERR_INVALID_ARG;
  if (p_lwtr > 0.f && (!tag_tok_off || (n_tag_tokens > 0 && !tag_tokens))) return NER_ERR_INVALID_ARG;
  RowArgs a{token_ids, label_ids, seq_len, mask, segment_ids, B, L, K, T, tag_class, type_tag, mention_type_off,
            mention_tok_off, mention_tokens, n_mentions, n_mention_tokens, tag_tok_off, tag_tokens, n_tag_tokens,
            threshold(p_row), threshold(p_mr), threshold(p_lwtr), threshold(p_sis), threshold(p_mlm), seed, pad_id,
            pad_tag, mask_id, token_out, label_out, seq_len_out, mask_out, segment_out, mlm_ids, mlm_positions};
  const size_t smem = ner_augment_rows_smem_bytes(L);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (smem > 48 * 1024) cudaFuncSetAttribute(augment_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  augment_rows_kernel<<<B, kRowThreads, smem, st>>>(a);
  return ner_launch_status();
}

extern "C" int ner_vocab_sample(const float* logits, int ld, int V, const uint8_t* eligible, const int32_t* positions,
                                int M, long long n_tokens, float temperature, uint64_t seed, int32_t* token_ids,
                                ner_stream_t stream) {
  if (M < 0 || V < 1 || ld < V || ld % 4 != 0 || n_tokens < 0) return NER_ERR_INVALID_ARG;
  if (V > NER_MLM_MAX_VOCAB) return NER_ERR_UNSUPPORTED;
  if (!(temperature > 0.f) || !std::isfinite(temperature)) return NER_ERR_INVALID_ARG;
  if (M == 0) return NER_OK;
  if (!logits || !eligible || !positions || !token_ids) return NER_ERR_INVALID_ARG;
  if (reinterpret_cast<uintptr_t>(logits) % 16) return NER_ERR_INVALID_ARG;
  vocab_sample_kernel<<<M, kSampleThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      logits, ld, V, eligible, positions, n_tokens, 1.f / temperature, seed, token_ids);
  return ner_launch_status();
}
