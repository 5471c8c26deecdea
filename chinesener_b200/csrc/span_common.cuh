// Span decoding shared by the two span heads, mrc_span.cu (start / end pointers and a match score per (t, i, j)) and
// global_pointer.cu (a score per (t, i, j)): the priority key, the run end of a BIO label span, and the greedy decode
// from a [B, T, L, L] score tensor to the span list and pred_ids.  The heads differ only in which types are candidates
// at (i, j); each passes that as a candidate policy (see greedy_span_decode).
#pragma once
#include "common.cuh"

namespace span {

constexpr int kDecodeRows = 512;      // positions of a sentence the decode holds in shared memory
constexpr int kDecodeThreads = 256;   // CTA size of a decode kernel

__device__ __forceinline__ int clamp_len(int32_t v, int L) { return min(max((int)v, 0), L); }

// End of the span starting at s: the last r >= s with y[s+1 .. r] all `inside` and r < len
__device__ __forceinline__ int run_end(const int32_t* y, int s, int len, int inside) {
  int r = s;
  while (r + 1 < len && y[r + 1] == inside) ++r;
  return r;
}

// Priority of span (t, i, j) with score zz > 0: higher zz first, then lower type, lower start, lower end.  i, j <= 510
// (the heads' sequence bounds) keep 0 out of the 9-bit fields, so 0 is "no span".
__device__ __forceinline__ unsigned long long span_key(float zz, int t, int i, int j) {
  return ((unsigned long long)__float_as_uint(zz) << 32) | ((unsigned)(31 - t) << 18) | ((unsigned)(511 - i) << 9) |
         (unsigned)(511 - j);
}

inline bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15u) == 0; }

// Decode of sentence b = blockIdx.x (kDecodeThreads threads, len <= L <= kDecodeRows) over the scores
// sc[b, t, i, j] of the candidates 1 <= i <= j <= len - 2, where span (t, i, j) is kept iff its score is > 0:
//   spans / probs[b, 0 .. cap): the span word i | (j + 1) << 12 | t << 24 and sigmoid(score), ordered by (start, end,
//     type) and zero past the count; span_counts[b] = the count, which may exceed cap;
//   pred_ids[b]: [CLS], the greedy non-overlapping projection of the spans (repeatedly keep the best remaining span that
//     overlaps nothing kept; B / I tags from type_tag, o_id elsewhere), [SEP], 0 past len.
// Each row i keeps the key of its best free span; keeping [a, e] clears rows a..e and rescans only the rows before a
// whose best span reached into [a, e].
// Cand states which types are candidates: cand.live(i) is false when row i holds none, and cand.for_each(i, j, f) calls
// f(t) for each candidate type t at (i, j) in ascending t until f returns false (the span list is full).  Shared memory
// the policy reads must be written before the call; the first barrier here publishes it.
template <class Cand>
__device__ __forceinline__ void greedy_span_decode(const Cand& cand, const float* __restrict__ sc, int T, int L, int len,
                                                   const int32_t* __restrict__ type_tag, int o_id, int cls_id, int sep_id,
                                                   int cap, int32_t* __restrict__ pred_ids, int32_t* __restrict__ spans,
                                                   float* __restrict__ probs, int32_t* __restrict__ span_counts) {
  __shared__ int32_t cnt[kDecodeRows + 1], tag[kDecodeRows];
  __shared__ unsigned long long rowkey[kDecodeRows];
  __shared__ uint8_t occ[kDecodeRows];
  const int b = blockIdx.x, tid = threadIdx.x, m = len - 2;
  auto score = [&](int t, int i, int j) { return __ldg(sc + (((size_t)b * T + t) * L + i) * L + j); };
  for (int s = tid; s < L; s += kDecodeThreads) {
    tag[s] = o_id;
    occ[s] = 0;
    rowkey[s] = 0ull;
    cnt[s] = 0;
  }
  __syncthreads();
  for (int i = 1 + tid; i <= m; i += kDecodeThreads) {
    int n = 0;
    unsigned long long best = 0ull;
    if (cand.live(i)) {
      for (int j = i; j <= m; ++j)
        cand.for_each(i, j, [&](int t) {
          const float zz = score(t, i, j);
          if (zz > 0.f) {
            ++n;
            const unsigned long long key = span_key(zz, t, i, j);
            best = key > best ? key : best;
          }
          return true;
        });
    }
    cnt[i] = n;
    rowkey[i] = best;
  }
  __syncthreads();
  if (tid == 0) {
    int run = 0;
    for (int i = 0; i < L; ++i) {
      const int c = cnt[i];
      cnt[i] = run;
      run += c;
    }
    span_counts[b] = run;
    cnt[L] = run;
  }
  __syncthreads();
  for (int o = cnt[L] + tid; o < cap; o += kDecodeThreads) {
    spans[(size_t)b * cap + o] = 0;
    probs[(size_t)b * cap + o] = 0.f;
  }
  for (int i = 1 + tid; i <= m; i += kDecodeThreads) {
    if (!cand.live(i)) continue;
    int o = cnt[i];
    for (int j = i; j <= m && o < cap; ++j)
      cand.for_each(i, j, [&](int t) {
        const float zz = score(t, i, j);
        if (zz > 0.f) {
          spans[(size_t)b * cap + o] = i | (j + 1) << 12 | t << 24;
          probs[(size_t)b * cap + o] = 1.f / (1.f + expf(-zz));
          ++o;
        }
        return o < cap;
      });
  }
  if (tid < 32) {
    const int lane = tid;
    for (;;) {
      unsigned long long best = 0ull;
      for (int i = 1 + lane; i <= m; i += 32) best = rowkey[i] > best ? rowkey[i] : best;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long v = __shfl_xor_sync(0xffffffffu, best, o);
        best = v > best ? v : best;
      }
      if (best == 0ull) break;
      const int t = 31 - (int)((best >> 18) & 31), a = 511 - (int)((best >> 9) & 511), e = 511 - (int)(best & 511);
      const int tb = __ldg(type_tag + 2 * t), tI = __ldg(type_tag + 2 * t + 1);
      for (int q = a + lane; q <= e; q += 32) {
        occ[q] = 1;
        tag[q] = q == a ? tb : tI;
        rowkey[q] = 0ull;
      }
      __syncwarp();
      for (int i = 1 + lane; i < a; i += 32) {
        const unsigned long long key = rowkey[i];
        if (key == 0ull || 511 - (int)(key & 511) < a) continue;
        unsigned long long nb = 0ull;
        for (int j = i; j <= m && !occ[j]; ++j)
          cand.for_each(i, j, [&](int tt) {
            const float zz = score(tt, i, j);
            if (zz > 0.f) {
              const unsigned long long k2 = span_key(zz, tt, i, j);
              nb = k2 > nb ? k2 : nb;
            }
            return true;
          });
        rowkey[i] = nb;
      }
      __syncwarp();
    }
  }
  __syncthreads();
  for (int s = tid; s < L; s += kDecodeThreads) {
    int out;
    if (s >= len) out = 0;
    else if (s == 0) out = cls_id;
    else if (s == len - 1) out = sep_id;
    else out = tag[s];
    pred_ids[(size_t)b * L + s] = out;
  }
}

}  // namespace span
