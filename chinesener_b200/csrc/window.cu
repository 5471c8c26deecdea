// Document mode of the BERT plugins (sm_90a): the window plan of documents longer than BERT's position table.
//
// ner_window_plan cuts each document of a [B, L] batch into overlapping W-token windows (run_squad's doc_stride
// windows, every window keeping the document's own [CLS] and [SEP]) and writes, for every document token, the encoder
// row of the window where that token has the most context (run_squad's _check_is_max_context).  The encoder then runs
// on the window batch and two row gathers stitch its output back into the document layout.  One launch, integer work
// only, no atomics: every output element is written by exactly one thread, so repeat calls are bit-identical.
#include "common.cuh"

namespace {

constexpr int kThreads = 128;

// Windows of a document with n tokens (m = n - 2 content tokens, C = W - 2 per window).
__device__ __forceinline__ int doc_windows(int n, int W, int S) {
  if (n <= 0) return 0;
  if (n <= W) return 1;
  const int excess = (n - 2) - (W - 2);
  return 1 + (excess + S - 1) / S;
}

// Window tokens of the document in the window-packed layout: n when it is its own window, else nw * W.
__device__ __forceinline__ long long doc_window_tokens(int n, int W, int S) {
  return n <= W ? (long long)max(n, 0) : (long long)doc_windows(n, W, S) * W;
}

__device__ __forceinline__ long long block_sum(long long v, long long* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();                                  // red may still be read by the previous call
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  long long s = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) s += red[w];
  return s;
}

// One CTA per document b.  Its first window, first window token and first packed document token are prefix sums over
// the documents before it, computed by the CTA itself (B is at most a few thousand rows).
__global__ void __launch_bounds__(kThreads)
window_plan_kernel(const int32_t* __restrict__ token_ids, const int32_t* __restrict__ segment_ids,
                   const int32_t* __restrict__ seq_len, int B, int L, int W, int S, int NW, int32_t* __restrict__ win_ids,
                   int32_t* __restrict__ win_seg, int32_t* __restrict__ win_mask, int32_t* __restrict__ doc_src_packed,
                   int32_t* __restrict__ doc_src_padded) {
  __shared__ long long red[kThreads / 32];
  const int b = blockIdx.x;
  long long w0 = 0, t0 = 0, d0 = 0;
  for (int j = threadIdx.x; j < b; j += kThreads) {
    const int nj = min(max(__ldg(seq_len + j), 0), L);
    w0 += doc_windows(nj, W, S);
    t0 += doc_window_tokens(nj, W, S);
    d0 += nj;
  }
  const long long win_base = block_sum(w0, red);
  const long long tok_base = block_sum(t0, red);
  const long long doc_base = block_sum(d0, red);

  const int n = min(max(__ldg(seq_len + b), 0), L);
  const int nw = doc_windows(n, W, S);
  const int C = W - 2, m = n - 2;
  const int32_t* tok = token_ids + (size_t)b * L;
  const int32_t* seg = segment_ids ? segment_ids + (size_t)b * L : nullptr;

  // window rows: k = j / W, position p = j % W; a window of n <= W tokens is the document itself, padded to W
  for (int j = threadIdx.x; j < nw * W; j += kThreads) {
    const int k = j / W, p = j - k * W;
    const long long w = win_base + k;
    if (w >= NW) break;
    int src = -1;
    if (n <= W) src = p < n ? p : -1;
    else if (p == 0) src = 0;
    else if (p == W - 1) src = n - 1;
    else src = min(k * S, m - C) + p;             // doc position 1 + a_k + (p - 1)
    const size_t o = (size_t)w * W + p;
    win_ids[o] = src >= 0 ? __ldg(tok + src) : 0;
    win_seg[o] = (src >= 0 && seg) ? __ldg(seg + src) : 0;
    win_mask[o] = src >= 0 ? 1 : 0;
  }
  // the last document also clears the windows past the plan's own count (a host NW larger than the batch needs)
  if (b == B - 1) {
    const long long used = win_base + nw;
    for (long long o = used * W + threadIdx.x; o < (long long)NW * W; o += kThreads) {
      win_ids[o] = 0;
      win_seg[o] = 0;
      win_mask[o] = 0;
    }
  }
  if (!doc_src_packed && !doc_src_padded) return;

  // owner of doc position t: window k, row p within it
  for (int t = threadIdx.x; t < n; t += kThreads) {
    int k = 0, p = t;
    if (n > W) {
      if (t == 0) {
        p = 0;
      } else if (t == n - 1) {
        k = nw - 1;
        p = W - 1;
      } else {
        // content index c: the candidate windows a_k <= c < a_k + C are consecutive, and the context
        // min(c - a_k, a_k + C - 1 - c) is unimodal in k, so walk up from the first one until it drops
        const int c = t - 1;
        const int lo = c - C + 1;
        int kk = lo > 0 ? (lo + S - 1) / S : 0;
        kk = min(kk, nw - 1);
        int best = -1;
        for (; kk < nw; ++kk) {
          const int a = min(kk * S, m - C);
          if (a > c) break;
          const int score = min(c - a, a + C - 1 - c);
          if (score > best) {
            best = score;
            k = kk;
            p = c - a + 1;
          } else if (score < best) {
            break;
          }
        }
      }
    }
    const long long w = win_base + k;
    if (doc_src_padded) doc_src_padded[doc_base + t] = (int32_t)(w * W + p);
    if (doc_src_packed) doc_src_packed[doc_base + t] = (int32_t)(tok_base + (n <= W ? t : (long long)k * W + p));
  }
}

}  // namespace

extern "C" int ner_window_plan(const int32_t* token_ids, const int32_t* segment_ids, const int32_t* seq_len, int B, int L,
                               int W, int S, int NW, int32_t* win_ids, int32_t* win_segment_ids, int32_t* win_mask,
                               int32_t* doc_src_packed, int32_t* doc_src_padded, ner_stream_t stream) {
  if (B < 0 || L < 1 || NW < 0 || W < 3) return NER_ERR_INVALID_ARG;
  if (S < 1 || S > W - 2) return NER_ERR_INVALID_ARG;
  if ((long long)NW * W > 0x7fffffffLL || (long long)B * L > 0x7fffffffLL) return NER_ERR_UNSUPPORTED;
  if (B == 0) return NER_OK;
  if (!token_ids || !seq_len) return NER_ERR_INVALID_ARG;
  if (NW > 0 && (!win_ids || !win_segment_ids || !win_mask)) return NER_ERR_INVALID_ARG;
  window_plan_kernel<<<B, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      token_ids, segment_ids, seq_len, B, L, W, S, NW, win_ids, win_segment_ids, win_mask, doc_src_packed, doc_src_padded);
  return ner_launch_status();
}
