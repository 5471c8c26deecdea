// MRC-style NER glue of the bert_mrc plugin (model/bert_mrc.py): one BERT query per entity type (sm_90a).
//
// ner_mrc_pairs expands a [B, L] BERT batch into the B*T query/context pairs p = b*T + t,
//   [CLS] query_t [SEP] sentence[1 : seq_len_b]      (n_bt = q_t + 1 + seq_len_b tokens; 0 when seq_len_b = 0)
// and writes the per-type BIO labels and the row index that turns pair rows back into the sentence-aligned [B*T, L]
// layout.  ner_mrc_merge folds the T per-type 3-class logits of each sentence position into one tag of the dataset's tag
// space.  Both kernels are a handful of integer or float ops per element: one launch each, no host synchronisation.
#include "common.cuh"

namespace {

constexpr int kThreads = 128;
constexpr int kMaxTypes = 32;

// One CTA per pair p: the L2 pair columns, then the L sentence positions.
__global__ void __launch_bounds__(kThreads)
mrc_pairs_kernel(const int32_t* __restrict__ token_ids, const int32_t* __restrict__ seq_len,
                 const int32_t* __restrict__ label_ids, const int32_t* __restrict__ query_ids,
                 const int32_t* __restrict__ query_len, const int32_t* __restrict__ type_tag, int L, int T, int Qmax,
                 int L2, int sep_id, int32_t* __restrict__ pair_ids, int32_t* __restrict__ pair_seg,
                 int32_t* __restrict__ pair_mask, int32_t* __restrict__ pair_seq_len, int32_t* __restrict__ pair_labels,
                 int32_t* __restrict__ align_rows) {
  const int p = blockIdx.x;
  const int b = p / T, t = p - b * T;
  const int len = min(max(__ldg(seq_len + b), 0), L);
  const int q = min(max(__ldg(query_len + t), 0), Qmax);
  const int n = len > 0 ? q + 1 + len : 0;
  const int32_t* tok = token_ids + (size_t)b * L;
  const int32_t* qry = query_ids + (size_t)t * Qmax;
  const size_t row = (size_t)p * L2;
  for (int j = threadIdx.x; j < L2; j += kThreads) {
    int id = 0, seg = 0;
    if (j < n) {
      if (j == 0) id = __ldg(tok);
      else if (j <= q) id = __ldg(qry + j - 1);
      else if (j == q + 1) id = sep_id;
      else {
        id = __ldg(tok + j - q - 1);
        seg = 1;
      }
    }
    pair_ids[row + j] = id;
    pair_seg[row + j] = seg;
    pair_mask[row + j] = j < n ? 1 : 0;
  }
  if (threadIdx.x == 0) pair_seq_len[p] = len;
  const int tag_b = __ldg(type_tag + 2 * t), tag_i = __ldg(type_tag + 2 * t + 1);
  for (int s = threadIdx.x; s < L; s += kThreads) {
    align_rows[(size_t)p * L + s] = (int32_t)(row + (s == 0 ? 0 : q + 1 + s));
    if (pair_labels != nullptr) {
      int y = 0;
      if (s < len) {
        const int tag = __ldg(label_ids + (size_t)b * L + s);
        y = tag == tag_b ? 1 : tag == tag_i ? 2 : 0;
      }
      pair_labels[(size_t)p * L + s] = y;
    }
  }
}

// One thread per sentence position (b, s).  Candidate t: first argmax a_t != O of its 3 logits, score z[a_t] - lse(z) =
// -log(sum_k exp(z_k - z[a_t])); the highest score wins, the lowest type index on a tie.
__global__ void __launch_bounds__(kThreads)
mrc_merge_kernel(const float* __restrict__ logits, const int32_t* __restrict__ seq_len, const int32_t* __restrict__ type_tag,
                 int B, int L, int T, int o_id, int cls_id, int sep_id, int32_t* __restrict__ pred_ids) {
  __shared__ int32_t s_tag[2 * kMaxTypes];
  for (int i = threadIdx.x; i < 2 * T; i += kThreads) s_tag[i] = __ldg(type_tag + i);
  __syncthreads();
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= (long long)B * L) return;
  const int b = (int)(i / L), s = (int)(i - (long long)b * L);
  const int len = min(max(__ldg(seq_len + b), 0), L);
  int out;
  if (s >= len) out = 0;
  else if (s == 0) out = cls_id;
  else if (s == len - 1) out = sep_id;
  else {
    out = o_id;
    float best = 0.f;
    bool any = false;
    for (int t = 0; t < T; ++t) {
      const float* z = logits + (((size_t)b * T + t) * L + s) * 3;
      const float z0 = __ldg(z), z1 = __ldg(z + 1), z2 = __ldg(z + 2);
      int a = 0;
      float m = z0;
      if (z1 > m) { m = z1; a = 1; }
      if (z2 > m) { m = z2; a = 2; }
      if (a == 0) continue;
      const float score = -logf(expf(z0 - m) + expf(z1 - m) + expf(z2 - m));
      if (!any || score > best) {
        any = true;
        best = score;
        out = s_tag[2 * t + a - 1];
      }
    }
  }
  pred_ids[i] = out;
}

}  // namespace

extern "C" int ner_mrc_pairs(const int32_t* token_ids, const int32_t* seq_len, const int32_t* label_ids,
                             const int32_t* query_ids, const int32_t* query_len, const int32_t* type_tag, int B, int L,
                             int T, int Qmax, int L2, int sep_id, int32_t* pair_ids, int32_t* pair_segment_ids,
                             int32_t* pair_mask, int32_t* pair_seq_len, int32_t* pair_labels, int32_t* align_rows,
                             ner_stream_t stream) {
  if (B < 0 || L < 1 || T < 1 || Qmax < 0) return NER_ERR_INVALID_ARG;
  if (T > kMaxTypes) return NER_ERR_UNSUPPORTED;
  if ((long long)L2 < (long long)Qmax + 1 + L) return NER_ERR_INVALID_ARG;
  if ((long long)B * T * L2 > 0x7fffffffLL) return NER_ERR_UNSUPPORTED;
  if (B == 0) return NER_OK;
  if (!token_ids || !seq_len || !query_len || !type_tag || (Qmax > 0 && !query_ids)) return NER_ERR_INVALID_ARG;
  if (!pair_ids || !pair_segment_ids || !pair_mask || !pair_seq_len || !align_rows) return NER_ERR_INVALID_ARG;
  if (pair_labels && !label_ids) return NER_ERR_INVALID_ARG;
  mrc_pairs_kernel<<<B * T, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      token_ids, seq_len, label_ids, query_ids, query_len, type_tag, L, T, Qmax, L2, sep_id, pair_ids, pair_segment_ids,
      pair_mask, pair_seq_len, pair_labels, align_rows);
  return ner_launch_status();
}

extern "C" int ner_mrc_merge(const float* logits, const int32_t* seq_len, const int32_t* type_tag, int B, int L, int T,
                             int o_id, int cls_id, int sep_id, int32_t* pred_ids, ner_stream_t stream) {
  if (B < 0 || L < 1 || T < 1) return NER_ERR_INVALID_ARG;
  if (T > kMaxTypes) return NER_ERR_UNSUPPORTED;
  if ((long long)B * T * L > 0x7fffffffLL) return NER_ERR_UNSUPPORTED;
  if (B == 0) return NER_OK;
  if (!logits || !seq_len || !type_tag || !pred_ids) return NER_ERR_INVALID_ARG;
  const long long n = (long long)B * L;
  mrc_merge_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      logits, seq_len, type_tag, B, L, T, o_id, cls_id, sep_id, pred_ids);
  return ner_launch_status();
}
