// GPU entity-span extraction (SURVEY 8(f) rank 2): the serving-side tail of PREDICT.
//
// Reference: extract_entity, tools/infer_utils.py:76-99 — a sequential scan over (token, tag) pairs:
//   tag kind 'I' (tag.split('-')[0] == 'I'):  the token joins the open n-gram iff the PREVIOUS tag's first character is 'B'
//                                            or 'I' (for the first token the previous tag is the token's own tag);
//   any other tag:                            a non-empty n-gram is emitted under the type of the previous tag
//                                            (prev_tag.split('-')[1]); 'B' opens a new n-gram with this token;
//   end of sequence:                          a non-empty n-gram is emitted under the type of the last tag.
// As a function of the tag sequence alone this is a set of spans [start, end) with a type:
//   in(p)    = kind(p) == B  or  (kind(p) == I and prevBI(p-1))            prevBI(-1) := prevBI(0)
//   start(p) = in(p) and (kind(p) == B or not in(p-1))
//   end      = first q > start with kind(q) != I (or L);   type = type(tag[end-1])
// (note the reference's quirks survive: "O I I" opens a span at the second I; "B-ORG I-PER" is one span typed PER).
// The kernel emits exactly these spans, in order, so the host only joins token strings: the [B, L] tag tensor never has
// to leave the device for serving, the device -> host traffic is 4 bytes per entity.
//
// One warp per sentence: the sentence's tag classes are staged in shared memory (one byte per position), each lane tests
// the positions p = 32 c + lane, ballots rank the starts, every start lane walks its own span to its end.
#include "common.cuh"

namespace {
constexpr int kWarpsPerCta = 4;

// tag class: bits 0-1 kind (0 other, 1 B, 2 I), bit 2 = "first character is B or I" (what the reference tests on the
// previous tag), bits 3.. entity type id: 5 bits in the byte-wide table (ner_extract_spans), 7 in the 16-bit one
// (ner_extract_spans_wide).
template <typename Cls>
__global__ void __launch_bounds__(kWarpsPerCta * 32) span_extract_kernel(const int32_t* __restrict__ pred_ids,
                                                                        const Cls* __restrict__ tag_class,
                                                                        int32_t* __restrict__ spans,
                                                                        int32_t* __restrict__ counts, int B, int L, int K,
                                                                        int cap) {
  extern __shared__ uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * kWarpsPerCta + warp;
  if (b >= B) return;
  Cls* cls = reinterpret_cast<Cls*>(smem) + (size_t)warp * L;
  const int32_t* row = pred_ids + (size_t)b * L;
  for (int p = lane; p < L; p += 32) {
    const int id = row[p];
    cls[p] = (id >= 0 && id < K) ? tag_class[id] : (Cls)0;
  }
  __syncwarp();
  int n_emitted = 0;
  for (int c0 = 0; c0 < L; c0 += 32) {
    const int p = c0 + lane;
    bool start = false;
    if (p < L) {
      const int cur = cls[p];
      const int kind = cur & 3;
      auto in_span = [&](int q) -> bool {       // q in [0, L)
        const int cq = cls[q], kq = cq & 3;
        if (kq == 1) return true;
        if (kq != 2) return false;
        const int prev = q == 0 ? cq : cls[q - 1];
        return (prev & 4) != 0;
      };
      const bool in = in_span(p);
      start = in && (kind == 1 || p == 0 || !in_span(p - 1));
    }
    const unsigned m = __ballot_sync(0xffffffffu, start);
    if (start) {
      const int slot = n_emitted + __popc(m & ((1u << lane) - 1u));
      int e = p + 1;
      while (e < L && (cls[e] & 3) == 2) ++e;
      if (slot < cap) spans[(size_t)b * cap + slot] = p | (e << 12) | ((int)(cls[e - 1] >> 3) << 24);
    }
    n_emitted += __popc(m);
  }
  if (lane == 0) counts[b] = n_emitted;
}

template <typename Cls>
int extract_spans(const int32_t* pred_ids, const Cls* tag_class, int32_t* spans, int32_t* counts, int B, int L, int K,
                  int cap, ner_stream_t stream) {
  if (B < 0 || L < 1 || K < 1 || cap < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!pred_ids || !tag_class || !spans || !counts) return NER_ERR_INVALID_ARG;
  if (L > 4095 || K > 256) return NER_ERR_UNSUPPORTED;      // span word: start 12 bits | end 12 bits | type
  const size_t smem = (size_t)kWarpsPerCta * L * sizeof(Cls);
  const int grid = (B + kWarpsPerCta - 1) / kWarpsPerCta;
  span_extract_kernel<Cls><<<grid, kWarpsPerCta * 32, smem, static_cast<cudaStream_t>(stream)>>>(pred_ids, tag_class, spans,
                                                                                               counts, B, L, K, cap);
  return ner_launch_status();
}
}  // namespace

extern "C" int ner_extract_spans(const int32_t* pred_ids, const uint8_t* tag_class, int32_t* spans, int32_t* counts, int B,
                                 int L, int K, int cap, ner_stream_t stream) {
  return extract_spans(pred_ids, tag_class, spans, counts, B, L, K, cap, stream);
}

extern "C" int ner_extract_spans_wide(const int32_t* pred_ids, const uint16_t* tag_class, int32_t* spans, int32_t* counts,
                                      int B, int L, int K, int cap, ner_stream_t stream) {
  return extract_spans(pred_ids, tag_class, spans, counts, B, L, K, cap, stream);
}
