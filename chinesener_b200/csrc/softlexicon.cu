// SoftLexicon B/M/E/S gather-and-pool (sm_90a), forward and backward.
//
// Replaces the embedding_lookup * weight -> reshape -> reduce_sum block of reference
// model/bilstm_crf_softlexicon.py:37-44 (same block in bert_bilstm_crf_softlexicon.py):
//   out[tok, g*E + e] = sum_{s<S} weights[tok, g*S + s] * table[ids[tok, g*S + s], e]
// with G = word_enhance_dim (4: B,M,E,S) groups of S = max_lexicon_len (10) slots
// (layout contract: data/word_enhance.py:163-205, data/base_preprocess.py:414-428).
//
// One warp per token.  The G*S (<= 64) ids/weights of a token are read coalesced, the
// non-zero-weight slots are compacted with a ballot (pad / <None> slots carry weight 0 and
// are never fetched), and each surviving slot is one 4*E-byte row gather spread over the
// lanes; the [B,L,G*S,E] intermediate the reference materialises never exists.
#include "common.cuh"

namespace {

using namespace nerdev;

constexpr int MAXE_PER_LANE = 4;  // E <= 128

__global__ void __launch_bounds__(256)
softlexicon_pool_fwd_kernel(const float* __restrict__ table, const int32_t* __restrict__ ids,
                            const float* __restrict__ weights, float* __restrict__ out, int n_tok, int G, int S,
                            int E, int V, int ld_out) {
  const int lane = threadIdx.x & 31;
  const int GS = G * S;
  const int wpb = blockDim.x >> 5;
  for (int tok = blockIdx.x * wpb + (threadIdx.x >> 5); tok < n_tok; tok += gridDim.x * wpb) {
    const int32_t* idp = ids + (size_t)tok * GS;
    const float* wp = weights + (size_t)tok * GS;
    // slots lane and lane+32
    int id0 = 0, id1 = 0;
    float w0 = 0.f, w1 = 0.f;
    if (lane < GS) {
      id0 = idp[lane];
      w0 = wp[lane];
    }
    if (lane + 32 < GS) {
      id1 = idp[lane + 32];
      w1 = wp[lane + 32];
    }
    uint32_t nz0 = __ballot_sync(0xffffffffu, w0 != 0.f);
    uint32_t nz1 = __ballot_sync(0xffffffffu, w1 != 0.f);
    float* op = out + (size_t)tok * ld_out;
    for (int g = 0; g < G; ++g) {
      float acc[MAXE_PER_LANE];
#pragma unroll
      for (int k = 0; k < MAXE_PER_LANE; ++k) acc[k] = 0.f;
      const int s_lo = g * S, s_hi = s_lo + S;  // slots of this group
      // walk the non-zero slots of group g in slot order (deterministic summation order)
      for (int s = s_lo; s < s_hi; ++s) {
        const bool hit = (s < 32) ? ((nz0 >> s) & 1u) : ((nz1 >> (s - 32)) & 1u);
        if (!hit) continue;
        const int id = (s < 32) ? __shfl_sync(0xffffffffu, id0, s) : __shfl_sync(0xffffffffu, id1, s - 32);
        const float w = (s < 32) ? __shfl_sync(0xffffffffu, w0, s) : __shfl_sync(0xffffffffu, w1, s - 32);
        const float* row = table + (size_t)min(max(id, 0), V - 1) * E;
#pragma unroll
        for (int k = 0; k < MAXE_PER_LANE; ++k) {
          const int e = lane + 32 * k;
          if (e < E) acc[k] = fmaf(w, __ldg(row + e), acc[k]);
        }
      }
#pragma unroll
      for (int k = 0; k < MAXE_PER_LANE; ++k) {
        const int e = lane + 32 * k;
        if (e < E) op[g * E + e] = acc[k];
      }
    }
  }
}

// d_table[ids[tok,slot], :] += weights[tok,slot] * d_out[tok, g(slot)*E : (g+1)*E]
__global__ void __launch_bounds__(256)
softlexicon_pool_bwd_kernel(float* __restrict__ d_table, const int32_t* __restrict__ ids,
                            const float* __restrict__ weights, const float* __restrict__ d_out, int n_tok, int G,
                            int S, int E, int V) {
  const int lane = threadIdx.x & 31;
  const int GS = G * S;
  const int wpb = blockDim.x >> 5;
  for (int tok = blockIdx.x * wpb + (threadIdx.x >> 5); tok < n_tok; tok += gridDim.x * wpb) {
    const int32_t* idp = ids + (size_t)tok * GS;
    const float* wp = weights + (size_t)tok * GS;
    const float* dp = d_out + (size_t)tok * G * E;
    for (int s = 0; s < GS; ++s) {
      const float w = wp[s];
      if (w == 0.f) continue;  // warp-uniform
      const int id = min(max(idp[s], 0), V - 1);
      const int g = s / S;
      for (int e = lane; e < E; e += 32) atomicAdd(d_table + (size_t)id * E + e, w * dp[g * E + e]);
    }
  }
}

}  // namespace

extern "C" int ner_softlexicon_pool_fwd(const float* table, const int32_t* ids, const float* weights, float* out,
                                        int n_tok, int G, int S, int E, int V, int ld_out, ner_stream_t stream) {
  if (n_tok < 0 || G < 1 || S < 1 || E < 1 || V < 1 || ld_out < G * E) return NER_ERR_INVALID_ARG;
  if (n_tok == 0) return NER_OK;
  if (!table || !ids || !weights || !out) return NER_ERR_INVALID_ARG;
  if (G * S > 64 || E > 32 * MAXE_PER_LANE) return NER_ERR_UNSUPPORTED;
  long grid = ((long)n_tok + 7) / 8;
  if (grid > (long)ner_num_sms() * 32) grid = (long)ner_num_sms() * 32;
  softlexicon_pool_fwd_kernel<<<(int)grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(table, ids, weights, out, n_tok,
                                                                                        G, S, E, V, ld_out);
  return ner_launch_status();
}

extern "C" int ner_softlexicon_pool_bwd(float* d_table, const int32_t* ids, const float* weights, const float* d_out,
                                        int n_tok, int G, int S, int E, int V, ner_stream_t stream) {
  if (n_tok < 0 || G < 1 || S < 1 || E < 1 || V < 1) return NER_ERR_INVALID_ARG;
  if (n_tok == 0) return NER_OK;
  if (!d_table || !ids || !weights || !d_out) return NER_ERR_INVALID_ARG;
  long grid = ((long)n_tok + 7) / 8;
  if (grid > (long)ner_num_sms() * 32) grid = (long)ner_num_sms() * 32;
  softlexicon_pool_bwd_kernel<<<(int)grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(d_table, ids, weights, d_out,
                                                                                        n_tok, G, S, E, V);
  return ner_launch_status();
}
