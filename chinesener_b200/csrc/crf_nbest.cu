// N-best CRF decoding (list Viterbi), sm_90a: the N highest-scoring tag paths of every sequence, best first.
//
// Extends tf.contrib.crf.crf_decode (ner_crf_viterbi) from the one best path to the N best.  Each (t, j) keeps a list
// of up to N entries (score, predecessor tag i, predecessor rank r), sorted by
//   1. s_{t-1}[i][r] + trans[i][j] descending (the sum ner_crf_viterbi compares; adding x[t][j] to it is monotone, so
//      the list is also sorted by its scores s_t[j][k] = (s_{t-1}[i][r] + trans[i][j]) + x[t][j]),
//   2. lower i,  3. lower r.
// The lists at t = n-1 are merged by score descending, lower last tag, lower rank, and the first N are backtracked.
// Rank 0 is then exactly ner_crf_viterbi's path and best_score (strict '>' first max, same fp32 association order), and
// every score is the fp32 left-to-right sum of its own path.
//
// Layout: crf_small.cu's lane-per-tag groups (crf::Lanes<K>: GS = 8/16/32 lanes per sequence, one warp per CTA).
// Lane j keeps the heads of the K predecessor lists in K compile-time-indexed registers and builds its new list by N
// rounds of a K-way merge over them; the lists of the previous step sit in a double-buffered shared-memory tile of the
// group.  Backpointers ((i, r) as one 16-bit i * 16 + r) go to the caller's workspace [B, L, K, N], so every L the
// plugins use (up to document mode's 4095) runs without allocation or host synchronisation.
#include "crf_common.cuh"

namespace {

using namespace nerdev;
using crf::Lanes;

constexpr int PF = 4;       // emission prefetch depth (time steps)
constexpr int NMAX = 16;    // largest N; the shared list tile has NMAX slots per tag

// N rounds of a K-way merge of K sorted lists.  head(i, r) = key of entry r of list i (lists hold `cnt` entries each);
// emit(k, key, i, r) receives the k-th largest, ties to the lower i, then the lower r.  A drained list's head is NaN,
// which loses every comparison.
template <int K, typename Head, typename Emit>
__device__ __forceinline__ void merge_lists(int cnt, int cnew, Head head, Emit emit) {
  float v[K];
  int h[K];
#pragma unroll
  for (int i = 0; i < K; ++i) {
    v[i] = head(i, 0);
    h[i] = 0;
  }
  for (int k = 0; k < cnew; ++k) {
    float best = v[0];
    int bi = 0, bh = h[0];
#pragma unroll
    for (int i = 1; i < K; ++i)
      if (v[i] > best || isnan(best)) {
        best = v[i];
        bi = i;
        bh = h[i];
      }
    emit(k, best, bi, bh);
    const int nh = bh + 1;
    const float nv = nh < cnt ? head(bi, nh) : __int_as_float(0x7fc00000);
#pragma unroll
    for (int i = 0; i < K; ++i)
      if (i == bi) {
        v[i] = nv;
        h[i] = nh;
      }
  }
}

template <int K>
__global__ void __launch_bounds__(32)
crf_nbest_lanes_kernel(const float* __restrict__ logits, const int32_t* __restrict__ seq_len,
                       const float* __restrict__ trans, int N, int32_t* __restrict__ tags_out,
                       float* __restrict__ scores_out, int32_t* __restrict__ count_out, uint16_t* __restrict__ bp,
                       int B, int L) {
  constexpr int GS = Lanes<K>::GS, SPW = Lanes<K>::SPW;
  __shared__ float s_tr[K * K];
  __shared__ float s_list[SPW][2][K][NMAX];   // [group][step parity][tag][rank] scores
  __shared__ uint16_t s_fin[SPW][NMAX];       // (last tag, rank) of each final path

  const int lane = threadIdx.x;
  const int g = lane / GS, j = lane % GS;
  const int b = blockIdx.x * SPW + g;
  const bool seq_ok = b < B;
  const bool tag_ok = j < K;
  for (int e = lane; e < K * K; e += 32) s_tr[e] = trans[e];
  int len = 1;
  if (seq_ok) len = min(max(seq_len[b], 1), L);  // len <= 0 decodes like len 1 (TF quirk, as ner_crf_viterbi)
  int wmax = len;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));

  const float* xp = logits + (size_t)(seq_ok ? b : 0) * L * K + (tag_ok ? j : 0);
  auto ld = [&](int t) -> float { return (seq_ok && tag_ok && t < len) ? xp[(size_t)t * K] : -INFINITY; };
  uint16_t* bpb = bp + (size_t)(seq_ok ? b : 0) * L * K * N;
  float(*lists)[K][NMAX] = s_list[g];
  if (tag_ok) lists[0][j][0] = ld(0);
  float xq[PF];
#pragma unroll
  for (int i = 0; i < PF; ++i) xq[i] = ld(1 + i);
  int cnt = 1;  // entries per list at the last decoded step: min(N, K^(t+1)), the same for every tag
  __syncwarp();

  for (int t0 = 1; t0 < wmax; t0 += PF) {
#pragma unroll
    for (int u = 0; u < PF; ++u) {
      const int t = t0 + u;
      const float x = xq[u];
      xq[u] = ld(t + PF);
      if (t < wmax) {
        if (t < len) {
          const int cnew = min(N, cnt * K);
          if (tag_ok) {
            const float(*prv)[NMAX] = lists[(t - 1) & 1];
            float* cur = lists[t & 1][j];
            uint16_t* bpt = bpb + ((size_t)t * K + j) * N;
            merge_lists<K>(
                cnt, cnew, [&](int i, int r) { return prv[i][r] + s_tr[i * K + j]; },
                [&](int k, float key, int i, int r) {
                  cur[k] = x + key;
                  bpt[k] = (uint16_t)(i * NMAX + r);
                });
          }
          cnt = cnew;
        }
        __syncwarp();
      }
    }
  }

  const int nfin = min(N, cnt * K);  // min(N, K^len), the paths there are
  if (j == 0 && seq_ok) {
    const float(*fin)[NMAX] = lists[(len - 1) & 1];
    float* so = scores_out + (size_t)b * N;
    merge_lists<K>(
        cnt, nfin, [&](int i, int r) { return fin[i][r]; },
        [&](int k, float key, int i, int r) {
          so[k] = key;
          s_fin[g][k] = (uint16_t)(i * NMAX + r);
        });
    for (int k = nfin; k < N; ++k) so[k] = -INFINITY;
    if (count_out != nullptr) count_out[b] = nfin;
  }
  __syncwarp();
  if (!seq_ok) return;
  // backtrack: lane j of the group follows ranks j, j + GS, ...
  for (int k = j; k < N; k += GS) {
    int32_t* out = tags_out + ((size_t)b * N + k) * L;
    int lim = 0;
    if (k < nfin) {
      const int p = s_fin[g][k];
      int y = p / NMAX, r = p % NMAX;
      for (int t = len - 1; t >= 1; --t) {
        out[t] = y;
        const int q = bpb[((size_t)t * K + y) * N + r];
        y = q / NMAX;
        r = q % NMAX;
      }
      out[0] = y;
      lim = len;
    }
    for (int t = lim; t < L; ++t) out[t] = 0;
  }
}

template <int K>
int launch_nbest(const float* logits, const int32_t* seq_len, const float* trans, int N, int32_t* tags_out,
                 float* scores_out, int32_t* count_out, uint16_t* bp, int B, int L, cudaStream_t st) {
  constexpr int SPW = Lanes<K>::SPW;
  crf_nbest_lanes_kernel<K><<<(B + SPW - 1) / SPW, 32, 0, st>>>(logits, seq_len, trans, N, tags_out, scores_out,
                                                                count_out, bp, B, L);
  return ner_launch_status();
}

}  // namespace

extern "C" size_t ner_crf_viterbi_nbest_workspace_bytes(int B, int L, int K, int N) {
  if (B < 1 || L < 1 || K < 1 || K > NER_MAX_TAGS || N < 1 || N > NMAX) return 0;
  return (size_t)B * L * K * N * sizeof(uint16_t);
}

extern "C" int ner_crf_viterbi_nbest(const float* logits, const int32_t* seq_len, const float* trans, int N,
                                     int32_t* tags_out, float* scores_out, int32_t* count_out, void* workspace,
                                     size_t workspace_bytes, int B, int L, int K, ner_stream_t stream) {
  if (K < 1 || K > NER_MAX_TAGS || N < 1 || N > NMAX) return NER_ERR_UNSUPPORTED;
  if (B < 0 || L < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!logits || !seq_len || !trans || !tags_out || !scores_out) return NER_ERR_INVALID_ARG;
  if (!workspace || workspace_bytes < ner_crf_viterbi_nbest_workspace_bytes(B, L, K, N)) return NER_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint16_t* bp = static_cast<uint16_t*>(workspace);
#define CALL(KK) return launch_nbest<KK>(logits, seq_len, trans, N, tags_out, scores_out, count_out, bp, B, L, st)
  NER_CRF_DISPATCH_K(K, CALL)
#undef CALL
  return NER_ERR_UNSUPPORTED;
}
