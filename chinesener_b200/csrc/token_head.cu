// Softmax token head of the bert_ce plugin (model/bert_ce.py + tools/loss.py): masked token cross-entropy, its gradient
// and the first-maximum argmax, in one pass over the logits [B, L, K <= 32] f32 (sm_90a).  Softmax is never stored.
//
// HBM-bound.  A CTA stages a tile of 256 rows (256 * K contiguous floats) through shared memory with coalesced loads, one
// thread then owns one row (the shared rows are laid out with an odd stride, K | 1, so the per-row reads are free of bank
// conflicts), and in TRAIN the gradient goes back through the same tile to coalesced stores.  The loss is reduced without
// float atomics: one partial per CTA, summed in index order by a one-CTA finaliser, so identical inputs give a
// bit-identical loss.  The token count N is summed on the device from seq_len before the main pass, which needs it to
// scale the gradient.
#include "common.cuh"

namespace {

using namespace nerdev;

constexpr int kRows = 256;          // rows per tile = threads per CTA
constexpr int kCtasPerSm = 8;       // grid cap, in CTAs per SM (also sizes the partials of the scratch)
constexpr int kScratchHead = 16;    // scratch[0] = d_loss / N, scratch[1] = N (int bits); partials from kScratchHead on

// N = sum_b clamp(seq_len[b], 0, L); scratch[0] = d_loss / N (0 when N = 0).
__global__ void __launch_bounds__(1024)
token_count_kernel(const int32_t* __restrict__ seq_len, int B, int L, float d_loss, float* __restrict__ scratch) {
  int acc = 0;
  for (int b = threadIdx.x; b < B; b += blockDim.x) acc += min(max(__ldg(seq_len + b), 0), L);
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

// Shared-memory slot of element e of a staged tile: rows of K floats at stride K | 1 (a pad float per row when K is even).
// e / K as a multiply-high: exact for e * K < 2^32 (e < 256 * 32 here).
__device__ __forceinline__ int tile_slot(int e, bool pad, uint32_t k_magic) {
  return pad ? e + (int)__umulhi((uint32_t)e, k_magic) : e;
}

// LABELS: labels / seq_len present, per-CTA loss partials written to scratch.  GRAD: d_logits written (every row).
template <bool LABELS, bool GRAD>
__global__ void __launch_bounds__(kRows)
token_xent_kernel(const float* __restrict__ logits, const int32_t* __restrict__ labels, const int32_t* __restrict__ seq_len,
                  int32_t* __restrict__ pred_ids, float* __restrict__ d_logits, float* __restrict__ scratch, int rows,
                  int L, int K, uint32_t k_magic) {
  extern __shared__ float tile[];
  const int Kp = K | 1;
  const bool pad = (K & 1) == 0;
  const float scale = GRAD ? scratch[0] : 0.f;
  float acc = 0.f;
  for (int r0 = blockIdx.x * kRows; r0 < rows; r0 += gridDim.x * kRows) {
    const int nr = min(kRows, rows - r0);
    const int ne = nr * K;
    const float* src = logits + (size_t)r0 * K;
    for (int e = threadIdx.x; e < ne; e += kRows) tile[tile_slot(e, pad, k_magic)] = __ldcs(src + e);
    __syncthreads();
    const int i = threadIdx.x;
    if (i < nr) {
      const int row = r0 + i;
      float* z = tile + i * Kp;
      float m = z[0];
      int arg = 0;
      for (int j = 1; j < K; ++j) {
        const float v = z[j];
        if (v > m) {                         // strict: the first maximum wins, as tf.argmax / np.argmax
          m = v;
          arg = j;
        }
      }
      if (pred_ids != nullptr) __stcs(pred_ids + row, arg);
      if (LABELS) {
        const int b = row / L, t = row - b * L;
        if (t < __ldg(seq_len + b)) {
          const int y = __ldcs(labels + row);
          const float zy = z[y];
          float s = 0.f;
          for (int j = 0; j < K; ++j) {
            const float ej = expf(z[j] - m);
            s += ej;
            if (GRAD) z[j] = ej;
          }
          acc += (m - zy) + logf(s);
          if (GRAD) {
            const float inv = scale / s;
            for (int j = 0; j < K; ++j) z[j] = z[j] * inv - (j == y ? scale : 0.f);
          }
        } else if (GRAD) {
          for (int j = 0; j < K; ++j) z[j] = 0.f;
        }
      }
    }
    if (GRAD) {
      __syncthreads();
      float* dst = d_logits + (size_t)r0 * K;
      for (int e = threadIdx.x; e < ne; e += kRows) __stcs(dst + e, tile[tile_slot(e, pad, k_magic)]);
    }
    __syncthreads();
  }
  if (LABELS) {
    acc = warp_sum(acc);
    __shared__ float part[kRows / 32];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float s = 0.f;
      for (int w = 0; w < kRows / 32; ++w) s += part[w];
      scratch[kScratchHead + blockIdx.x] = s;
    }
  }
}

// loss[0] = (sum of the partials, in index order) / N, 0 when N = 0.
__global__ void __launch_bounds__(256)
token_xent_final_kernel(const float* __restrict__ scratch, int n_part, float* __restrict__ loss) {
  __shared__ double part[256];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n_part; i += 256) acc += (double)scratch[kScratchHead + i];
  part[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) part[threadIdx.x] += part[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const int n = reinterpret_cast<const int*>(scratch)[1];
    loss[0] = n > 0 ? (float)(part[0] / (double)n) : 0.f;
  }
}

template <bool LABELS, bool GRAD>
void launch_main(int grid, size_t smem, cudaStream_t st, const float* logits, const int32_t* labels, const int32_t* seq_len,
                 int32_t* pred_ids, float* d_logits, float* scratch, int rows, int L, int K, uint32_t k_magic) {
  token_xent_kernel<LABELS, GRAD><<<grid, kRows, smem, st>>>(logits, labels, seq_len, pred_ids, d_logits, scratch, rows, L,
                                                             K, k_magic);
}

}  // namespace

extern "C" size_t ner_token_xent_scratch_floats(void) { return (size_t)kScratchHead + (size_t)ner_num_sms() * kCtasPerSm; }

extern "C" int ner_token_xent(const float* logits, const int32_t* labels, const int32_t* seq_len, int32_t* pred_ids,
                              float* loss, float* d_logits, float d_loss, float* scratch, int B, int L, int K,
                              ner_stream_t stream) {
  if (B < 0 || L < 1 || K < 1) return NER_ERR_INVALID_ARG;
  if (K > NER_MAX_TAGS) return NER_ERR_UNSUPPORTED;
  if ((long long)B * L > 0x7fffffffLL) return NER_ERR_UNSUPPORTED;
  if (B == 0) return NER_OK;
  if (!logits) return NER_ERR_INVALID_ARG;
  const bool with_labels = labels != nullptr;
  if (!with_labels && (loss || d_logits)) return NER_ERR_INVALID_ARG;      // no labels: argmax only
  if (with_labels && (!seq_len || !scratch)) return NER_ERR_INVALID_ARG;
  if (!pred_ids && !loss && !d_logits) return NER_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int rows = B * L;
  const int tiles = (rows + kRows - 1) / kRows;
  const int grid = min(tiles, ner_num_sms() * kCtasPerSm);
  const size_t smem = (size_t)kRows * (K | 1) * sizeof(float);
  const uint32_t k_magic = K > 1 ? 0xffffffffu / (uint32_t)K + 1u : 0u;
  if (!with_labels) {
    launch_main<false, false>(grid, smem, st, logits, nullptr, nullptr, pred_ids, nullptr, nullptr, rows, L, K, k_magic);
    return ner_launch_status();
  }
  token_count_kernel<<<1, 1024, 0, st>>>(seq_len, B, L, d_loss, scratch);
  if (d_logits)
    launch_main<true, true>(grid, smem, st, logits, labels, seq_len, pred_ids, d_logits, scratch, rows, L, K, k_magic);
  else
    launch_main<true, false>(grid, smem, st, logits, labels, seq_len, pred_ids, nullptr, scratch, rows, L, K, k_magic);
  if (loss) token_xent_final_kernel<<<1, 256, 0, st>>>(scratch, grid, loss);
  return ner_launch_status();
}
