// Softmax token heads of the bert_ce and bert_dice plugins (model/bert_ce.py, model/bert_dice.py + tools/loss.py): a masked
// token loss, its gradient and the first-maximum argmax, in one pass over the logits [B, L, K <= 32] f32 (sm_90a).  The
// softmax is never stored.  Two losses share the pass: cross-entropy (ner_token_xent) and the self-adjusting Dice loss
// (ner_token_dice); each is a row functor (XentLoss, DiceLoss) of the one kernel template.
//
// HBM-bound.  A CTA stages a tile of 256 rows (256 * K contiguous floats) through shared memory with coalesced loads, one
// thread then owns one row (the shared rows are laid out with an odd stride, K | 1, so the per-row reads are free of bank
// conflicts), and in TRAIN the gradient goes back through the same tile to coalesced stores.  The loss is reduced without
// float atomics: one partial per CTA, summed in index order by a one-CTA finaliser, so identical inputs give a
// bit-identical loss.  The token count N is summed on the device from seq_len before the main pass, which needs it to
// scale the gradient.
#include <cmath>

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

// A row functor adds the loss of one valid row z[0..K) (in shared memory; m = max, arg = first argmax, y = label) to acc
// and, when GRAD, overwrites z with scale * d loss / d z.  kGradTiles: shared tiles its GRAD pass needs; the row w[0..K)
// of the second one is free for per-class intermediates.

// Cross-entropy: logsumexp(z) - z[y]; gradient softmax - onehot.
struct XentLoss {
  static constexpr int kGradTiles = 1;
  template <bool GRAD>
  __device__ __forceinline__ void row(float* z, float* /*w*/, int K, int y, float m, int /*arg*/, float scale,
                                      float& acc) const {
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
  }
};

// Self-adjusting Dice loss (Li et al., ACL 2020) summed over the K classes; formula and gradient in ner_b200.h.  With
// e_k = exp(z_k - m) and s = sum e, u_k = 1 - p_k is computed as s_{-k} / s: s - e_k is accurate for k != arg (s_{-k} >= 1
// there), s_{-arg} is summed directly because s - e_arg cancels to 0 as soon as p_arg rounds to 1.
struct DiceLoss {
  static constexpr int kGradTiles = 2;
  float alpha, gamma;

  // Class k from e = e_k, sm = s_{-k}, inv_s = 1 / s: returns l_k and sets c = c_k, r = c_k / s_{-k} (0 when s_{-k} = 0,
  // where c_k is 0 too).
  __device__ __forceinline__ float term(float e, float sm, float inv_s, bool is_y, float& c, float& r) const {
    const float p = e * inv_s, u = sm * inv_s;
    const float ua = alpha == 1.f ? u : powf(u, alpha);    // powf(u, 0) = 1 at u = 0 too
    const float q = ua * p;
    const float inv = 1.f / (q + (is_y ? 1.f + gamma : gamma));
    c = (is_y ? -(2.f + gamma) : gamma) * inv * inv * p * ua * (u - alpha * p);
    r = sm > 0.f ? c / sm : 0.f;
    return (is_y ? 1.f - q : q) * inv;
  }

  // z holds e_k after the first loop, w the c_k of the second (GRAD).  R - r_arg is summed directly as well:
  // r_arg = c_arg / s_{-arg} grows like u_arg^(alpha-1) on a confident row and would swamp the other r_k in R.
  template <bool GRAD>
  __device__ __forceinline__ void row(float* z, float* w, int K, int y, float m, int arg, float scale, float& acc) const {
    float s = 0.f, s_arg = 0.f;
    for (int j = 0; j < K; ++j) {
      const float ej = expf(z[j] - m);
      s += ej;
      if (j != arg) s_arg += ej;
      z[j] = ej;
    }
    const float inv_s = 1.f / s;
    float l = 0.f, r_arg = 0.f, R_arg = 0.f, c, r;
    for (int j = 0; j < K; ++j) {
      const float ej = z[j];
      l += term(ej, j == arg ? s_arg : s - ej, inv_s, j == y, c, r);
      if (GRAD) w[j] = c;
      if (j == arg) r_arg = r;
      else R_arg += r;
    }
    if (GRAD) {
      const float R = r_arg + R_arg;
      for (int j = 0; j < K; ++j) {
        const float ej = z[j], cj = w[j];
        const float rest = j == arg ? R_arg : R - cj / (s - ej);         // R - r_j; s - e_j >= e_arg = 1
        z[j] = scale * (cj - ej * rest);
      }
    }
    acc += l;
  }
};

// LABELS: labels / seq_len present, per-CTA loss partials written to scratch.  GRAD: d_logits written (every row).
template <class Loss, bool LABELS, bool GRAD>
__global__ void __launch_bounds__(kRows)
token_head_kernel(const float* __restrict__ logits, const int32_t* __restrict__ labels, const int32_t* __restrict__ seq_len,
                  int32_t* __restrict__ pred_ids, float* __restrict__ d_logits, float* __restrict__ scratch, int rows,
                  int L, int K, uint32_t k_magic, Loss fn) {
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
          fn.template row<GRAD>(z, z + kRows * Kp, K, __ldcs(labels + row), m, arg, scale, acc);
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
token_loss_final_kernel(const float* __restrict__ scratch, int n_part, float* __restrict__ loss) {
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

template <class Loss, bool LABELS, bool GRAD>
void launch_main(const Loss& fn, int grid, cudaStream_t st, const float* logits, const int32_t* labels,
                 const int32_t* seq_len, int32_t* pred_ids, float* d_logits, float* scratch, int rows, int L, int K,
                 uint32_t k_magic) {
  const size_t smem = (size_t)(GRAD ? Loss::kGradTiles : 1) * kRows * (K | 1) * sizeof(float);
  if (smem > 48 * 1024)       // above the default dynamic shared-memory limit (two tiles at K > 23)
    cudaFuncSetAttribute(token_head_kernel<Loss, LABELS, GRAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  token_head_kernel<Loss, LABELS, GRAD><<<grid, kRows, smem, st>>>(logits, labels, seq_len, pred_ids, d_logits, scratch,
                                                                   rows, L, K, k_magic, fn);
}

// Both entry points: validation in the order ner_b200.h documents, then the launches.  need_labels: the loss has no
// argmax-only mode (ner_token_dice).
template <class Loss>
int token_head(const Loss& fn, bool need_labels, const float* logits, const int32_t* labels, const int32_t* seq_len,
               int32_t* pred_ids, float* loss, float* d_logits, float d_loss, float* scratch, int B, int L, int K,
               ner_stream_t stream) {
  if (B < 0 || L < 1 || K < 1) return NER_ERR_INVALID_ARG;
  if (K > NER_MAX_TAGS) return NER_ERR_UNSUPPORTED;
  if ((long long)B * L > 0x7fffffffLL) return NER_ERR_UNSUPPORTED;
  if (B == 0) return NER_OK;
  if (!logits) return NER_ERR_INVALID_ARG;
  const bool with_labels = labels != nullptr;
  if (need_labels && !with_labels) return NER_ERR_INVALID_ARG;
  if (!with_labels && (loss || d_logits)) return NER_ERR_INVALID_ARG;      // no labels: argmax only
  if (with_labels && (!seq_len || !scratch)) return NER_ERR_INVALID_ARG;
  if (!pred_ids && !loss && !d_logits) return NER_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int rows = B * L;
  const int tiles = (rows + kRows - 1) / kRows;
  const int grid = min(tiles, ner_num_sms() * kCtasPerSm);
  const uint32_t k_magic = K > 1 ? 0xffffffffu / (uint32_t)K + 1u : 0u;
  if (!with_labels) {
    launch_main<XentLoss, false, false>(XentLoss{}, grid, st, logits, nullptr, nullptr, pred_ids, nullptr, nullptr,
                                        rows, L, K, k_magic);
    return ner_launch_status();
  }
  token_count_kernel<<<1, 1024, 0, st>>>(seq_len, B, L, d_loss, scratch);
  if (d_logits)
    launch_main<Loss, true, true>(fn, grid, st, logits, labels, seq_len, pred_ids, d_logits, scratch, rows, L, K,
                                  k_magic);
  else
    launch_main<Loss, true, false>(fn, grid, st, logits, labels, seq_len, pred_ids, nullptr, scratch, rows, L, K,
                                   k_magic);
  if (loss) token_loss_final_kernel<<<1, 256, 0, st>>>(scratch, grid, loss);
  return ner_launch_status();
}

}  // namespace

extern "C" size_t ner_token_xent_scratch_floats(void) { return (size_t)kScratchHead + (size_t)ner_num_sms() * kCtasPerSm; }

extern "C" int ner_token_xent(const float* logits, const int32_t* labels, const int32_t* seq_len, int32_t* pred_ids,
                              float* loss, float* d_logits, float d_loss, float* scratch, int B, int L, int K,
                              ner_stream_t stream) {
  return token_head(XentLoss{}, false, logits, labels, seq_len, pred_ids, loss, d_logits, d_loss, scratch, B, L, K, stream);
}

extern "C" int ner_token_dice(const float* logits, const int32_t* labels, const int32_t* seq_len, int32_t* pred_ids,
                              float* loss, float* d_logits, float d_loss, float alpha, float gamma, float* scratch, int B,
                              int L, int K, ner_stream_t stream) {
  if (!(std::isfinite(alpha) && alpha >= 0.f && std::isfinite(gamma) && gamma > 0.f)) return NER_ERR_INVALID_ARG;
  return token_head(DiceLoss{alpha, gamma}, true, logits, labels, seq_len, pred_ids, loss, d_logits, d_loss, scratch, B, L,
                    K, stream);
}
