// Span-pointer MRC NER of the bert_mrc_span plugin (model/bert_mrc_span.py; Li et al., "A Unified MRC Framework for Named
// Entity Recognition", ACL 2020): the match head over every (start i, end j) pair of a query/context pair p,
//   z[p,i,j] = sum_k w2[k] * drop(GELU_tanh(U[p,i,k] + V[p,j,k] + b1[k])) + b2,   [U | V] = rows . [W1[0:H] | W1[H:2H]]
// its targets, its BCE loss and gradient, and the PREDICT decode (starts x ends -> spans -> greedy tag projection).
//
// The match head is not a GEMM (the GELU sits between the two layers) and is bound by the tanh unit (MUFU, 16 / clk / SM)
// and the FP32 pipe, not the tensor cores.  Forward: a CTA owns a 32 x 32 (i, j) tile of one pair, stages 32-wide k-chunks of
// U and V rows in shared memory (cp.async, double buffered) and every thread accumulates a 4 x 4 register micro-tile over k
// in a fixed order; tiles below the diagonal or past the pair's length are skipped.  Backward: the activations are
// recomputed; a CTA owns 32 k-columns of one pair and each warp a row i (dU: sum over j) or a column j (dV: sum over i), so
// every output element has one owner and the k-sums and pair-sums are per-CTA partials added in index order (no float
// atomics).  The decode runs the forward tile kernel on the compacted start x end lists only, so PREDICT never evaluates the
// whole triangle unless every position is a start and an end.
#include "common.cuh"
#include "span_common.cuh"

namespace {

using nerdev::cp_async16;
using nerdev::cp_async_commit;
using nerdev::cp_async_wait;
using nerdev::hash3;
using nerdev::keep_threshold;
using namespace span;

constexpr int kMaxTypes = 32;
constexpr int kMaxLen = 511;      // the pair bound: a key packs i and j in 9 bits each
static_assert(kMaxLen <= kDecodeRows, "the decode holds a whole pair in shared memory");
constexpr int kMaxInter = 4096;
constexpr int kTile = 32;         // i x j tile of the match kernel
constexpr int kKc = 32;           // k-chunk staged per step
constexpr int kLd = kKc + 4;      // smem row stride (floats): 16-byte rows, conflict-free float4 reads of rows r + 8b
constexpr int kTileThreads = 64;  // 8 x 8 threads, 4 x 4 outputs each
constexpr int kRowThreads = 256;  // backward: 8 warps x 32 k-columns
constexpr int kRowWarps = kRowThreads / 32;

constexpr float kC0 = 0.7978845608028654f;            // sqrt(2 / pi)
constexpr float kC1 = 0.7978845608028654f * 0.044715f;

__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// 0.5 * w * x * (1 + tanh(c0 x + c1 x^3)) = w * GELU_tanh(x); hw = 0.5 * w (times the dropout scale)
__device__ __forceinline__ float gelu_w(float x, float hw) {
  const float x2 = __fmul_rn(x, x);
  const float t = tanh_approx(__fmul_rn(x, __fmaf_rn(kC1, x2, kC0)));
  const float hx = __fmul_rn(x, hw);
  return __fmaf_rn(hx, t, hx);
}

// keep decision of element (p, i, j, k): shared by the forward and the backward
__device__ __forceinline__ bool span_keep(uint32_t seed_lo, uint32_t seed_hi, int p, int i, int j, int k, int L, int I,
                                          uint32_t thr) {
  return hash3(seed_lo, seed_hi ^ (uint32_t)(p * L + i), (uint32_t)(j * I + k)) < thr;
}

struct TileSmem;
__device__ __forceinline__ void stage_chunk(TileSmem& s, const float* __restrict__ uv, int ld, const float* __restrict__ b1,
                                            const float* __restrict__ w2, int p, int L, int I, int c, int buf, int tid);

struct TileSmem {
  float u[2][kTile][kLd];
  float v[2][kTile][kLd];
  float b1[2][kKc];
  float w2[2][kKc];
  int32_t rowi[kTile];
  int32_t rowj[kTile];
  int32_t end_of[kTile];
  float red[kTileThreads];
};

// U rows rowi[], V rows rowj[], b1 and w2 of k-chunk c -> buffer buf (one cp.async group)
__device__ __forceinline__ void stage_chunk(TileSmem& s, const float* __restrict__ uv, int ld, const float* __restrict__ b1,
                                            const float* __restrict__ w2, int p, int L, int I, int c, int buf, int tid) {
  const int k0 = c * kKc;
  for (int idx = tid; idx < 2 * kTile * (kKc / 4); idx += kTileThreads) {
    const int side = idx >> 8, r = (idx >> 3) & 31, q = idx & 7;
    const int row = side ? s.rowj[r] : s.rowi[r];
    const float* src = uv + ((size_t)p * L + row) * ld + (side ? I : 0) + k0 + q * 4;
    cp_async16(side ? &s.v[buf][r][q * 4] : &s.u[buf][r][q * 4], src);
  }
  if (tid < kKc / 4) cp_async16(&s.b1[buf][tid * 4], b1 + k0 + tid * 4);
  else if (tid < kKc / 2) cp_async16(&s.w2[buf][(tid - kKc / 4) * 4], w2 + k0 + (tid - kKc / 4) * 4);
  cp_async_commit();
}

// z over one 32 x 32 tile of pair p.
//   kCompact = false (ner_mrc_span_match_fwd): rows i0 + r, columns j0 + c; z is written at every (i, j) < L of the tile
//     (0 off the candidates 1 <= i <= j <= len - 2), and the tile's BCE sum goes to partial[] when it is not NULL.
//   kCompact = true (ner_mrc_span_decode): rows S[a0 + r], columns E[b0 + c] of the pair's start / end lists; z is written
//     at (S[a], E[b]) for S[a] <= E[b] only.  Same per-element arithmetic and k order, so z is bit-identical to the
//     forward's at keep = 1.
template <bool kDrop, bool kCompact>
__global__ void __launch_bounds__(kTileThreads)
span_tile_kernel(const float* __restrict__ uv, int ld, const float* __restrict__ b1, const float* __restrict__ w2,
                 const float* __restrict__ b2, const int32_t* __restrict__ seq_len, int T,
                 const int32_t* __restrict__ span_end, const int32_t* __restrict__ lists, const int32_t* __restrict__ counts,
                 int L, int I, float keep, uint64_t seed, float* __restrict__ z, float* __restrict__ partial) {
  __shared__ __align__(16) TileSmem s;
  const int tid = threadIdx.x, tx = tid & 7, ty = tid >> 3;
  const int p = blockIdx.y;
  const int nt = (L + kTile - 1) / kTile;
  const int ti = blockIdx.x / nt, tj = blockIdx.x - ti * nt;
  const int len = clamp_len(__ldg(seq_len + p / T), L), m = len - 2;
  const int i0 = ti * kTile, j0 = tj * kTile;
  int ns = 0, ne = 0;
  bool need;
  if (kCompact) {
    ns = __ldg(counts + 2 * p);
    ne = __ldg(counts + 2 * p + 1);
    need = i0 < ns && j0 < ne &&
           __ldg(lists + (size_t)p * 2 * L + i0) <= __ldg(lists + (size_t)p * 2 * L + L + min(j0 + kTile - 1, ne - 1));
  } else {
    need = j0 <= m && max(i0, 1) <= min(j0 + kTile - 1, m);
  }
  if (!need) {
    if (!kCompact) {
      for (int e = tid; e < kTile * kTile; e += kTileThreads) {
        const int i = i0 + (e >> 5), j = j0 + (e & 31);
        if (i < L && j < L) z[((size_t)p * L + i) * L + j] = 0.f;
      }
      if (partial != nullptr && tid == 0) partial[(size_t)p * gridDim.x + blockIdx.x] = 0.f;
    }
    return;
  }
  if (tid < kTile) {
    if (kCompact) {
      s.rowi[tid] = __ldg(lists + (size_t)p * 2 * L + min(i0 + tid, ns - 1));
      s.rowj[tid] = __ldg(lists + (size_t)p * 2 * L + L + min(j0 + tid, ne - 1));
    } else {
      s.rowi[tid] = min(i0 + tid, L - 1);
      s.rowj[tid] = min(j0 + tid, L - 1);
      s.end_of[tid] = span_end != nullptr ? __ldg(span_end + (size_t)p * L + min(i0 + tid, L - 1)) : -1;
    }
  }
  __syncthreads();

  const float inv_keep = kDrop ? 1.f / keep : 1.f;
  const uint32_t thr = keep_threshold(keep);
  const uint32_t seed_lo = (uint32_t)seed, seed_hi = (uint32_t)(seed >> 32);
  int gi[4] = {0, 0, 0, 0}, gj[4] = {0, 0, 0, 0};   // positions of the thread's rows / columns (dropout hash)
  if (kDrop) {
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      gi[a] = s.rowi[ty + 8 * a];
      gj[a] = s.rowj[tx + 8 * a];
    }
  }
  float acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;

  const int nk = I / kKc;
  stage_chunk(s, uv, ld, b1, w2, p, L, I, 0, 0, tid);
  for (int c = 0; c < nk; ++c) {
    const int buf = c & 1;
    if (c + 1 < nk) {
      stage_chunk(s, uv, ld, b1, w2, p, L, I, c + 1, buf ^ 1, tid);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
#pragma unroll 1
    for (int kk = 0; kk < kKc; kk += 4) {
      const float4 bb = *reinterpret_cast<const float4*>(&s.b1[buf][kk]);
      const float4 ww = *reinterpret_cast<const float4*>(&s.w2[buf][kk]);
      float4 ua[4], vb[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) ua[a] = *reinterpret_cast<const float4*>(&s.u[buf][ty + 8 * a][kk]);
#pragma unroll
      for (int b = 0; b < 4; ++b) vb[b] = *reinterpret_cast<const float4*>(&s.v[buf][tx + 8 * b][kk]);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float bq = q == 0 ? bb.x : q == 1 ? bb.y : q == 2 ? bb.z : bb.w;
        const float hw = 0.5f * (q == 0 ? ww.x : q == 1 ? ww.y : q == 2 ? ww.z : ww.w);
        const float hwk = __fmul_rn(hw, inv_keep);
        const int k = c * kKc + kk + q;
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          const float uq = __fadd_rn(q == 0 ? ua[a].x : q == 1 ? ua[a].y : q == 2 ? ua[a].z : ua[a].w, bq);
#pragma unroll
          for (int b = 0; b < 4; ++b) {
            const float vq = q == 0 ? vb[b].x : q == 1 ? vb[b].y : q == 2 ? vb[b].z : vb[b].w;
            float h = hw;
            if (kDrop) h = span_keep(seed_lo, seed_hi, p, gi[a], gj[b], k, L, I, thr) ? hwk : 0.f;
            acc[a][b] = __fadd_rn(acc[a][b], gelu_w(__fadd_rn(uq, vq), h));
          }
        }
      }
    }
    __syncthreads();
  }

  const float bias2 = __ldg(b2);
  float lsum = 0.f;
#pragma unroll
  for (int a = 0; a < 4; ++a) {
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const float zz = __fadd_rn(acc[a][b], bias2);
      if (kCompact) {
        const int ri = s.rowi[ty + 8 * a], rj = s.rowj[tx + 8 * b];
        if (i0 + ty + 8 * a < ns && j0 + tx + 8 * b < ne && ri <= rj) z[((size_t)p * L + ri) * L + rj] = zz;
      } else {
        const int i = i0 + ty + 8 * a, j = j0 + tx + 8 * b;
        if (i < L && j < L) {
          const bool cand = i >= 1 && i <= j && j <= m;
          z[((size_t)p * L + i) * L + j] = cand ? zz : 0.f;
          if (cand && partial != nullptr) {
            const float y = s.end_of[ty + 8 * a] == j ? 1.f : 0.f;
            lsum += fmaxf(zz, 0.f) - zz * y + log1pf(expf(-fabsf(zz)));
          }
        }
      }
    }
  }
  if (!kCompact && partial != nullptr) {
    s.red[tid] = lsum;
    __syncthreads();
    if (tid == 0) {
      float t = 0.f;
      for (int e = 0; e < kTileThreads; ++e) t += s.red[e];
      partial[(size_t)p * gridDim.x + blockIdx.x] = t;
    }
  }
}

// Candidates of the batch: sum over pairs of m (m + 1) / 2, m = len - 2 (1 <= i <= j <= len - 2).
__device__ __forceinline__ long long pair_candidates(int len) {
  const long long m = len - 2;
  return m > 0 ? m * (m + 1) / 2 : 0;
}

// loss = sum of the tile partials (index order) / candidate count, 0 without candidates.  One CTA.
__global__ void __launch_bounds__(1024)
span_loss_kernel(const float* __restrict__ partial, int n_part, const int32_t* __restrict__ seq_len, int P, int L,
                 float* __restrict__ loss) {
  __shared__ double s_sum[1024];
  __shared__ long long s_cnt[1024];
  const int tid = threadIdx.x;
  double acc = 0.0;
  for (int e = tid; e < n_part; e += 1024) acc += (double)__ldg(partial + e);
  long long cnt = 0;
  for (int q = tid; q < P; q += 1024) cnt += pair_candidates(clamp_len(__ldg(seq_len + q), L));
  s_sum[tid] = acc;
  s_cnt[tid] = cnt;
  __syncthreads();
  for (int w = 512; w > 0; w >>= 1) {
    if (tid < w) {
      s_sum[tid] += s_sum[tid + w];
      s_cnt[tid] += s_cnt[tid + w];
    }
    __syncthreads();
  }
  if (tid == 0) *loss = s_cnt[0] > 0 ? (float)(s_sum[0] / (double)s_cnt[0]) : 0.f;
}

// Backward, one pass per side.  kCols = false: warp row i, sum over j in [i, m] -> dU[p,i,:] (and the per-pair partials of
// dw2, db1, db2); kCols = true: warp column j, sum over i in [1, j] -> dV[p,j,:].  dz = d_loss / N * (sigmoid(z) - y).
template <bool kCols, bool kDrop>
__global__ void __launch_bounds__(kRowThreads)
span_bwd_rows_kernel(const float* __restrict__ uv, int ld, const float* __restrict__ z, const float* __restrict__ b1,
                     const float* __restrict__ w2, const int32_t* __restrict__ seq_len,
                     const int32_t* __restrict__ span_end, int P, int L, int I, float d_loss, float keep, uint64_t seed,
                     float* __restrict__ d_uv, float* __restrict__ part_w2, float* __restrict__ part_b1,
                     float* __restrict__ part_b2) {
  extern __shared__ float smem[];
  float* sx = smem;                        // [L][32]: the other side's rows of this k-chunk
  float* sdz = smem + (size_t)L * 32;      // [8][L]: dz of the warp's current row / column
  __shared__ long long s_n;
  __shared__ float s_w[kRowWarps][32], s_b[kRowWarps][32], s_b2[kRowWarps];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int p = blockIdx.y, kc = blockIdx.x, k = kc * 32 + lane;
  const int len = clamp_len(__ldg(seq_len + p), L), m = len - 2;
  const size_t ld2 = (size_t)2 * I;
  if (warp == 0) {
    long long n = 0;
    for (int q = lane; q < P; q += 32) n += pair_candidates(clamp_len(__ldg(seq_len + q), L));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
    if (lane == 0) s_n = n;
  }
  const int other = kCols ? 0 : I;
  if (m >= 1) {
    for (int idx = tid; idx < (m + 1) * 32; idx += kRowThreads) {
      const int r = idx >> 5, c = idx & 31;
      sx[idx] = __ldg(uv + ((size_t)p * L + r) * ld + other + kc * 32 + c);
    }
  }
  __syncthreads();
  const float inv = s_n > 0 ? d_loss / (float)s_n : 0.f;
  const float w2k = __ldg(w2 + k), b1k = __ldg(b1 + k);
  const float inv_keep = kDrop ? 1.f / keep : 1.f;
  const uint32_t thr = keep_threshold(keep);
  const uint32_t seed_lo = (uint32_t)seed, seed_hi = (uint32_t)(seed >> 32);
  float dw2_acc = 0.f, db1_acc = 0.f, db2_acc = 0.f;
  float* sd = sdz + (size_t)warp * L;
  for (int r = 1 + warp; r <= m; r += kRowWarps) {
    const int o_lo = kCols ? 1 : r, o_hi = kCols ? r : m;
    const int se = kCols ? -1 : __ldg(span_end + (size_t)p * L + r);
    for (int o = o_lo + lane; o <= o_hi; o += 32) {
      const float zz = kCols ? __ldg(z + ((size_t)p * L + o) * L + r) : __ldg(z + ((size_t)p * L + r) * L + o);
      const bool y = kCols ? __ldg(span_end + (size_t)p * L + o) == r : se == o;
      const float d = (1.f / (1.f + expf(-zz)) - (y ? 1.f : 0.f)) * inv;
      sd[o] = d;
      if (!kCols) db2_acc += d;
    }
    __syncwarp();
    const float own = __ldg(uv + ((size_t)p * L + r) * ld + (kCols ? I : 0) + k) + b1k;
    float acc = 0.f;
    for (int o = o_lo; o <= o_hi; ++o) {
      const float x = own + sx[o * 32 + lane];
      const float d = sd[o];
      float mk = 1.f;
      if (kDrop) mk = span_keep(seed_lo, seed_hi, p, kCols ? o : r, kCols ? r : o, k, L, I, thr) ? inv_keep : 0.f;
      const float x2 = x * x;
      const float t = tanh_approx(x * fmaf(kC1, x2, kC0));
      const float ht = fmaf(0.5f, t, 0.5f);                           // 0.5 (1 + t)
      const float sech2 = fmaf(-t, t, 1.f);
      const float gp = fmaf(0.5f * x * sech2, fmaf(3.f * kC1, x2, kC0), ht);   // GELU'(x)
      const float dm = d * mk;
      acc = fmaf(dm * w2k, gp, acc);
      if (!kCols) dw2_acc = fmaf(dm, x * ht, dw2_acc);
    }
    d_uv[((size_t)p * L + r) * ld2 + (kCols ? I : 0) + k] = acc;
    if (!kCols) db1_acc += acc;
    __syncwarp();
  }
  for (int r = warp; r < L; r += kRowWarps)
    if (r < 1 || r > m) d_uv[((size_t)p * L + r) * ld2 + (kCols ? I : 0) + k] = 0.f;
  if (!kCols) {
    s_w[warp][lane] = dw2_acc;
    s_b[warp][lane] = db1_acc;
    const float b2w = nerdev::warp_sum(db2_acc);
    if (lane == 0) s_b2[warp] = b2w;
    __syncthreads();
    if (warp == 0) {
      float sw = 0.f, sb = 0.f;
      for (int w = 0; w < kRowWarps; ++w) {
        sw += s_w[w][lane];
        sb += s_b[w][lane];
      }
      part_w2[(size_t)p * I + k] = sw;
      part_b1[(size_t)p * I + k] = sb;
      if (kc == 0 && lane == 0) {
        float t = 0.f;
        for (int w = 0; w < kRowWarps; ++w) t += s_b2[w];
        part_b2[p] = t;
      }
    }
  }
}

// d_w2[k], d_b1[k] = sum over pairs of the partials (pair order); d_b2 = sum of the pair partials.
__global__ void __launch_bounds__(256)
span_bwd_reduce_kernel(const float* __restrict__ part_w2, const float* __restrict__ part_b1,
                       const float* __restrict__ part_b2, int P, int I, float* __restrict__ d_w2,
                       float* __restrict__ d_b1, float* __restrict__ d_b2) {
  const int k = blockIdx.x * 256 + threadIdx.x;
  if (k < I) {
    float sw = 0.f, sb = 0.f;
    for (int p = 0; p < P; ++p) {
      sw += __ldg(part_w2 + (size_t)p * I + k);
      sb += __ldg(part_b1 + (size_t)p * I + k);
    }
    d_w2[k] = sw;
    d_b1[k] = sb;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    float t = 0.f;
    for (int p = 0; p < P; ++p) t += __ldg(part_b2 + p);
    *d_b2 = t;
  }
}

__device__ __forceinline__ bool first_argmax_is_1(const float* __restrict__ lg, size_t row) {
  return __ldg(lg + 2 * row + 1) > __ldg(lg + 2 * row);
}

// Targets: one CTA per pair.  start_y[s] = [y_s = 1]; span_end[s] = r(s) (the last j >= s with y[s+1..j] all 2, j < len) for
// a start, else -1; end_y[j] = [j = r(s) for some start s].  Every start closes before the next one, so each j has at most
// one writer.
__global__ void __launch_bounds__(128)
span_targets_kernel(const int32_t* __restrict__ labels, const int32_t* __restrict__ seq_len, int L,
                    int32_t* __restrict__ start_y, int32_t* __restrict__ end_y, int32_t* __restrict__ span_end) {
  __shared__ int32_t y[kMaxLen + 1];
  const int p = blockIdx.x;
  const int len = clamp_len(__ldg(seq_len + p), L);
  const size_t base = (size_t)p * L;
  for (int s = threadIdx.x; s < L; s += 128) {
    y[s] = s < len ? __ldg(labels + base + s) : 0;
    end_y[base + s] = 0;
  }
  __syncthreads();
  for (int s = threadIdx.x; s < L; s += 128) {
    const bool st = s < len && y[s] == 1;
    start_y[base + s] = st ? 1 : 0;
    span_end[base + s] = st ? run_end(y, s, len, 2) : -1;
  }
  __syncthreads();
  for (int s = threadIdx.x; s < L; s += 128) {
    const int r = span_end[base + s];
    if (r >= 0) end_y[base + r] = 1;
  }
}

// Decode 1: the ascending start / end lists of every pair (positions 1..len-2 whose logits' first argmax is 1).
__global__ void __launch_bounds__(128)
span_flags_kernel(const float* __restrict__ start_logits, const float* __restrict__ end_logits,
                  const int32_t* __restrict__ seq_len, int T, int L, int32_t* __restrict__ lists,
                  int32_t* __restrict__ counts) {
  __shared__ int s_wc[2][4];
  const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int m = clamp_len(__ldg(seq_len + p / T), L) - 2;
  int base[2] = {0, 0};
  for (int c0 = 0; c0 < L; c0 += 128) {
    const int pos = c0 + tid;
    const bool in = pos >= 1 && pos <= m;
    const size_t row = (size_t)p * L + pos;
    bool f[2];
    f[0] = in && first_argmax_is_1(start_logits, row);
    f[1] = in && first_argmax_is_1(end_logits, row);
    unsigned bal[2];
#pragma unroll
    for (int sd = 0; sd < 2; ++sd) {
      bal[sd] = __ballot_sync(0xffffffffu, f[sd]);
      if (lane == 0) s_wc[sd][warp] = __popc(bal[sd]);
    }
    __syncthreads();
#pragma unroll
    for (int sd = 0; sd < 2; ++sd) {
      int off = base[sd], tot = 0;
      for (int w = 0; w < 4; ++w) {
        if (w < warp) off += s_wc[sd][w];
        tot += s_wc[sd][w];
      }
      if (f[sd]) lists[(size_t)p * 2 * L + sd * L + off + __popc(bal[sd] & ((1u << lane) - 1u))] = pos;
      base[sd] += tot;
    }
    __syncthreads();
  }
  if (tid == 0) {
    counts[2 * p] = base[0];
    counts[2 * p + 1] = base[1];
  }
}

// Candidates of the decode: the types t with position i a start and j an end of t.
struct StartEndCandidates {
  const uint32_t* smask;
  const uint32_t* emask;
  __device__ __forceinline__ bool live(int i) const { return smask[i] != 0; }
  template <class F>
  __device__ __forceinline__ void for_each(int i, int j, F&& f) const {
    uint32_t bits = smask[i] & emask[j];
    while (bits) {
      const int t = __ffs(bits) - 1;
      bits &= bits - 1;
      if (!f(t)) return;
    }
  }
};

// Decode 3: one CTA per sentence: the start / end bits of every position, then span_common.cuh's greedy decode.
__global__ void __launch_bounds__(kDecodeThreads)
span_decode_kernel(const float* __restrict__ start_logits, const float* __restrict__ end_logits,
                   const float* __restrict__ zf, const int32_t* __restrict__ seq_len, const int32_t* __restrict__ type_tag,
                   int T, int L, int o_id, int cls_id, int sep_id, int cap, int32_t* __restrict__ pred_ids,
                   int32_t* __restrict__ spans, float* __restrict__ probs, int32_t* __restrict__ span_counts) {
  __shared__ uint32_t smask[kMaxLen + 1], emask[kMaxLen + 1];
  const int b = blockIdx.x;
  const int len = clamp_len(__ldg(seq_len + b), L), m = len - 2;
  for (int s = threadIdx.x; s < L; s += kDecodeThreads) {
    uint32_t sm = 0, em = 0;
    if (s >= 1 && s <= m) {
#pragma unroll 1
      for (int t = 0; t < T; ++t) {
        const size_t row = ((size_t)b * T + t) * L + s;
        sm |= (first_argmax_is_1(start_logits, row) ? 1u : 0u) << t;
        em |= (first_argmax_is_1(end_logits, row) ? 1u : 0u) << t;
      }
    }
    smask[s] = sm;
    emask[s] = em;
  }
  greedy_span_decode(StartEndCandidates{smask, emask}, zf, T, L, len, type_tag, o_id, cls_id, sep_id, cap, pred_ids,
                     spans, probs, span_counts);
}

// shared checks of the match entry points: 0 or the status to return
int check_match_shape(int P, int L, int I, int ld_uv) {
  if (P < 0 || L < 1 || I < 1 || ld_uv < 1) return NER_ERR_INVALID_ARG;
  if (L > kMaxLen || I % 32 != 0 || I > kMaxInter) return NER_ERR_UNSUPPORTED;
  if (ld_uv < 2 * I || ld_uv % 4 != 0) return NER_ERR_INVALID_ARG;
  if ((long long)P * L * L >= 0x7fffffffLL) return NER_ERR_UNSUPPORTED;
  return NER_OK;
}

int tile_count(int L) {
  const int nt = (L + kTile - 1) / kTile;
  return nt * nt;
}

template <typename K>
int set_smem(K kern, size_t bytes) {
  if (bytes <= 48 * 1024) return NER_OK;
  if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) != cudaSuccess)
    return ner_launch_status();
  return NER_OK;
}

}  // namespace

extern "C" int ner_mrc_span_targets(const int32_t* pair_labels, const int32_t* pair_seq_len, int P, int L, int32_t* start_y,
                                    int32_t* end_y, int32_t* span_end, ner_stream_t stream) {
  if (P < 0 || L < 1) return NER_ERR_INVALID_ARG;
  if (L > kMaxLen) return NER_ERR_UNSUPPORTED;
  if ((long long)P * L >= 0x7fffffffLL) return NER_ERR_UNSUPPORTED;
  if (P == 0) return NER_OK;
  if (!pair_labels || !pair_seq_len || !start_y || !end_y || !span_end) return NER_ERR_INVALID_ARG;
  span_targets_kernel<<<P, 128, 0, static_cast<cudaStream_t>(stream)>>>(pair_labels, pair_seq_len, L, start_y, end_y,
                                                                         span_end);
  return ner_launch_status();
}

extern "C" size_t ner_mrc_span_match_fwd_workspace_bytes(int P, int L) {
  if (P <= 0 || L < 1 || L > kMaxLen) return 0;
  return (size_t)P * tile_count(L) * sizeof(float);
}

extern "C" int ner_mrc_span_match_fwd(const float* uv, int ld_uv, const float* b1, const float* w2, const float* b2,
                                      const int32_t* pair_seq_len, const int32_t* span_end, int P, int L, int I,
                                      float keep_prob, uint64_t seed, float* z, float* loss, void* workspace,
                                      size_t workspace_bytes, ner_stream_t stream) {
  const int shape = check_match_shape(P, L, I, ld_uv);
  if (shape != NER_OK) return shape;
  if (!(keep_prob > 0.f && keep_prob <= 1.f)) return NER_ERR_INVALID_ARG;
  if (P == 0) return NER_OK;
  if (!uv || !b1 || !w2 || !b2 || !pair_seq_len || !z) return NER_ERR_INVALID_ARG;
  if (!aligned16(uv) || !aligned16(b1) || !aligned16(w2)) return NER_ERR_INVALID_ARG;
  if (loss && !span_end) return NER_ERR_INVALID_ARG;
  if (loss && (!workspace || workspace_bytes < ner_mrc_span_match_fwd_workspace_bytes(P, L))) return NER_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* partial = loss ? static_cast<float*>(workspace) : nullptr;
  const dim3 grid(tile_count(L), P);
  if (keep_prob < 1.f)
    span_tile_kernel<true, false><<<grid, kTileThreads, 0, st>>>(uv, ld_uv, b1, w2, b2, pair_seq_len, 1, span_end, nullptr,
                                                                  nullptr, L, I, keep_prob, seed, z, partial);
  else
    span_tile_kernel<false, false><<<grid, kTileThreads, 0, st>>>(uv, ld_uv, b1, w2, b2, pair_seq_len, 1, span_end, nullptr,
                                                                   nullptr, L, I, 1.f, seed, z, partial);
  if (loss) {
    const int rc = ner_launch_status();
    if (rc != NER_OK) return rc;
    span_loss_kernel<<<1, 1024, 0, st>>>(partial, P * tile_count(L), pair_seq_len, P, L, loss);
  }
  return ner_launch_status();
}

extern "C" size_t ner_mrc_span_match_bwd_workspace_bytes(int P, int I) {
  if (P <= 0 || I < 1) return 0;
  return ((size_t)2 * P * I + P) * sizeof(float);
}

extern "C" int ner_mrc_span_match_bwd(const float* uv, int ld_uv, const float* z, const float* b1, const float* w2,
                                      const int32_t* pair_seq_len, const int32_t* span_end, int P, int L, int I,
                                      float d_loss, float keep_prob, uint64_t seed, float* d_uv, float* d_b1, float* d_w2,
                                      float* d_b2, void* workspace, size_t workspace_bytes, ner_stream_t stream) {
  const int shape = check_match_shape(P, L, I, ld_uv);
  if (shape != NER_OK) return shape;
  if (!(keep_prob > 0.f && keep_prob <= 1.f)) return NER_ERR_INVALID_ARG;
  if (P == 0) return NER_OK;
  if (!uv || !z || !b1 || !w2 || !pair_seq_len || !span_end || !d_uv || !d_b1 || !d_w2 || !d_b2)
    return NER_ERR_INVALID_ARG;
  if (!workspace || workspace_bytes < ner_mrc_span_match_bwd_workspace_bytes(P, I)) return NER_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* part_w2 = static_cast<float*>(workspace);
  float* part_b1 = part_w2 + (size_t)P * I;
  float* part_b2 = part_b1 + (size_t)P * I;
  const size_t smem = ((size_t)L * 32 + (size_t)kRowWarps * L) * sizeof(float);
  const dim3 grid(I / 32, P);
  const bool drop = keep_prob < 1.f;
  auto rows = drop ? span_bwd_rows_kernel<false, true> : span_bwd_rows_kernel<false, false>;
  auto cols = drop ? span_bwd_rows_kernel<true, true> : span_bwd_rows_kernel<true, false>;
  int rc = set_smem(rows, smem);
  if (rc == NER_OK) rc = set_smem(cols, smem);
  if (rc != NER_OK) return rc;
  rows<<<grid, kRowThreads, smem, st>>>(uv, ld_uv, z, b1, w2, pair_seq_len, span_end, P, L, I, d_loss, keep_prob, seed, d_uv,
                                        part_w2, part_b1, part_b2);
  if ((rc = ner_launch_status()) != NER_OK) return rc;
  cols<<<grid, kRowThreads, smem, st>>>(uv, ld_uv, z, b1, w2, pair_seq_len, span_end, P, L, I, d_loss, keep_prob, seed, d_uv,
                                        part_w2, part_b1, part_b2);
  if ((rc = ner_launch_status()) != NER_OK) return rc;
  span_bwd_reduce_kernel<<<(I + 255) / 256, 256, 0, st>>>(part_w2, part_b1, part_b2, P, I, d_w2, d_b1, d_b2);
  return ner_launch_status();
}

extern "C" size_t ner_mrc_span_decode_workspace_bytes(int P, int L) {
  if (P <= 0 || L < 1 || L > kMaxLen) return 0;
  return ((size_t)P * L * L + (size_t)P * 2 * L + (size_t)P * 2) * 4;
}

extern "C" int ner_mrc_span_decode(const float* start_logits, const float* end_logits, const float* uv, int ld_uv,
                                   const float* b1, const float* w2, const float* b2, const int32_t* seq_len,
                                   const int32_t* type_tag, int B, int T, int L, int I, int o_id, int cls_id, int sep_id,
                                   int cap, int32_t* pred_ids, int32_t* spans, float* span_probs, int32_t* span_counts,
                                   void* workspace, size_t workspace_bytes, ner_stream_t stream) {
  if (B < 0 || T < 1 || cap < 0) return NER_ERR_INVALID_ARG;
  if (T > kMaxTypes) return NER_ERR_UNSUPPORTED;
  const int shape = check_match_shape(B * T, L, I, ld_uv);
  if (shape != NER_OK) return shape;
  if (B == 0) return NER_OK;
  if (!start_logits || !end_logits || !uv || !b1 || !w2 || !b2 || !seq_len || !type_tag || !pred_ids || !span_counts)
    return NER_ERR_INVALID_ARG;
  if (cap > 0 && (!spans || !span_probs)) return NER_ERR_INVALID_ARG;
  if (!aligned16(uv) || !aligned16(b1) || !aligned16(w2)) return NER_ERR_INVALID_ARG;
  const int P = B * T;
  if (!workspace || workspace_bytes < ner_mrc_span_decode_workspace_bytes(P, L)) return NER_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* zf = static_cast<float*>(workspace);
  int32_t* lists = reinterpret_cast<int32_t*>(zf + (size_t)P * L * L);
  int32_t* counts = lists + (size_t)P * 2 * L;
  span_flags_kernel<<<P, 128, 0, st>>>(start_logits, end_logits, seq_len, T, L, lists, counts);
  int rc = ner_launch_status();
  if (rc != NER_OK) return rc;
  span_tile_kernel<false, true><<<dim3(tile_count(L), P), kTileThreads, 0, st>>>(
      uv, ld_uv, b1, w2, b2, seq_len, T, nullptr, lists, counts, L, I, 1.f, 0, zf, nullptr);
  if ((rc = ner_launch_status()) != NER_OK) return rc;
  span_decode_kernel<<<B, kDecodeThreads, 0, st>>>(start_logits, end_logits, zf, seq_len, type_tag, T, L, o_id, cls_id,
                                                   sep_id, cap, pred_ids, spans, span_probs, span_counts);
  return ner_launch_status();
}
