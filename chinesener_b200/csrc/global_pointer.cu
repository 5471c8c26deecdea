// GlobalPointer span head of the bert_global_pointer plugin (model/bert_global_pointer.py; Su, 2021): for every entity
// type t and span (i, j) of sentence b,
//   s[b,t,i,j] = q'_i . k'_j / sqrt(D),   q' = RoPE_i(P[b,i, t*2D : t*2D+D]),   k' = RoPE_j(P[b,j, t*2D+D : (t+1)*2D])
// with D = 64 and P = h W + b the projection GEMM's output; its targets, its multilabel categorical cross-entropy
// (bert4keras' global_pointer_crossentropy) and gradient, and the PREDICT decode.
//
// The rotated operands are bf16 [rows, T, 2, D] (q with 1/8 folded in, then k), written once by ner_gp_rope; the span
// scores are a batched Q'K'^T on the tensor cores (mma.sync.m16n8k16, bf16 -> fp32).  A CTA owns a 64-row query tile of
// one (b, t) and walks only the key tiles of the upper triangle inside len_b; the 64 x 64 score tile stays in registers
// (4 warps x 16 rows), so [B, T, L, L] never exists in training.  The loss keeps per-row online (max, sum) pairs of the
// negative set {e^s} and the positive set {e^-s}, reduces them to one pair per CTA in a fixed order and writes it as a
// per-tile partial; a second launch merges the partials in index order.  The backward recomputes S per tile: one launch
// owns query tiles (dQ' = dS K'), one owns key tiles (dK' = dS^T Q'), so every output row has one owner.  A split mode
// (hi + lo operands, hi.hi + hi.lo + lo.hi) serves the fp32-accurate encoder in PREDICT / EVAL.
#include <math.h>

#include <type_traits>

#include "common.cuh"
#include "mma_tile.cuh"
#include "span_common.cuh"

namespace {

using namespace nerdev;
using namespace mma_tile;
using namespace span;

constexpr int kMaxTypes = 32;
constexpr int kMaxLen = 512;     // i, j <= 510 fit the 9-bit fields of the decode's priority key
static_assert(kMaxLen <= kDecodeRows, "the decode holds a whole sentence in shared memory");
constexpr int kTile = 64;        // query / key tile
constexpr int kThreads = 128;    // 4 warps x 16 rows
constexpr float kQScale = 0.125f;   // 1 / sqrt(D), exact in every format

// Row layout of sentence b: first row and row count (padded b*L, L rows; packed cu[b], cu[b+1] - cu[b] rows)
struct Rows {
  size_t base;
  int n;
};
__device__ __forceinline__ Rows sentence_rows(const int32_t* __restrict__ cu, int b, int L) {
  if (cu == nullptr) return Rows{(size_t)b * L, L};
  const int c0 = __ldg(cu + b), c1 = __ldg(cu + b + 1);
  return Rows{(size_t)c0, min(max(c1 - c0, 0), L)};
}

// 64 rows (s0 + r, clamped to s_max) of one side of type t -> smem [64][PITCH] (one cp.async group per call site)
__device__ __forceinline__ void stage_tile(__nv_bfloat16* dst, const __nv_bfloat16* __restrict__ rot, size_t base, int T,
                                           int t, int side, int s0, int s_max, int tid) {
  for (int idx = tid; idx < kTile * (D / 8); idx += kThreads) {
    const int r = idx >> 3, c = idx & 7;
    const int s = min(s0 + r, s_max);
    cp_async16(dst + r * PITCH + c * 8, rot + ((base + s) * T + t) * (2 * D) + side * D + c * 8);
  }
}

// (max, sum) of a set of exponentials, merged: m = -inf / s = 0 is the empty set
__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
  if (s2 == 0.f) return;
  if (s == 0.f) {
    m = m2;
    s = s2;
    return;
  }
  const float mx = fmaxf(m, m2);
  s = s * expf(m - mx) + s2 * expf(m2 - mx);
  m = mx;
}

// log(1 + sum) of a merged set: the 0 term of the multilabel cross-entropy included
__device__ __forceinline__ float lse_with_zero(float m, float s) {
  if (s == 0.f) return 0.f;
  const float M = fmaxf(m, 0.f);
  return M + logf(expf(-M) + s * expf(m - M));
}

struct TileSmem {
  __nv_bfloat16 a_hi[kTile * PITCH];
  __nv_bfloat16 b_hi[kTile * PITCH];
  int32_t se[kTile];
  float red[4][4];
};
struct TileSmemSplit {
  __nv_bfloat16 a_hi[kTile * PITCH];
  __nv_bfloat16 b_hi[kTile * PITCH];
  __nv_bfloat16 a_lo[kTile * PITCH];
  __nv_bfloat16 b_lo[kTile * PITCH];
  int32_t se[kTile];
  float red[4][4];
};

// Scores of one query tile of (b, t) against the key tiles of the upper triangle.
//   kScores = false (ner_gp_loss_fwd): per-tile partial (max, sum) of the negatives' e^s and the positives' e^-s ->
//     partial[bt * nq + qt] (float4: m_neg, s_neg, m_pos, s_pos).
//   kScores = true (ner_gp_decode): s written to scores[((bt * L) + i) * L + j] at the candidates only.
template <bool kSplit, bool kScores>
__global__ void __launch_bounds__(kThreads)
gp_tile_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo,
               const int32_t* __restrict__ seq_len, const int32_t* __restrict__ cu, const int32_t* __restrict__ span_end,
               int T, int L, float4* __restrict__ partial, float* __restrict__ scores) {
  using Smem = typename std::conditional<kSplit, TileSmemSplit, TileSmem>::type;
  __shared__ __align__(16) Smem sm;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, cq = (lane & 3) * 2;
  const int qt = blockIdx.x, bt = blockIdx.y, b = bt / T, t = bt - b * T, nq = gridDim.x;
  const Rows rw = sentence_rows(cu, b, L);
  const int len = min(clamp_len(__ldg(seq_len + b), L), rw.n), m = len - 2;
  const int i0 = qt * kTile;
  if (m < 1 || i0 > m) {
    if (!kScores && tid == 0) partial[(size_t)bt * nq + qt] = make_float4(-INFINITY, 0.f, -INFINITY, 0.f);
    return;
  }
  stage_tile(sm.a_hi, hi, rw.base, T, t, 0, i0, len - 1, tid);
  if constexpr (kSplit) stage_tile(sm.a_lo, lo, rw.base, T, t, 0, i0, len - 1, tid);
  cp_async_commit();
  if (!kScores && tid < kTile) sm.se[tid] = __ldg(span_end + ((size_t)bt) * L + min(i0 + tid, L - 1));
  cp_async_wait<0>();
  __syncthreads();
  uint32_t qa[4][4], qla[4][4];
  load_a_frags(qa, sm.a_hi, warp * 16 + (lane >> 2), cq);
  if constexpr (kSplit) load_a_frags(qla, sm.a_lo, warp * 16 + (lane >> 2), cq);
  const int ra = warp * 16 + (lane >> 2);           // tile rows ra, ra + 8
  int se_row[2] = {-1, -1};
  if (!kScores) {
    se_row[0] = sm.se[ra];
    se_row[1] = sm.se[ra + 8];
  }
  float mn[2] = {-INFINITY, -INFINITY}, sn[2] = {0.f, 0.f}, mp[2] = {-INFINITY, -INFINITY}, sp[2] = {0.f, 0.f};
  const int kt_end = m / kTile;
  for (int kt = qt; kt <= kt_end; ++kt) {
    const int j0 = kt * kTile;
    __syncthreads();                                  // the previous key tile is consumed
    stage_tile(sm.b_hi, hi, rw.base, T, t, 1, j0, len - 1, tid);
    if constexpr (kSplit) stage_tile(sm.b_lo, lo, rw.base, T, t, 1, j0, len - 1, tid);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    float acc[8][4];
    clear_tile(acc);
    mma_a_bt(acc, qa, sm.b_hi, 0, lane, cq);
    if constexpr (kSplit) {
      mma_a_bt(acc, qa, sm.b_lo, 0, lane, cq);
      mma_a_bt(acc, qla, sm.b_hi, 0, lane, cq);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int i = i0 + ra + 8 * h;
      const bool row_ok = i >= 1 && i <= m;
      if (kScores) {
        if (row_ok) {
#pragma unroll
          for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int j = j0 + nt * 8 + cq + e;
              if (j >= i && j <= m) scores[((size_t)bt * L + i) * L + j] = acc[nt][2 * h + e];
            }
        }
        continue;
      }
      if (!row_ok) continue;
      float tn = -INFINITY, tp = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int j = j0 + nt * 8 + cq + e;
          const float v = acc[nt][2 * h + e];
          if (j >= i && j <= m) {
            if (j == se_row[h]) tp = fmaxf(tp, -v);
            else tn = fmaxf(tn, v);
          }
        }
      if (tn == -INFINITY && tp == -INFINITY) continue;
      const float nmn = fmaxf(mn[h], tn), nmp = fmaxf(mp[h], tp);
      if (sn[h] != 0.f && nmn != mn[h]) sn[h] *= __expf(mn[h] - nmn);
      if (sp[h] != 0.f && nmp != mp[h]) sp[h] *= __expf(mp[h] - nmp);
      mn[h] = nmn;
      mp[h] = nmp;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int j = j0 + nt * 8 + cq + e;
          const float v = acc[nt][2 * h + e];
          if (j >= i && j <= m) {
            const bool pos = j == se_row[h];
            const float x = __expf(pos ? -v - nmp : v - nmn);
            if (pos) sp[h] += x;
            else sn[h] += x;
          }
        }
    }
  }
  if (kScores) return;
  // thread (two rows) -> warp (butterfly: every lane merges the same two values) -> CTA (warps in order)
  lse_merge(mn[0], sn[0], mn[1], sn[1]);
  lse_merge(mp[0], sp[0], mp[1], sp[1]);
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, mn[0], o), s2 = __shfl_xor_sync(0xffffffffu, sn[0], o);
    const float m3 = __shfl_xor_sync(0xffffffffu, mp[0], o), s3 = __shfl_xor_sync(0xffffffffu, sp[0], o);
    if (lane & o) {
      float a = m2, c = s2;
      lse_merge(a, c, mn[0], sn[0]);
      mn[0] = a;
      sn[0] = c;
      a = m3;
      c = s3;
      lse_merge(a, c, mp[0], sp[0]);
      mp[0] = a;
      sp[0] = c;
    } else {
      lse_merge(mn[0], sn[0], m2, s2);
      lse_merge(mp[0], sp[0], m3, s3);
    }
  }
  if (lane == 0) {
    sm.red[warp][0] = mn[0];
    sm.red[warp][1] = sn[0];
    sm.red[warp][2] = mp[0];
    sm.red[warp][3] = sp[0];
  }
  __syncthreads();
  if (tid == 0) {
    float a = -INFINITY, c = 0.f, d = -INFINITY, e = 0.f;
    for (int w = 0; w < 4; ++w) {
      lse_merge(a, c, sm.red[w][0], sm.red[w][1]);
      lse_merge(d, e, sm.red[w][2], sm.red[w][3]);
    }
    partial[(size_t)bt * nq + qt] = make_float4(a, c, d, e);
  }
}

// Partials of every (b, t) merged in tile order -> lse [B*T, 2] (neg, pos; each with the 0 term) and the loss = mean over
// B*T of lse_neg + lse_pos (per-thread sums in (b, t) order, then a fixed tree).  One CTA.
__global__ void __launch_bounds__(1024)
gp_loss_finalize_kernel(const float4* __restrict__ partial, int BT, int nq, float* __restrict__ lse, float* __restrict__ loss) {
  __shared__ double s_sum[1024];
  const int tid = threadIdx.x;
  double acc = 0.0;
  for (int bt = tid; bt < BT; bt += 1024) {
    float a = -INFINITY, c = 0.f, d = -INFINITY, e = 0.f;
    for (int q = 0; q < nq; ++q) {
      const float4 p = partial[(size_t)bt * nq + q];
      lse_merge(a, c, p.x, p.y);
      lse_merge(d, e, p.z, p.w);
    }
    const float ln = lse_with_zero(a, c), lp = lse_with_zero(d, e);
    lse[2 * bt] = ln;
    lse[2 * bt + 1] = lp;
    acc += (double)ln + (double)lp;
  }
  s_sum[tid] = acc;
  __syncthreads();
  for (int w = 512; w > 0; w >>= 1) {
    if (tid < w) s_sum[tid] += s_sum[tid + w];
    __syncthreads();
  }
  if (tid == 0) *loss = (float)(s_sum[0] / (double)BT);
}

// dS of one score: e^(s - lse_neg) on a negative, -e^(-s - lse_pos) on a positive, times g = d_loss / (B T)
__device__ __forceinline__ float gp_ds(float v, bool pos, float ln, float lp, float g) {
  return pos ? -__expf(-v - lp) * g : __expf(v - ln) * g;
}

// Backward.  kKeys = false: the CTA owns query tile qt of (b, t), walks key tiles kt >= qt: dQ' = dS K'.
//            kKeys = true:  the CTA owns key tile kt, walks query tiles qt <= kt with S^T = K' Q'^T: dK' = dS^T Q'.
// d_rot [rows, T, 2, D] f32: side 0 (dQ') / side 1 (dK') of every row of the sentence is written (0 off the candidates).
template <bool kKeys>
__global__ void __launch_bounds__(kThreads)
gp_bwd_kernel(const __nv_bfloat16* __restrict__ rot, const int32_t* __restrict__ seq_len, const int32_t* __restrict__ cu,
              const int32_t* __restrict__ span_end, const float* __restrict__ lse, int T, int L, float g,
              float* __restrict__ d_rot) {
  __shared__ __align__(16) TileSmem sm;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, cq = (lane & 3) * 2;
  const int ot = blockIdx.x, bt = blockIdx.y, b = bt / T, t = bt - b * T;
  const Rows rw = sentence_rows(cu, b, L);
  const int len = min(clamp_len(__ldg(seq_len + b), L), rw.n), m = len - 2;
  const int o0 = ot * kTile;
  const int own_side = kKeys ? 1 : 0;
  const int ra = warp * 16 + (lane >> 2);
  float out[8][4];
  clear_tile(out);
  if (m >= 1 && o0 <= m) {
    const float ln = __ldg(lse + 2 * bt), lp = __ldg(lse + 2 * bt + 1);
    stage_tile(sm.a_hi, rot, rw.base, T, t, own_side, o0, len - 1, tid);
    cp_async_commit();
    if (!kKeys && tid < kTile) sm.se[tid] = __ldg(span_end + (size_t)bt * L + min(o0 + tid, L - 1));
    cp_async_wait<0>();
    __syncthreads();
    uint32_t oa[4][4];
    load_a_frags(oa, sm.a_hi, ra, cq);
    int se_row[2] = {-1, -1};
    if (!kKeys) {
      se_row[0] = sm.se[ra];
      se_row[1] = sm.se[ra + 8];
    }
    const int first = kKeys ? 0 : ot, last = kKeys ? ot : m / kTile;
    for (int xt = first; xt <= last; ++xt) {
      const int x0 = xt * kTile;
      __syncthreads();
      stage_tile(sm.b_hi, rot, rw.base, T, t, 1 - own_side, x0, len - 1, tid);
      cp_async_commit();
      if (kKeys && tid < kTile) sm.se[tid] = __ldg(span_end + (size_t)bt * L + min(x0 + tid, L - 1));
      cp_async_wait<0>();
      __syncthreads();
      float acc[8][4];
      clear_tile(acc);
      mma_a_bt(acc, oa, sm.b_hi, 0, lane, cq);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = o0 + ra + 8 * h;                // own index: i (queries) or j (keys)
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = x0 + nt * 8 + cq + e;       // other index
            const int i = kKeys ? c : r, j = kKeys ? r : c;
            float ds = 0.f;
            if (i >= 1 && i <= j && j <= m) {
              const int se = kKeys ? sm.se[nt * 8 + cq + e] : se_row[h];
              ds = gp_ds(acc[nt][2 * h + e], se == j, ln, lp, g);
            }
            acc[nt][2 * h + e] = ds;
          }
      }
      mma_p_b(out, acc, sm.b_hi, 0, lane);
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = o0 + ra + 8 * h;
    if (r >= rw.n) continue;
    float* dst = d_rot + ((rw.base + r) * T + t) * (2 * D) + own_side * D;
#pragma unroll
    for (int dt = 0; dt < 8; ++dt)
      *reinterpret_cast<float2*>(dst + dt * 8 + cq) = make_float2(out[dt][2 * h], out[dt][2 * h + 1]);
  }
}

// RoPE angles of position s: cos / sin(s * 10000^(-2i/D)), i < D/2, in double (exact to fp32 rounding up to s = 511)
__device__ __forceinline__ void rope_table(float* cs, float* sn, int s) {
  if (threadIdx.x < D / 2) {
    const double theta = pow(10000.0, -2.0 * (double)threadIdx.x / (double)D);
    double sv, cv;
    sincos((double)s * theta, &sv, &cv);
    cs[threadIdx.x] = (float)cv;
    sn[threadIdx.x] = (float)sv;
  }
  __syncthreads();
}

// Forward rotation: one CTA per (position s, sentence b); column c of P and of the output is the same (t*2D + side*D + d).
__global__ void __launch_bounds__(256)
gp_rope_kernel(const float* __restrict__ proj, int ld, const int32_t* __restrict__ cu, int T, int L,
               __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  __shared__ float cs[D / 2], sn[D / 2];
  const int s = blockIdx.x, b = blockIdx.y;
  const Rows rw = sentence_rows(cu, b, L);
  if (s >= rw.n) return;
  rope_table(cs, sn, s);
  const size_t row = rw.base + s;
  for (int p = threadIdx.x; p < T * D; p += 256) {
    const int i = p & (D / 2 - 1);
    const bool q = ((p >> 5) & 1) == 0;
    const float2 x = *reinterpret_cast<const float2*>(proj + row * ld + 2 * p);
    float r0 = fmaf(x.x, cs[i], -x.y * sn[i]);
    float r1 = fmaf(x.y, cs[i], x.x * sn[i]);
    if (q) {
      r0 *= kQScale;
      r1 *= kQScale;
    }
    const __nv_bfloat16 h0 = __float2bfloat16_rn(r0), h1 = __float2bfloat16_rn(r1);
    __nv_bfloat162 hv;
    hv.x = h0;
    hv.y = h1;
    *reinterpret_cast<__nv_bfloat162*>(hi + row * (size_t)T * 2 * D + 2 * p) = hv;
    if (lo != nullptr) {
      __nv_bfloat162 lv;
      lv.x = __float2bfloat16_rn(r0 - __bfloat162float(h0));
      lv.y = __float2bfloat16_rn(r1 - __bfloat162float(h1));
      *reinterpret_cast<__nv_bfloat162*>(lo + row * (size_t)T * 2 * D + 2 * p) = lv;
    }
  }
}

// Transposed rotation of the operand gradient (and the 1/8 of q): d_proj = R^T d_rot.
__global__ void __launch_bounds__(256)
gp_rope_bwd_kernel(const float* __restrict__ d_rot, const int32_t* __restrict__ cu, int T, int L, float* __restrict__ d_proj,
                   int ld) {
  __shared__ float cs[D / 2], sn[D / 2];
  const int s = blockIdx.x, b = blockIdx.y;
  const Rows rw = sentence_rows(cu, b, L);
  if (s >= rw.n) return;
  rope_table(cs, sn, s);
  const size_t row = rw.base + s;
  for (int p = threadIdx.x; p < T * D; p += 256) {
    const int i = p & (D / 2 - 1);
    const bool q = ((p >> 5) & 1) == 0;
    const float2 g = *reinterpret_cast<const float2*>(d_rot + row * (size_t)T * 2 * D + 2 * p);
    float d0 = fmaf(g.x, cs[i], g.y * sn[i]);
    float d1 = fmaf(g.y, cs[i], -g.x * sn[i]);
    if (q) {
      d0 *= kQScale;
      d1 *= kQScale;
    }
    *reinterpret_cast<float2*>(d_proj + row * ld + 2 * p) = make_float2(d0, d1);
  }
}

// Targets: one CTA per sentence.  span_end[b,t,s] = the end of the I-X_t run after a B-X_t at s (< len), else -1.
__global__ void __launch_bounds__(256)
gp_targets_kernel(const int32_t* __restrict__ labels, const int32_t* __restrict__ seq_len,
                  const int32_t* __restrict__ type_tag, int T, int L, int32_t* __restrict__ span_end) {
  __shared__ int32_t y[kMaxLen];
  const int b = blockIdx.x;
  const int len = clamp_len(__ldg(seq_len + b), L);
  for (int s = threadIdx.x; s < L; s += 256) y[s] = s < len ? __ldg(labels + (size_t)b * L + s) : -1;
  __syncthreads();
  for (int e = threadIdx.x; e < T * L; e += 256) {
    const int t = e / L, s = e - t * L;
    const int tb = __ldg(type_tag + 2 * t), ti = __ldg(type_tag + 2 * t + 1);
    span_end[((size_t)b * T + t) * L + s] = s < len && y[s] == tb ? run_end(y, s, len, ti) : -1;
  }
}

// Candidates of the decode: every type at every (i, j).
struct AllTypes {
  int T;
  __device__ __forceinline__ bool live(int) const { return true; }
  template <class F>
  __device__ __forceinline__ void for_each(int, int, F&& f) const {
    for (int t = 0; t < T; ++t)
      if (!f(t)) return;
  }
};

// Decode: one CTA per sentence over the candidate scores (span_common.cuh).
__global__ void __launch_bounds__(kDecodeThreads)
gp_decode_kernel(const float* __restrict__ sc, const int32_t* __restrict__ seq_len, const int32_t* __restrict__ type_tag,
                 int T, int L, int o_id, int cls_id, int sep_id, int cap, int32_t* __restrict__ pred_ids,
                 int32_t* __restrict__ spans, float* __restrict__ probs, int32_t* __restrict__ span_counts) {
  __builtin_assume(T >= 1);   // check_shape; keeps the empty-type test out of the (i, j) loops
  const int len = clamp_len(__ldg(seq_len + blockIdx.x), L);
  greedy_span_decode(AllTypes{T}, sc, T, L, len, type_tag, o_id, cls_id, sep_id, cap, pred_ids, spans, probs,
                     span_counts);
}

// shared shape checks: 0 or the status to return
int check_shape(int B, int T, int L) {
  if (B < 0 || T < 1 || L < 1) return NER_ERR_INVALID_ARG;
  if (T > kMaxTypes || L > kMaxLen) return NER_ERR_UNSUPPORTED;
  if ((long long)B * T * L * L >= 0x7fffffffLL) return NER_ERR_UNSUPPORTED;
  return NER_OK;
}

int n_tiles(int L) { return (L + kTile - 1) / kTile; }

}  // namespace

extern "C" int ner_gp_targets(const int32_t* label_ids, const int32_t* seq_len, const int32_t* type_tag, int B, int T, int L,
                              int32_t* span_end, ner_stream_t stream) {
  const int shape = check_shape(B, T, L);
  if (shape != NER_OK) return shape;
  if (B == 0) return NER_OK;
  if (!label_ids || !seq_len || !type_tag || !span_end) return NER_ERR_INVALID_ARG;
  gp_targets_kernel<<<B, 256, 0, static_cast<cudaStream_t>(stream)>>>(label_ids, seq_len, type_tag, T, L, span_end);
  return ner_launch_status();
}

extern "C" int ner_gp_rope(const float* proj, int ld_proj, const int32_t* cu_seqlens, int B, int T, int L, void* rot_hi,
                           void* rot_lo, ner_stream_t stream) {
  const int shape = check_shape(B, T, L);
  if (shape != NER_OK) return shape;
  if (ld_proj < 2 * D * T || ld_proj % 2 != 0) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!proj || !rot_hi) return NER_ERR_INVALID_ARG;
  if ((reinterpret_cast<uintptr_t>(proj) & 7u) != 0 || !aligned16(rot_hi) || (rot_lo && !aligned16(rot_lo)))
    return NER_ERR_INVALID_ARG;
  gp_rope_kernel<<<dim3(L, B), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      proj, ld_proj, cu_seqlens, T, L, static_cast<__nv_bfloat16*>(rot_hi), static_cast<__nv_bfloat16*>(rot_lo));
  return ner_launch_status();
}

extern "C" int ner_gp_rope_bwd(const float* d_rot, const int32_t* cu_seqlens, int B, int T, int L, float* d_proj,
                               int ld_dproj, ner_stream_t stream) {
  const int shape = check_shape(B, T, L);
  if (shape != NER_OK) return shape;
  if (ld_dproj < 2 * D * T || ld_dproj % 2 != 0) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!d_rot || !d_proj) return NER_ERR_INVALID_ARG;
  if (!aligned16(d_rot) || (reinterpret_cast<uintptr_t>(d_proj) & 7u) != 0) return NER_ERR_INVALID_ARG;
  gp_rope_bwd_kernel<<<dim3(L, B), 256, 0, static_cast<cudaStream_t>(stream)>>>(d_rot, cu_seqlens, T, L, d_proj,
                                                                               ld_dproj);
  return ner_launch_status();
}

extern "C" size_t ner_gp_loss_workspace_bytes(int B, int T, int L) {
  if (check_shape(B, T, L) != NER_OK || B == 0) return 0;
  return (size_t)B * T * n_tiles(L) * sizeof(float4);
}

extern "C" int ner_gp_loss_fwd(const void* rot_hi, const void* rot_lo, const int32_t* seq_len, const int32_t* cu_seqlens,
                               const int32_t* span_end, int B, int T, int L, float* loss, float* lse, void* workspace,
                               size_t workspace_bytes, ner_stream_t stream) {
  const int shape = check_shape(B, T, L);
  if (shape != NER_OK) return shape;
  if (B == 0) return NER_OK;
  if (!rot_hi || !seq_len || !span_end || !loss || !lse) return NER_ERR_INVALID_ARG;
  if (!aligned16(rot_hi) || (rot_lo && !aligned16(rot_lo))) return NER_ERR_INVALID_ARG;
  if (!workspace || workspace_bytes < ner_gp_loss_workspace_bytes(B, T, L)) return NER_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const auto* hi = static_cast<const __nv_bfloat16*>(rot_hi);
  const auto* lo = static_cast<const __nv_bfloat16*>(rot_lo);
  float4* partial = static_cast<float4*>(workspace);
  const dim3 grid(n_tiles(L), B * T);
  if (lo)
    gp_tile_kernel<true, false><<<grid, kThreads, 0, st>>>(hi, lo, seq_len, cu_seqlens, span_end, T, L, partial, nullptr);
  else
    gp_tile_kernel<false, false><<<grid, kThreads, 0, st>>>(hi, lo, seq_len, cu_seqlens, span_end, T, L, partial, nullptr);
  const int rc = ner_launch_status();
  if (rc != NER_OK) return rc;
  gp_loss_finalize_kernel<<<1, 1024, 0, st>>>(partial, B * T, n_tiles(L), lse, loss);
  return ner_launch_status();
}

extern "C" int ner_gp_loss_bwd(const void* rot, const int32_t* seq_len, const int32_t* cu_seqlens, const int32_t* span_end,
                               const float* lse, int B, int T, int L, float d_loss, float* d_rot, ner_stream_t stream) {
  const int shape = check_shape(B, T, L);
  if (shape != NER_OK) return shape;
  if (B == 0) return NER_OK;
  if (!rot || !seq_len || !span_end || !lse || !d_rot) return NER_ERR_INVALID_ARG;
  if (!aligned16(rot) || !aligned16(d_rot)) return NER_ERR_INVALID_ARG;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const auto* r = static_cast<const __nv_bfloat16*>(rot);
  const float g = d_loss / (float)(B * T);
  const dim3 grid(n_tiles(L), B * T);
  gp_bwd_kernel<false><<<grid, kThreads, 0, st>>>(r, seq_len, cu_seqlens, span_end, lse, T, L, g, d_rot);
  const int rc = ner_launch_status();
  if (rc != NER_OK) return rc;
  gp_bwd_kernel<true><<<grid, kThreads, 0, st>>>(r, seq_len, cu_seqlens, span_end, lse, T, L, g, d_rot);
  return ner_launch_status();
}

extern "C" size_t ner_gp_decode_workspace_bytes(int B, int T, int L) {
  if (check_shape(B, T, L) != NER_OK || B == 0) return 0;
  return (size_t)B * T * L * L * sizeof(float);
}

extern "C" int ner_gp_decode(const void* rot_hi, const void* rot_lo, const int32_t* seq_len, const int32_t* cu_seqlens,
                             const int32_t* type_tag, int B, int T, int L, int o_id, int cls_id, int sep_id, int cap,
                             int32_t* pred_ids, int32_t* spans, float* span_probs, int32_t* span_counts, void* workspace,
                             size_t workspace_bytes, ner_stream_t stream) {
  if (cap < 0) return NER_ERR_INVALID_ARG;
  const int shape = check_shape(B, T, L);
  if (shape != NER_OK) return shape;
  if (B == 0) return NER_OK;
  if (!rot_hi || !seq_len || !type_tag || !pred_ids || !span_counts) return NER_ERR_INVALID_ARG;
  if (cap > 0 && (!spans || !span_probs)) return NER_ERR_INVALID_ARG;
  if (!aligned16(rot_hi) || (rot_lo && !aligned16(rot_lo))) return NER_ERR_INVALID_ARG;
  if (!workspace || workspace_bytes < ner_gp_decode_workspace_bytes(B, T, L)) return NER_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const auto* hi = static_cast<const __nv_bfloat16*>(rot_hi);
  const auto* lo = static_cast<const __nv_bfloat16*>(rot_lo);
  float* sc = static_cast<float*>(workspace);
  const dim3 grid(n_tiles(L), B * T);
  if (lo)
    gp_tile_kernel<true, true><<<grid, kThreads, 0, st>>>(hi, lo, seq_len, cu_seqlens, nullptr, T, L, nullptr, sc);
  else
    gp_tile_kernel<false, true><<<grid, kThreads, 0, st>>>(hi, lo, seq_len, cu_seqlens, nullptr, T, L, nullptr, sc);
  const int rc = ner_launch_status();
  if (rc != NER_OK) return rc;
  gp_decode_kernel<<<B, kDecodeThreads, 0, st>>>(sc, seq_len, type_tag, T, L, o_id, cls_id, sep_id, cap, pred_ids, spans,
                                                 span_probs, span_counts);
  return ner_launch_status();
}
