// Lattice LSTM recurrence (Zhang & Yang, ACL 2018, "Chinese NER Using Lattice LSTM") and its back-propagation through
// time, as persistent thread-block-cluster kernels (sm_90a).  model/lattice_lstm_crf.py states the definition.
//
// Same decomposition as bilstm.cu / bigru.cu: a cluster of C CTAs owns R batch rows of one direction for every step; CTA
// `rank` owns the hidden units [rank * HU, (rank + 1) * HU), HU = H / C, and keeps its slice of the recurrent weights in
// shared memory for the whole sequence.  The input halves of every gate (chars and word slots) are hoisted GEMMs done by
// the caller.  Per step s (forward):
//   1. GEMV [W_hh | W_whh]^T h_{s-1}: char gates of step s and the word gates of the words whose cell reads the state after
//      step s - 1 ("new" words: fw, words starting at s - 1; bw, words ending there).  W_whh h is shared by all of them.
//   2. c^w = σ(f) c_{s-1} + σ(i^w) tanh(g^w) for each new word (the cell thread's own units), published to every CTA
//      through DSMEM in chunks of 8 words; then W_ac^T c^w for the owned units.  c^w and W_ac^T c^w wait in a per-CTA ring
//      keyed by the word's slot (start % 10, k) until the step that merges the word (words have 2..10 characters, so a
//      ring entry is consumed before the slot that reuses it is written).
//   3. c_s: the coupled gate (1 - i) c_{s-1} + i g when no word ends at s, else the e^i / e^a-weighted mean of g and the
//      merged c^w; h_s = o tanh(c_s), published to every CTA through DSMEM.  One cluster barrier per step, one more per
//      chunk of new words.
// The backward kernel walks the steps in reverse.  A word's cell gradient dc^w is complete when the sweep reaches the
// step that created the cell (every merge is later in forward order), so each accumulation has one owner in a fixed
// order: no float atomics, and repeated calls are bit-identical.
#include <cooperative_groups.h>

#include "common.cuh"
#include "rnn_cluster.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int kMaxWordLen = 10;                       // MaxWordLen, data/word_enhance.py
constexpr int kMaxKw = 8;
constexpr int kMaxList = (kMaxWordLen - 1) * kMaxKw;  // words one step can create or merge (9 starts x Kw slots)
constexpr int kChunk = 8;                             // words exchanged per cluster round
constexpr int kThreads = 512;
constexpr int kRing = kMaxWordLen;                    // ring rows: slot start % 10

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }

// Length of the word in slot (p, k) of a row, 0 when the slot is empty or malformed (length outside [2, 10] or reaching
// past the row's length).
__device__ __forceinline__ int slot_len(const int32_t* lat, int p, int k, int Kw, int len) {
  const int n = lat[p * Kw + k];
  return (n >= 2 && n <= kMaxWordLen && p + n - 1 < len) ? n : 0;
}

// One warp lists, for row r at step s, the slots (p * Kw + k) of the new words (cell after step s - 1) and of the merged
// words (merge at step s), in a fixed order.  Slots starting at p: "S(p)"; slots ending at e: "E(e)", starts ascending.
__device__ void build_lists(const int32_t* lat, int len, int dir, int s, int Kw, int* new_list, int* n_new,
                            int* merge_list, int* n_merge) {
  const int lane = threadIdx.x & 31;
  for (int which = 0; which < 2; ++which) {
    int* list = which == 0 ? new_list : merge_list;
    int cnt = 0;
    const int st = which == 0 ? s - 1 : s;               // step whose position the list is keyed on
    const bool ok_step = s < len && st >= 0;
    const int pos = dir == 0 ? st : len - 1 - st;
    // fw: new = S(pos), merge = E(pos); bw: new = E(pos), merge = S(pos)
    const bool by_start = (which == 0) == (dir == 0);
    const int ncand = ok_step ? (by_start ? Kw : (kMaxWordLen - 1) * Kw) : 0;
    for (int c0 = 0; c0 < ncand; c0 += 32) {
      const int c = c0 + lane;
      bool ok = false;
      int code = 0;
      if (c < ncand) {
        if (by_start) {
          ok = slot_len(lat, pos, c, Kw, len) > 0;
          code = pos * Kw + c;
        } else {
          const int b = pos - (kMaxWordLen - 1) + c / Kw, k = c % Kw;
          if (b >= 0) {
            const int n = slot_len(lat, b, k, Kw, len);
            ok = n > 0 && b + n - 1 == pos;
            code = b * Kw + k;
          }
        }
      }
      const unsigned m = __ballot_sync(0xffffffffu, ok);
      if (ok) list[cnt + __popc(m & ((1u << lane) - 1u))] = code;
      cnt += __popc(m);
    }
    if (lane == 0) *(which == 0 ? n_new : n_merge) = cnt;
  }
}

__device__ __forceinline__ int ring_of(int code, int Kw) { return ((code / Kw) % kRing) * Kw + code % Kw; }

template <int R>
__global__ void __launch_bounds__(kThreads, 1)
lattice_fwd_kernel(const float* __restrict__ xproj, const float* __restrict__ wproj, const int32_t* __restrict__ lat_len,
                   const float* __restrict__ wrec_fw, const float* __restrict__ wrec_bw, const float* __restrict__ wac_fw,
                   const float* __restrict__ wac_bw, const int32_t* __restrict__ seq_len, float* __restrict__ out, int B,
                   int L, int H, int Kw, int C, float* __restrict__ gates, float* __restrict__ cstate,
                   float* __restrict__ norm, float* __restrict__ wgates, float* __restrict__ cw_out,
                   float* __restrict__ aw_out, float* __restrict__ hw_out) {
  cg::cluster_group cluster = cg::this_cluster();
  const int HU = H / C, NC = 6 * HU, RK = kRing * Kw;
  const rnn::RowGroup grp = rnn::row_group(C, B, R);
  const int rank = grp.rank, dir = grp.dir, b0 = grp.b0;
  const int tid = threadIdx.x;
  const bool save = gates != nullptr;

  extern __shared__ __align__(16) float smem[];
  float* W1 = smem;                              // [H][6HU]: column q * HU + u = wrec[:, q * H + rank * HU + u]
  float* W2 = W1 + (size_t)H * NC;               // [H][HU]: wac[:, rank * HU + u]
  float* hbuf = W2 + (size_t)H * HU;             // [2][R][H]
  float* zb = hbuf + 2 * R * H;                  // [R][6HU] recurrent parts of this step's gates
  float* cwx = zb + R * NC;                      // [R][kChunk][H] new word cells, all units (DSMEM target)
  float* cw_ring = cwx + R * kChunk * H;         // [R][10 * Kw][HU]
  float* acw_ring = cw_ring + R * RK * HU;       // [R][10 * Kw][HU]: W_ac^T c^w
  int* new_list = reinterpret_cast<int*>(acw_ring + R * RK * HU);   // [R][kMaxList]
  int* merge_list = new_list + R * kMaxList;                        // [R][kMaxList]
  int* n_new = merge_list + R * kMaxList;                           // [R]
  int* n_merge = n_new + R;                                         // [R]
  int* s_len = n_merge + R;                                         // [R]

  const float* wrec = dir == 0 ? wrec_fw : wrec_bw;
  const float* wac = dir == 0 ? wac_fw : wac_bw;
  for (int idx = tid; idx < H * NC; idx += blockDim.x) {
    const int k = idx / NC, c = idx - k * NC;
    W1[idx] = wrec[(size_t)k * 6 * H + (c / HU) * H + rank * HU + c % HU];
  }
  for (int idx = tid; idx < H * HU; idx += blockDim.x) {
    const int k = idx / HU, u = idx - k * HU;
    W2[idx] = wac[(size_t)k * H + rank * HU + u];
  }
  for (int idx = tid; idx < 2 * R * H; idx += blockDim.x) hbuf[idx] = 0.f;
  const int maxlen = rnn::load_lengths<R>(s_len, seq_len, b0, B, L);
  cluster.sync();   // every CTA's hbuf is zeroed before anyone writes remotely

  // cell role: thread (r, u) for tid < R * HU
  const bool cell_ok = tid < R * HU;
  const int cr = cell_ok ? tid / HU : 0, cu = cell_ok ? tid - cr * HU : 0;
  const int ug = rank * HU + cu;
  const int my_len = cell_ok ? s_len[cr] : 0;
  const int my_b = b0 + cr;
  float c_state = 0.f;

  for (int s = 0; s < maxlen; ++s) {
    const float* hcur = hbuf + (s & 1) * R * H;
    float* hnxt = hbuf + ((s + 1) & 1) * R * H;
    const int warp = tid >> 5;
    if (warp < R) {
      const int b = b0 + warp;
      build_lists(lat_len + (size_t)(b < B ? b : 0) * L * Kw, s_len[warp], dir, s, Kw, new_list + warp * kMaxList,
                  n_new + warp, merge_list + warp * kMaxList, n_merge + warp);
    }
    // 1. recurrent parts of the char gates and of the new words' gates
    for (int col = tid; col < NC; col += blockDim.x) {
      float acc[R];
#pragma unroll
      for (int r = 0; r < R; ++r) acc[r] = 0.f;
#pragma unroll 4
      for (int k = 0; k < H; ++k) {
        const float w = W1[k * NC + col];
#pragma unroll
        for (int r = 0; r < R; ++r) acc[r] = fmaf(hcur[r * H + k], w, acc[r]);
      }
#pragma unroll
      for (int r = 0; r < R; ++r) zb[r * NC + col] = acc[r];
    }
    __syncthreads();
    int max_new = 0;
#pragma unroll
    for (int r = 0; r < R; ++r) max_new = max(max_new, n_new[r]);
    // 2. word cells of the new words, W_ac^T c^w
    for (int j0 = 0; j0 < max_new; j0 += kChunk) {
      if (cell_ok) {
        const int nn = n_new[cr];
        for (int jj = 0; jj < kChunk && j0 + jj < nn; ++jj) {
          const int code = new_list[cr * kMaxList + j0 + jj];
          const size_t gs = (size_t)my_b * L * Kw + code;
          const float* wp = wproj + gs * 6 * H + (size_t)dir * 3 * H;
          const float f = sigm(wp[ug] + zb[cr * NC + 3 * HU + cu]);
          const float iw = sigm(wp[H + ug] + zb[cr * NC + 4 * HU + cu]);
          const float gw = tanhf(wp[2 * H + ug] + zb[cr * NC + 5 * HU + cu]);
          const float cwv = f * c_state + iw * gw;
          cw_ring[(cr * RK + ring_of(code, Kw)) * HU + cu] = cwv;
          float* dst = cwx + (cr * kChunk + jj) * H + ug;
          for (int q = 0; q < C; ++q) *cluster.map_shared_rank(dst, q) = cwv;
          if (save) {
            float* wg = wgates + gs * 6 * H + (size_t)dir * 3 * H;
            wg[ug] = f;
            wg[H + ug] = iw;
            wg[2 * H + ug] = gw;
            cw_out[gs * 2 * H + (size_t)dir * H + ug] = cwv;
            hw_out[gs * 2 * H + (size_t)dir * H + ug] = hcur[cr * H + ug];
          }
        }
      }
      cluster.sync();
      for (int idx = tid; idx < R * kChunk * HU; idx += blockDim.x) {
        const int r = idx / (kChunk * HU), jj = (idx / HU) % kChunk, u = idx % HU;
        if (j0 + jj >= n_new[r]) continue;
        const float* x = cwx + (r * kChunk + jj) * H;
        float acc = 0.f;
#pragma unroll 4
        for (int k = 0; k < H; ++k) acc = fmaf(x[k], W2[k * HU + u], acc);
        acw_ring[(r * RK + ring_of(new_list[r * kMaxList + j0 + jj], Kw)) * HU + u] = acc;
      }
      if (j0 + kChunk < max_new) cluster.sync();   // peers are done reading cwx before the next chunk overwrites it
      else __syncthreads();
    }
    // 3. the cell
    if (cell_ok) {
      const bool live = s < my_len;
      const int pos = dir == 0 ? s : my_len - 1 - s;
      if (live) {
        const size_t row = (size_t)my_b * L + pos;
        const float* xp = xproj + row * 8 * H + (size_t)dir * 4 * H;
        const float i_s = sigm(xp[ug] + zb[cr * NC + cu]);
        const float o_s = sigm(xp[H + ug] + zb[cr * NC + HU + cu]);
        const float g_a = tanhf(xp[2 * H + ug] + zb[cr * NC + 2 * HU + cu]);
        const int nm = n_merge[cr];
        float nrm = 0.f;
        if (nm == 0) {
          c_state = (1.f - i_s) * c_state + i_s * g_a;
        } else {
          const float xa = xp[3 * H + ug];
          const float ei = expf(i_s);
          float num = ei * g_a;
          nrm = ei;
          for (int j = 0; j < nm; ++j) {
            const int code = merge_list[cr * kMaxList + j];
            const int ri = (cr * RK + ring_of(code, Kw)) * HU + cu;
            const float a = sigm(xa + acw_ring[ri]);
            const float ea = expf(a);
            nrm += ea;
            num += ea * cw_ring[ri];
            if (save) aw_out[((size_t)my_b * L * Kw + code) * 2 * H + (size_t)dir * H + ug] = a;
          }
          c_state = num / nrm;
        }
        const float h = o_s * tanhf(c_state);
        float* dst = hnxt + cr * H + ug;
        for (int q = 0; q < C; ++q) *cluster.map_shared_rank(dst, q) = h;
        out[row * 2 * H + (size_t)dir * H + ug] = h;
        if (save) {
          float* gp = gates + row * 6 * H + (size_t)dir * 3 * H;
          gp[ug] = i_s;
          gp[H + ug] = o_s;
          gp[2 * H + ug] = g_a;
          cstate[row * 2 * H + (size_t)dir * H + ug] = c_state;
          norm[row * 2 * H + (size_t)dir * H + ug] = nrm;
        }
      } else if (my_b < B) {
        out[((size_t)my_b * L + s) * 2 * H + (size_t)dir * H + ug] = 0.f;   // past this row's end: zeros
      }
    }
    cluster.sync();
  }
  rnn::zero_past_maxlen(out, R, b0, B, L, H, dir, rank, HU, maxlen);
}

template <int R>
__global__ void __launch_bounds__(kThreads, 1)
lattice_bwd_kernel(const float* __restrict__ d_out, const float* __restrict__ gates, const float* __restrict__ cstate,
                   const float* __restrict__ norm, const float* __restrict__ wgates, const float* __restrict__ cw,
                   const float* __restrict__ aw, const int32_t* __restrict__ lat_len, const float* __restrict__ wrec_fw,
                   const float* __restrict__ wrec_bw, const float* __restrict__ wac_fw, const float* __restrict__ wac_bw,
                   const int32_t* __restrict__ seq_len, float* __restrict__ d_xproj, float* __restrict__ d_wproj,
                   float* __restrict__ d_alpha, int B, int L, int H, int Kw, int C) {
  cg::cluster_group cluster = cg::this_cluster();
  const int HU = H / C, H6 = 6 * H, RK = kRing * Kw;
  const rnn::RowGroup grp = rnn::row_group(C, B, R);
  const int rank = grp.rank, dir = grp.dir, b0 = grp.b0;
  const int tid = threadIdx.x;

  extern __shared__ __align__(16) float smem[];
  float* W1 = smem;                              // [HU][6H]: rows rank * HU + u of wrec
  float* W2 = W1 + (size_t)HU * H6;              // [H][HU]: W2[j][u] = wac[rank * HU + u][j]
  float* dzx = W2 + (size_t)H * HU;              // [2][R][6H]: dz_char of step s + 1 | sum of dz_w of words created after s
  float* dhb = dzx + 2 * R * H6;                 // [R][HU]
  float* dax = dhb + R * HU;                     // [R][kChunk][H] alpha gradients of merged words, all units
  float* dcw_ring = dax + R * kChunk * H;        // [R][10 * Kw][HU]
  int* new_list = reinterpret_cast<int*>(dcw_ring + R * RK * HU);
  int* merge_list = new_list + R * kMaxList;
  int* n_new = merge_list + R * kMaxList;
  int* n_merge = n_new + R;
  int* s_len = n_merge + R;

  const float* wrec = dir == 0 ? wrec_fw : wrec_bw;
  const float* wac = dir == 0 ? wac_fw : wac_bw;
  for (int idx = tid; idx < HU * H6; idx += blockDim.x) W1[idx] = wrec[(size_t)rank * HU * H6 + idx];
  for (int idx = tid; idx < H * HU; idx += blockDim.x) {
    const int j = idx / HU, u = idx - j * HU;
    W2[idx] = wac[(size_t)(rank * HU + u) * H + j];
  }
  for (int idx = tid; idx < 2 * R * H6; idx += blockDim.x) dzx[idx] = 0.f;
  const int maxlen = rnn::load_lengths<R>(s_len, seq_len, b0, B, L);
  // positions no step visits: d_xproj = 0
  for (int idx = tid; idx < R * HU; idx += blockDim.x) {
    const int r = idx / HU, u = idx - r * HU;
    const int b = b0 + r;
    if (b < B)
      for (int t = s_len[r]; t < L; ++t)
        for (int q = 0; q < 4; ++q) d_xproj[((size_t)b * L + t) * 8 * H + (size_t)dir * 4 * H + q * H + rank * HU + u] = 0.f;
  }
  cluster.sync();

  const bool cell_ok = tid < R * HU;
  const int cr = cell_ok ? tid / HU : 0, cu = cell_ok ? tid - cr * HU : 0;
  const int ug = rank * HU + cu;
  const int my_len = cell_ok ? s_len[cr] : 0;
  const int my_b = b0 + cr;
  // GEMV teams: tpt threads per (r, u) output of W_rec dz
  int tpt = 1;
  while (tpt < 32 && R * HU * tpt * 2 <= kThreads) tpt *= 2;
  const int team = tid / tpt, part = tid - team * tpt;
  float dc_carry = 0.f;

  for (int s = maxlen - 1; s >= 0; --s) {
    const float* dzcur = dzx + ((s + 1) & 1) * R * H6;
    float* dznxt = dzx + (s & 1) * R * H6;
    const int warp = tid >> 5;
    if (warp < R) {
      const int b = b0 + warp;
      build_lists(lat_len + (size_t)(b < B ? b : 0) * L * Kw, s_len[warp], dir, s, Kw, new_list + warp * kMaxList,
                  n_new + warp, merge_list + warp * kMaxList, n_merge + warp);
    }
    // dh_s (recurrent part) = W_hh dz_char(s + 1) + W_whh sum dz_w(words created after s)
    {
      float partial = 0.f;
      if (team < R * HU) {
        const int r = team / HU, u = team - r * HU;
        const float* w = W1 + (size_t)u * H6;
        const float* z = dzcur + r * H6;
        for (int j = part; j < H6; j += tpt) partial = fmaf(w[j], z[j], partial);
      }
      for (int o = tpt >> 1; o > 0; o >>= 1) partial += __shfl_xor_sync(0xffffffffu, partial, o);
      if (team < R * HU && part == 0) dhb[team] = partial;
    }
    __syncthreads();
    float dzi = 0.f, dzo = 0.f, dzg = 0.f, c_prev = 0.f;
    const bool live = cell_ok && s < my_len;
    const int pos = dir == 0 ? s : my_len - 1 - s;
    const size_t row = (size_t)my_b * L + pos;
    if (live) {
      const float* gp = gates + row * 6 * H + (size_t)dir * 3 * H;
      const float i_s = gp[ug], o_s = gp[H + ug], g_a = gp[2 * H + ug];
      const size_t ci = row * 2 * H + (size_t)dir * H + ug;
      const float c_t = cstate[ci], nrm = norm[ci];
      if (s > 0) c_prev = cstate[((size_t)my_b * L + (dir == 0 ? pos - 1 : pos + 1)) * 2 * H + (size_t)dir * H + ug];
      const float dh = d_out[ci] + dhb[cr * HU + cu];
      const float tc = tanhf(c_t);
      float dc = dc_carry + dh * o_s * (1.f - tc * tc);
      dzo = dh * tc * o_s * (1.f - o_s);
      float da_sum = 0.f;
      const int nm = n_merge[cr];
      if (nm == 0) {
        dzi = dc * (g_a - c_prev) * i_s * (1.f - i_s);
        dzg = dc * i_s * (1.f - g_a * g_a);
        dc_carry = dc * (1.f - i_s);
      } else {
        const float inv = 1.f / nrm, ei = expf(i_s);
        dzi = dc * (g_a - c_t) * inv * ei * i_s * (1.f - i_s);
        dzg = dc * ei * inv * (1.f - g_a * g_a);
        dc_carry = 0.f;
        for (int j = 0; j < nm; ++j) {
          const int code = merge_list[cr * kMaxList + j];
          const size_t si = ((size_t)my_b * L * Kw + code) * 2 * H + (size_t)dir * H + ug;
          const float a = aw[si], cwv = cw[si], ea = expf(a);
          const float dpre = dc * (cwv - c_t) * inv * ea * a * (1.f - a);
          da_sum += dpre;
          d_alpha[si] = dpre;
          dcw_ring[(cr * RK + ring_of(code, Kw)) * HU + cu] = dc * ea * inv;
        }
      }
      float* dx = d_xproj + row * 8 * H + (size_t)dir * 4 * H;
      dx[ug] = dzi;
      dx[H + ug] = dzo;
      dx[2 * H + ug] = dzg;
      dx[3 * H + ug] = da_sum;
    }
    int max_m = 0;
#pragma unroll
    for (int r = 0; r < R; ++r) max_m = max(max_m, n_merge[r]);
    // dc^w += W_ac da of the words merged at s
    for (int j0 = 0; j0 < max_m; j0 += kChunk) {
      if (live) {
        const int nm = n_merge[cr];
        for (int jj = 0; jj < kChunk && j0 + jj < nm; ++jj) {
          const int code = merge_list[cr * kMaxList + j0 + jj];
          const float v = d_alpha[((size_t)my_b * L * Kw + code) * 2 * H + (size_t)dir * H + ug];
          float* dst = dax + (cr * kChunk + jj) * H + ug;
          for (int q = 0; q < C; ++q) *cluster.map_shared_rank(dst, q) = v;
        }
      }
      cluster.sync();
      for (int idx = tid; idx < R * kChunk * HU; idx += blockDim.x) {
        const int r = idx / (kChunk * HU), jj = (idx / HU) % kChunk, u = idx % HU;
        if (j0 + jj >= n_merge[r]) continue;
        const float* x = dax + (r * kChunk + jj) * H;
        float acc = 0.f;
#pragma unroll 4
        for (int k = 0; k < H; ++k) acc = fmaf(x[k], W2[k * HU + u], acc);
        dcw_ring[(r * RK + ring_of(merge_list[r * kMaxList + j0 + jj], Kw)) * HU + u] += acc;
      }
      if (j0 + kChunk < max_m) cluster.sync();
      else __syncthreads();
    }
    // word cells created after step s - 1: their dc^w is complete (every merge comes later in forward order)
    float sf = 0.f, si_ = 0.f, sg = 0.f;
    if (live) {
      const int nn = n_new[cr];
      for (int j = 0; j < nn; ++j) {
        const int code = new_list[cr * kMaxList + j];
        const size_t gs = (size_t)my_b * L * Kw + code;
        const float dcw = dcw_ring[(cr * RK + ring_of(code, Kw)) * HU + cu];
        const float* wg = wgates + gs * 6 * H + (size_t)dir * 3 * H;
        const float f = wg[ug], iw = wg[H + ug], gw = wg[2 * H + ug];
        const float df = dcw * c_prev * f * (1.f - f);
        const float di = dcw * gw * iw * (1.f - iw);
        const float dg = dcw * iw * (1.f - gw * gw);
        float* dw = d_wproj + gs * 6 * H + (size_t)dir * 3 * H;
        dw[ug] = df;
        dw[H + ug] = di;
        dw[2 * H + ug] = dg;
        sf += df;
        si_ += di;
        sg += dg;
        dc_carry += dcw * f;
      }
    }
    if (cell_ok) {
      const float v[6] = {dzi, dzo, dzg, sf, si_, sg};
      for (int q = 0; q < C; ++q) {
        float* dst = cluster.map_shared_rank(dznxt + cr * H6 + ug, q);
#pragma unroll
        for (int k = 0; k < 6; ++k) dst[k * H] = v[k];
      }
    }
    cluster.sync();
  }
}

size_t fwd_smem(int H, int C, int R, int Kw) {
  const size_t HU = H / C;
  return (7 * (size_t)H * HU + 2 * R * H + R * 6 * HU + (size_t)R * kChunk * H + 2 * (size_t)R * kRing * Kw * HU) * 4 +
         ((size_t)2 * R * kMaxList + 3 * R) * 4;
}

size_t bwd_smem(int H, int C, int R, int Kw) {
  const size_t HU = H / C;
  return (7 * (size_t)H * HU + 2 * (size_t)R * 6 * H + R * HU + (size_t)R * kChunk * H + (size_t)R * kRing * Kw * HU) * 4 +
         ((size_t)2 * R * kMaxList + 3 * R) * 4;
}

constexpr size_t kSmemLimit = 226 * 1024;

// Smallest cluster (1, 2, 4, 8 CTAs, dividing H) whose weight slice and buffers fit one SM at R rows; 0 when none does.
int pick_cluster(int H, int R, int Kw) {
  for (int C = 1; C <= 8; C *= 2) {
    if (H % C != 0 || R * (H / C) > kThreads) continue;
    if (fwd_smem(H, C, R, Kw) <= kSmemLimit && bwd_smem(H, C, R, Kw) <= kSmemLimit) return C;
  }
  return 0;
}

}  // namespace

// Rows per cluster: one wave of CTAs over the SMs when the batch allows, as in bilstm.cu.
int rnn::lattice_config(int B, int H, int Kw, int num_sms, int* R_out, int* C_out) {
  if (B < 0 || H < 1 || Kw < 1) return NER_ERR_INVALID_ARG;
  if (Kw > kMaxKw) return NER_ERR_UNSUPPORTED;
  int R = 1, C = pick_cluster(H, 1, Kw);
  if (C == 0) return NER_ERR_UNSUPPORTED;
  for (int r = 2; r <= 4; r *= 2) {
    if ((long)2 * ((B + R - 1) / R) * C <= num_sms) break;
    const int c = pick_cluster(H, r, Kw);
    if (c == 0) break;
    R = r;
    C = c;
  }
  *R_out = R;
  *C_out = C;
  return NER_OK;
}

namespace {

// The instantiation of a call of `kernel`: NER_OK and (R, C) from ner_rnn_plan, or the status to return.
int check_shape(int kernel, int B, int L, int H, int Kw, int* R, int* C) {
  if (L < 1) return NER_ERR_INVALID_ARG;
  return ner_rnn_plan(kernel, B, H, Kw, ner_num_sms(), R, C, nullptr);
}

}  // namespace

extern "C" int ner_lattice_recurrence(const float* xproj, const float* wproj, const int32_t* lat_len, const float* wrec_fw,
                                      const float* wrec_bw, const float* wac_fw, const float* wac_bw,
                                      const int32_t* seq_len, float* out, int B, int L, int H, int Kw, float* gates,
                                      float* cstate, float* norm, float* wgates, float* cw, float* aw, float* hw,
                                      ner_stream_t stream) {
  int R, C;
  const int st = check_shape(NER_RNN_LATTICE_FWD, B, L, H, Kw, &R, &C);
  if (st != NER_OK) return st;
  if (B == 0) return NER_OK;
  if (!xproj || !wproj || !lat_len || !wrec_fw || !wrec_bw || !wac_fw || !wac_bw || !seq_len || !out)
    return NER_ERR_INVALID_ARG;
  const int n_saved = (gates != nullptr) + (cstate != nullptr) + (norm != nullptr) + (wgates != nullptr) +
                      (cw != nullptr) + (aw != nullptr) + (hw != nullptr);
  if (n_saved != 0 && n_saved != 7) return NER_ERR_INVALID_ARG;
  const size_t smem = fwd_smem(H, C, R, Kw);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
#define GO(RR)                                                                                                        \
  return rnn::launch_cluster(lattice_fwd_kernel<RR>, B, RR, C, kThreads, smem, s, xproj, wproj, lat_len, wrec_fw,     \
                             wrec_bw, wac_fw, wac_bw, seq_len, out, B, L, H, Kw, C, gates, cstate, norm, wgates, cw, aw, hw)
  if (R == 4) GO(4);
  if (R == 2) GO(2);
  GO(1);
#undef GO
}

extern "C" int ner_lattice_recurrence_bwd(const float* d_out, const float* gates, const float* cstate, const float* norm,
                                          const float* wgates, const float* cw, const float* aw, const int32_t* lat_len,
                                          const float* wrec_fw, const float* wrec_bw, const float* wac_fw,
                                          const float* wac_bw, const int32_t* seq_len, float* d_xproj, float* d_wproj,
                                          float* d_alpha, int B, int L, int H, int Kw, ner_stream_t stream) {
  int R, C;
  const int st = check_shape(NER_RNN_LATTICE_BWD, B, L, H, Kw, &R, &C);
  if (st != NER_OK) return st;
  if (B == 0) return NER_OK;
  if (!d_out || !gates || !cstate || !norm || !wgates || !cw || !aw || !lat_len || !wrec_fw || !wrec_bw || !wac_fw ||
      !wac_bw || !seq_len || !d_xproj || !d_wproj || !d_alpha)
    return NER_ERR_INVALID_ARG;
  const size_t smem = bwd_smem(H, C, R, Kw);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
#define GO(RR)                                                                                                         \
  return rnn::launch_cluster(lattice_bwd_kernel<RR>, B, RR, C, kThreads, smem, s, d_out, gates, cstate, norm, wgates, cw,  \
                             aw, lat_len, wrec_fw, wrec_bw, wac_fw, wac_bw, seq_len, d_xproj, d_wproj, d_alpha, B, L, H, \
                             Kw, C)
  if (R == 4) GO(4);
  if (R == 2) GO(2);
  GO(1);
#undef GO
}
