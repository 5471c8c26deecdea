// BiLSTM recurrence as a persistent thread-block-cluster kernel (sm_90a).
//
// Replaces tf.nn.bidirectional_dynamic_rnn over tf.nn.rnn_cell.LSTMCell as built by
// reference tools/layer.py:10-41 (gate order i,j,f,o; forget_bias 1.0; zero initial state;
// outputs zero and state carried for t >= seq_len; the backward direction runs over
// reverse_sequence(x, seq_len) and is reversed back — SURVEY.md Appendix A.2).
//
// The input half of the LSTMCell matmul ([x_t] · kernel[:D]) + bias is hoisted out of the
// recurrence into ONE wgmma GEMM for both directions (xproj [B*L, 8H], gemm_tc.cu).  This
// kernel runs the sequential half: a cluster of C CTAs owns R batch rows of one direction for
// all time steps.  Each CTA keeps its slice of the recurrent matrix kernel[D:, :] resident in
// shared memory for the whole sequence (fp32, [H][4*H/C] laid out so one LDS.128 yields four
// consecutive k for one gate column), computes the 4*H/C gate pre-activations of its H/C
// hidden units, applies the cell, and broadcasts the new h slice to every CTA of the cluster
// through distributed shared memory; one cluster barrier per time step.
#include <cooperative_groups.h>

#include "common.cuh"
#include "rnn_cluster.cuh"

namespace cg = cooperative_groups;

namespace {

// H4REG > 0: this thread's gate column of W_h (H4REG float4 = H fp32 values) is register-resident
// for the whole sequence (H <= 128); H4REG == 0: the slice is read from shared memory each step.
template <int R, int ACT, int H4REG>
__global__ void __launch_bounds__(H4REG > 0 ? 256 : 512, 1) bilstm_rec_kernel(const float* __restrict__ xproj, const float* __restrict__ wh_fw,
                                  const float* __restrict__ wh_bw, const int32_t* __restrict__ seq_len,
                                  float* __restrict__ out, int B, int L, int H, int C, float forget_bias,
                                  const int32_t* __restrict__ cu_seqlens, float* __restrict__ gates_out,
                                  float* __restrict__ cstate_out, float* __restrict__ hstate_out, float keep_prob,
                                  uint32_t seed_lo, uint32_t seed_hi) {
  cg::cluster_group cluster = cg::this_cluster();
  const int HU = H / C;       // hidden units owned by this CTA
  const int NC = 4 * HU;      // gate columns owned by this CTA
  const int H4 = H / 4;
  const rnn::RowGroup grp = rnn::row_group(C, B, R);
  const int rank = grp.rank, dir = grp.dir, b0 = grp.b0;
  const int tid = threadIdx.x;

  extern __shared__ __align__(16) float smem[];
  constexpr bool WREG = H4REG > 0;
  float4* Ws4 = reinterpret_cast<float4*>(smem);                 // [H4][NC] float4 (4 consecutive k), smem path only
  float* hbuf = smem + (WREG ? 0 : (size_t)H * NC);              // [2][R][H]
  int* s_len = reinterpret_cast<int*>(hbuf + 2 * R * H);         // [R] (8 ints reserved)
  uint64_t* hbar = reinterpret_cast<uint64_t*>(s_len + 8);      // [2] one mbarrier per h buffer

  const float* wh = dir == 0 ? wh_fw : wh_bw;                    // [H][4H], columns (i,j,f,o) x H
  float4 wreg[WREG ? H4REG : 1];
  if constexpr (WREG) {
    if (tid < NC) {
      const int g0 = tid & 3, u0 = tid >> 2;   // unit-major: the 4 gates of a hidden unit sit in 4 adjacent lanes
      const size_t gc = (size_t)g0 * H + rank * HU + u0;
#pragma unroll
      for (int k4 = 0; k4 < H4REG; ++k4) {
        wreg[k4].x = wh[(size_t)(4 * k4 + 0) * 4 * H + gc];
        wreg[k4].y = wh[(size_t)(4 * k4 + 1) * 4 * H + gc];
        wreg[k4].z = wh[(size_t)(4 * k4 + 2) * 4 * H + gc];
        wreg[k4].w = wh[(size_t)(4 * k4 + 3) * 4 * H + gc];
      }
    }
  } else {
    for (int idx = tid; idx < H4 * NC; idx += blockDim.x) {
      const int k4 = idx / NC, col = idx - k4 * NC;
      const int g = col & 3, u = col >> 2;
      const size_t gc = (size_t)g * H + rank * HU + u;
      float4 w;
      w.x = wh[(size_t)(4 * k4 + 0) * 4 * H + gc];
      w.y = wh[(size_t)(4 * k4 + 1) * 4 * H + gc];
      w.z = wh[(size_t)(4 * k4 + 2) * 4 * H + gc];
      w.w = wh[(size_t)(4 * k4 + 3) * 4 * H + gc];
      Ws4[idx] = w;
    }
  }
  for (int idx = tid; idx < 2 * R * H; idx += blockDim.x) hbuf[idx] = 0.f;
  if (tid == 0) {
    rnn::mbar_init_(&hbar[0], 1);
    rnn::mbar_init_(&hbar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  const int maxlen = rnn::load_lengths<R>(s_len, seq_len, b0, B, L);
  cluster.sync();  // every CTA's hbuf is zeroed before anyone writes remotely

  // Thread t < NC owns gate g = t & 3 of hidden unit u = t >> 2 (of this CTA's slice): the four
  // pre-activations of a unit live in four adjacent lanes, so the cell update gathers them with
  // three shuffles — no shared-memory round trip and no CTA barrier between the dot products and
  // the cell; the only synchronisation per time step is the (cluster) barrier that publishes h.
  const bool col_ok = tid < NC;
  const int g = tid & 3, u = tid >> 2;
  const int ug = rank * HU + u;
  const size_t xcol = (size_t)dir * 4 * H + (size_t)g * H + ug;
  // cell role: lane g of a unit's quad updates rows r = g, g + 4, ... (RC = ceil(R / 4) rows per lane; R <= 4: one row, all
  // R cell updates in parallel)
  constexpr int RC = (R + 3) / 4;
  float c_state[RC];
#pragma unroll
  for (int rr = 0; rr < RC; ++rr) c_state[rr] = 0.f;

  // xproj row of (row r, position pos): padded layout b*L + pos, or packed layout cu_seqlens[b] + pos
  size_t xrow0[R];
#pragma unroll
  for (int r = 0; r < R; ++r)
    xrow0[r] = (b0 + r < B) ? (cu_seqlens ? (size_t)cu_seqlens[b0 + r] : (size_t)(b0 + r) * L) : 0;
  float xp[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    xp[r] = 0.f;
    const int len = s_len[r];
    if (col_ok && 0 < len) {
      const int pos = dir == 0 ? 0 : len - 1;
      xp[r] = xproj[(xrow0[r] + pos) * 8 * H + xcol];
    }
  }
  const uint32_t thr = nerdev::keep_threshold(keep_prob);
  const float inv_keep = 1.f / keep_prob;

  const uint32_t h_bytes = (uint32_t)(R * H * 4);   // every CTA receives the full h of its R rows each step
  for (int s = 0; s < maxlen; ++s) {
    const float* hcur = hbuf + (s & 1) * R * H;
    float* hnxt = hbuf + ((s + 1) & 1) * R * H;
    if (C > 1) {
      if (tid == 0) rnn::mbar_arrive_expect_tx_(&hbar[(s + 1) & 1], h_bytes);   // arm the buffer written this step
      if (s > 0) rnn::mbar_wait_(&hbar[s & 1], (uint32_t)((s - 1) >> 1) & 1u);   // h of step s-1 has landed (k-th use of the buffer)
    }
    nerdev::f32x2 pa[R], pb[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      pa[r] = nerdev::pk2(xp[r], 0.f);
      pb[r] = nerdev::pk2(0.f, 0.f);
    }
    if (col_ok) {
      // prefetch next step's input projection while the dot products run
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int len = s_len[r];
        xp[r] = 0.f;
        if (s + 1 < len) {
          const int pos = dir == 0 ? s + 1 : len - 2 - s;
          xp[r] = xproj[(xrow0[r] + pos) * 8 * H + xcol];
        }
      }
      const float4* hc4 = reinterpret_cast<const float4*>(hcur);
      if constexpr (WREG) {
#pragma unroll
        for (int k4 = 0; k4 < H4REG; ++k4) rnn::fma2_rows<R>(pa, pb, wreg[k4], hc4, H4, k4);
      } else {
#pragma unroll 4
        for (int k4 = 0; k4 < H4; ++k4) rnn::fma2_rows<R>(pa, pb, Ws4[k4 * NC + tid], hc4, H4, k4);
      }
    }
    // quad transpose: lane g of the quad receives (z_i, z_j, z_f, z_o) of its rows g, g + 4, ...
    float zi[RC], zj[RC], zf[RC], zo[RC];
#pragma unroll
    for (int rr = 0; rr < RC; ++rr) zi[rr] = zj[rr] = zf[rr] = zo[rr] = 0.f;
    const int qb = (tid & 31) & ~3;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const float z = rnn::sum_chains(pa[r], pb[r]);
      const float a0 = __shfl_sync(0xffffffffu, z, qb + 0);
      const float a1 = __shfl_sync(0xffffffffu, z, qb + 1);
      const float a2 = __shfl_sync(0xffffffffu, z, qb + 2);
      const float a3 = __shfl_sync(0xffffffffu, z, qb + 3);
      if (g == (r & 3)) {
        zi[r >> 2] = a0;
        zj[r >> 2] = a1;
        zf[r >> 2] = a2;
        zo[r >> 2] = a3;
      }
    }
    // h is published with st.async + mbarrier transaction bytes (see the helpers above): with
    // barrier.cluster the release fence of the arrive stalled every step until this thread's global stores
    // had been acknowledged (ncu: 20 % of the kernel's samples on the barrier's ERRBAR) and the wait
    // invalidated L1.
#pragma unroll
    for (int rr = 0; rr < RC; ++rr) {
      const int r = g + 4 * rr;
      const bool cell_ok = col_ok && r < R;
      float i_s = 0.f, j_a = 0.f, f_s = 0.f, o_s = 0.f, h_out = 0.f, h_state = 0.f;
      const int len = cell_ok ? s_len[r] : 0;
      const int b = b0 + r;
      const bool live = cell_ok && s < len;
      const int pos = dir == 0 ? s : len - 1 - s;
      if (live) {
        i_s = rnn::sigmoid_fast(zi[rr]);
        j_a = rnn::act_fast<ACT>(zj[rr]);
        f_s = rnn::sigmoid_fast(zf[rr] + forget_bias);
        o_s = rnn::sigmoid_fast(zo[rr]);
        c_state[rr] = f_s * c_state[rr] + i_s * j_a;
        h_out = h_state = o_s * rnn::act_fast<ACT>(c_state[rr]);
        if (keep_prob < 1.f)   // (c is not dropped)
          rnn::dropout_out_state(h_out, h_state, seed_lo, seed_hi, thr, inv_keep, b, L, pos, H, dir, ug);
      }
      if (cell_ok) {
        // (h of a finished row is never read again — its own recurrence has stopped — so 0 is as good as
        // the carried value dynamic_rnn keeps)
        if (C > 1) {
          const uint32_t la = nerdev::smem_u32(hnxt + r * H + ug), lb = nerdev::smem_u32(&hbar[(s + 1) & 1]);
          rnn::publish_all(la, lb, h_state, C);
        } else {
          hnxt[r * H + ug] = h_state;
        }
      }
      if (live) {
        out[((size_t)b * L + pos) * 2 * H + (size_t)dir * H + ug] = h_out;
        if (hstate_out != nullptr) hstate_out[((size_t)b * L + pos) * 2 * H + (size_t)dir * H + ug] = h_state;
        if (gates_out != nullptr) {  // saved for back-propagation through time (bilstm_bwd.cu)
          const size_t gi = ((size_t)b * L + pos) * 8 * H + (size_t)dir * 4 * H;
          gates_out[gi + 0 * H + ug] = i_s;
          gates_out[gi + 1 * H + ug] = j_a;
          gates_out[gi + 2 * H + ug] = f_s;
          gates_out[gi + 3 * H + ug] = o_s;
          cstate_out[((size_t)b * L + pos) * 2 * H + (size_t)dir * H + ug] = c_state[rr];
        }
      } else if (cell_ok && b < B) {
        out[((size_t)b * L + s) * 2 * H + (size_t)dir * H + ug] = 0.f;   // past this row's end: dynamic_rnn emits zeros
      }
    }
    if (C == 1) __syncthreads();
  }
  if (C > 1) cluster.sync();   // nobody exits while a peer may still be sending into its shared memory
  rnn::zero_past_maxlen(out, R, b0, B, L, H, dir, rank, HU, maxlen);
}

template <int R, int ACT, int H4REG>
int launch_rec(const float* xproj, const float* wh_fw, const float* wh_bw, const int32_t* seq_len, float* out, int B,
               int L, int H, int C, float forget_bias, const int32_t* cu_seqlens, float* gates_out, float* cstate_out,
               float* hstate_out, float keep_prob, uint64_t seed, cudaStream_t st) {
  const int HU = H / C, NC = 4 * HU;
  const size_t smem = ((H4REG > 0 ? 0 : (size_t)H * NC) + 2 * R * H + 32) * 4;   // + s_len[8] + 2 mbarriers (16-B aligned: R*H even)
  return rnn::launch_cluster(bilstm_rec_kernel<R, ACT, H4REG>, B, R, C, (NC + 31) / 32 * 32, smem, st, xproj, wh_fw, wh_bw,
                             seq_len, out, B, L, H, C, forget_bias, cu_seqlens, gates_out, cstate_out, hstate_out,
                             keep_prob, (uint32_t)seed, (uint32_t)(seed >> 32));
}

}  // namespace

extern "C" int ner_bilstm_recurrence(const float* xproj, const float* wh_fw, const float* wh_bw,
                                     const int32_t* seq_len, float* out, int B, int L, int H, int activation,
                                     float forget_bias, const int32_t* cu_seqlens, float* gates_out,
                                     float* cstate_out, float* hstate_out, float keep_prob, uint64_t seed,
                                     ner_stream_t stream) {
  if (B < 0 || L < 1 || H < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!xproj || !wh_fw || !wh_bw || !seq_len || !out) return NER_ERR_INVALID_ARG;
  if ((gates_out == nullptr) != (cstate_out == nullptr)) return NER_ERR_INVALID_ARG;
  if (!(keep_prob > 0.f) || keep_prob > 1.f) return NER_ERR_INVALID_ARG;
  if (activation != 0 && activation != 1) return NER_ERR_INVALID_ARG;
  int R, C, resident;
  const int status = ner_rnn_plan(NER_RNN_LSTM_FWD, B, H, 0, ner_num_sms(), &R, &C, &resident);
  if (status != NER_OK) return status;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define GO(RR, HR)                                                                                          \
  return activation == 1 ? launch_rec<RR, 1, HR>(xproj, wh_fw, wh_bw, seq_len, out, B, L, H, C, forget_bias, cu_seqlens, gates_out, cstate_out, hstate_out, keep_prob, seed, st) \
                         : launch_rec<RR, 0, HR>(xproj, wh_fw, wh_bw, seq_len, out, B, L, H, C, forget_bias, cu_seqlens, gates_out, cstate_out, hstate_out, keep_prob, seed, st)
  if (resident) {   // register-resident W_h (H = 128: the bert_bilstm_crf / bilstm_crf shape)
    if (R == 8) GO(8, 32);
    if (R == 2) GO(2, 32);
    GO(1, 32);
  }
  if (R == 4) GO(4, 0);
  if (R == 2) GO(2, 0);
  GO(1, 0);
#undef GO
}
