// Bidirectional GRU recurrence as a persistent thread-block-cluster kernel (sm_90a).
//
// Replaces tf.nn.bidirectional_dynamic_rnn over tf.nn.rnn_cell.GRUCell as built by reference tools/layer.py:10-41 with
// cell_type='gru' (SURVEY.md Appendix A.2):
//   r, u = split(sigmoid([x_t, h] · gates/kernel + gates/bias), 2)
//   c    = act([x_t, r ⊙ h] · candidate/kernel + candidate/bias)
//   h'   = u ⊙ h + (1 - u) ⊙ c
// zero initial state, outputs zero and state carried for t >= seq_len, the backward direction over
// reverse_sequence(x, seq_len) and reversed back.
//
// As for the LSTM (bilstm.cu), the input half ([x_t] · kernel[:D] + bias) of both matmuls is hoisted into ONE GEMM for
// both directions: xproj [rows, ld >= 6H] = x · [Wg_x_fw | Wc_x_fw | Wg_x_bw | Wc_x_bw] + biases (the GEMM's N is padded
// to its 32-column granule when 6H is not a multiple of 32).  A cluster of C CTAs owns R
// batch rows of one direction for all time steps; each CTA owns H/C hidden units and keeps their three recurrent columns
// (reset gate, update gate, candidate) resident in shared memory.  Unlike the LSTM a step has two DEPENDENT
// matrix-vector products over the full hidden state, because GRUCell applies the reset gate before the candidate's
// recurrent matmul: (r ⊙ h) · W_c^h.  So each step publishes twice through DSMEM (st.async + mbarrier):
//   1. z_r, z_u = h · W_g^h over the full h; each CTA forms r ⊙ h for its units and publishes that slice;
//   2. z_c = (r ⊙ h) · W_c^h over the gathered r ⊙ h; each CTA forms h' for its units and publishes that slice.
// Recomputing every reset gate in every CTA would save the first exchange at C times the gate work (DESIGN.md §3.4).
//
// Four lanes serve one hidden unit.  Product 1: lane q computes the reset (q < 2) or update (q >= 2) column over the even
// (q even) or odd float4s of h; product 2: lane q computes the candidate column over the float4s k4 = q (mod 4).  The
// weights are stored in the order the lanes consume them, so every step of a dot product is one conflict-free LDS.128.
#include <cooperative_groups.h>

#include "common.cuh"
#include "rnn_cluster.cuh"

namespace cg = cooperative_groups;

namespace {

template <int R, int ACT>
__global__ void __launch_bounds__(512, 1)
bigru_rec_kernel(const float* __restrict__ xproj, const float* __restrict__ wh_fw, const float* __restrict__ wh_bw,
                 const int32_t* __restrict__ seq_len, float* __restrict__ out, int B, int L, int H, int ldx, int C,
                 const int32_t* __restrict__ cu_seqlens, float* __restrict__ gates_out, float* __restrict__ hstate_out,
                 float* __restrict__ rh_out, float keep_prob, uint32_t seed_lo, uint32_t seed_hi) {
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int HU = H / C, NT = 4 * HU, H4 = H / 4;
  const int N1 = (H4 + 1) / 2, N2 = (H4 + 3) / 4;   // float4 steps of products 1 and 2 per lane
  const int ngroups = (B + R - 1) / R;
  const int cid = blockIdx.x / C;
  const int dir = cid / ngroups;
  const int b0 = (cid % ngroups) * R;
  const int tid = threadIdx.x;

  extern __shared__ __align__(16) float smem[];
  float4* W1 = reinterpret_cast<float4*>(smem);                   // [N1][NT] gate columns
  float4* W2 = W1 + (size_t)N1 * NT;                              // [N2][NT] candidate columns
  float* hbuf = reinterpret_cast<float*>(W2 + (size_t)N2 * NT);   // [2][R][H] carried h
  float* rhbuf = hbuf + 2 * R * H;                                // [2][R][H] r ⊙ h
  int* s_len = reinterpret_cast<int*>(rhbuf + 2 * R * H);         // [R] (8 ints reserved)
  uint64_t* hbar = reinterpret_cast<uint64_t*>(s_len + 8);        // [2] one mbarrier per h buffer
  uint64_t* rhbar = hbar + 2;                                     // [2] one mbarrier per r ⊙ h buffer

  const float* wh = dir == 0 ? wh_fw : wh_bw;                     // [H][3H], columns (r, u, c) x H
  for (int idx = tid; idx < N1 * NT; idx += blockDim.x) {
    const int i = idx / NT, t = idx - i * NT, q = t & 3;
    const int k0 = 4 * (2 * i + (q & 1));
    const size_t col = (size_t)(q >> 1) * H + rank * HU + (t >> 2);
    float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k0 < H) {
      w.x = wh[(size_t)(k0 + 0) * 3 * H + col];
      w.y = wh[(size_t)(k0 + 1) * 3 * H + col];
      w.z = wh[(size_t)(k0 + 2) * 3 * H + col];
      w.w = wh[(size_t)(k0 + 3) * 3 * H + col];
    }
    W1[idx] = w;
  }
  for (int idx = tid; idx < N2 * NT; idx += blockDim.x) {
    const int i = idx / NT, t = idx - i * NT, q = t & 3;
    const int k0 = 4 * (4 * i + q);
    const size_t col = (size_t)2 * H + rank * HU + (t >> 2);
    float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k0 < H) {
      w.x = wh[(size_t)(k0 + 0) * 3 * H + col];
      w.y = wh[(size_t)(k0 + 1) * 3 * H + col];
      w.z = wh[(size_t)(k0 + 2) * 3 * H + col];
      w.w = wh[(size_t)(k0 + 3) * 3 * H + col];
    }
    W2[idx] = w;
  }
  for (int idx = tid; idx < 4 * R * H; idx += blockDim.x) hbuf[idx] = 0.f;   // hbuf and rhbuf
  if (tid < R) s_len[tid] = (b0 + tid < B) ? min(max(seq_len[b0 + tid], 0), L) : 0;
  if (tid == 0) {
    for (int k = 0; k < 4; ++k) rnn::mbar_init_(&hbar[k], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  int maxlen = 0;
#pragma unroll
  for (int r = 0; r < R; ++r) maxlen = max(maxlen, s_len[r]);
  cluster.sync();  // every CTA's buffers are zeroed and its barriers initialised before anyone writes remotely

  const bool ok = tid < NT;
  const int q = tid & 3, ug = rank * HU + (tid >> 2);
  const int qb = (tid & 31) & ~3;
  // cell role: lane q of a unit's quad updates rows q, q + 4, ... (RC rows per lane)
  constexpr int RC = (R + 3) / 4;
  float hown[RC];      // carried (state-dropped) h of (row, unit ug)
  float nxr[RC], nxu[RC], nxc[RC];   // input projections of the next step, fetched one step ahead
  int lenr[RC];
  size_t xrow0[RC];
#pragma unroll
  for (int rr = 0; rr < RC; ++rr) {
    const int row = q + 4 * rr;
    hown[rr] = 0.f;
    lenr[rr] = (ok && row < R) ? s_len[row] : 0;
    const int b = b0 + row;
    xrow0[rr] = (row < R && b < B) ? (cu_seqlens ? (size_t)cu_seqlens[b] : (size_t)b * L) : 0;
  }
  auto fetch = [&](int s) {
#pragma unroll
    for (int rr = 0; rr < RC; ++rr) {
      nxr[rr] = nxu[rr] = nxc[rr] = 0.f;
      if (s < lenr[rr]) {
        const int pos = dir == 0 ? s : lenr[rr] - 1 - s;
        const float* p = xproj + (xrow0[rr] + pos) * ldx + (size_t)dir * 3 * H + ug;
        nxr[rr] = p[0];
        nxu[rr] = p[H];
        nxc[rr] = p[2 * H];
      }
    }
  };
  fetch(0);
  const uint32_t thr = nerdev::keep_threshold(keep_prob);
  const float inv_keep = 1.f / keep_prob;
  const uint32_t vec_bytes = (uint32_t)(R * H * 4);   // every CTA receives the full vector of its R rows per exchange
  const int k4a = q & 1, k4b = q;                     // first float4 of this lane in products 1 and 2

  for (int s = 0; s < maxlen; ++s) {
    const int pb = s & 1;
    const float* hcur = hbuf + pb * R * H;          // h of step s - 1
    float* hnxt = hbuf + (pb ^ 1) * R * H;          // h of step s
    float* rhcur = rhbuf + pb * R * H;              // r ⊙ h of step s
    if (tid == 0) {
      rnn::mbar_arrive_expect_tx_(&hbar[pb ^ 1], vec_bytes);
      rnn::mbar_arrive_expect_tx_(&rhbar[pb], vec_bytes);
    }
    float xr[RC], xu[RC], xc[RC];
#pragma unroll
    for (int rr = 0; rr < RC; ++rr) {
      xr[rr] = nxr[rr];
      xu[rr] = nxu[rr];
      xc[rr] = nxc[rr];
    }
    fetch(s + 1);
    if (s > 0) rnn::mbar_wait_(&hbar[pb], (uint32_t)((s - 1) >> 1) & 1u);   // h of step s-1 has landed

    // ---- product 1: reset / update pre-activations over the full h (packed FFMA2, two chains per row)
    nerdev::f32x2 pa[R], pc[R];
#pragma unroll
    for (int r = 0; r < R; ++r) pa[r] = pc[r] = nerdev::pk2(0.f, 0.f);
    if (ok) {
      const float4* h4 = reinterpret_cast<const float4*>(hcur);
#pragma unroll 4
      for (int i = 0; i < N1; ++i) {
        const float4 w = W1[i * NT + tid];
        const int k4 = min(2 * i + k4a, H4 - 1);   // past H the weights are zero
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const float4 hv = h4[r * H4 + k4];
          pa[r] = nerdev::fma2(nerdev::pk2(w.x, w.y), nerdev::pk2(hv.x, hv.y), pa[r]);
          pc[r] = nerdev::fma2(nerdev::pk2(w.z, w.w), nerdev::pk2(hv.z, hv.w), pc[r]);
        }
      }
    }
    float zr[RC], zu[RC];
#pragma unroll
    for (int rr = 0; rr < RC; ++rr) zr[rr] = zu[rr] = 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float z0, z1, z2, z3;
      nerdev::upk2(pa[r], z0, z1);
      nerdev::upk2(pc[r], z2, z3);
      float z = (z0 + z1) + (z2 + z3);
      z += __shfl_xor_sync(0xffffffffu, z, 1);
      const float a_r = __shfl_sync(0xffffffffu, z, qb + 0);
      const float a_u = __shfl_sync(0xffffffffu, z, qb + 2);
      if (q == (r & 3)) {
        zr[r >> 2] = a_r;
        zu[r >> 2] = a_u;
      }
    }
    float r_s[RC], u_s[RC], rh[RC];
#pragma unroll
    for (int rr = 0; rr < RC; ++rr) {
      const int row = q + 4 * rr;
      r_s[rr] = u_s[rr] = rh[rr] = 0.f;
      if (s < lenr[rr]) {
        r_s[rr] = rnn::sigmoid_fast(zr[rr] + xr[rr]);
        u_s[rr] = rnn::sigmoid_fast(zu[rr] + xu[rr]);
        rh[rr] = r_s[rr] * hown[rr];
      }
      if (ok && row < R)
        rnn::publish_all(nerdev::smem_u32(rhcur + row * H + ug), nerdev::smem_u32(&rhbar[pb]), rh[rr], C);
    }
    rnn::mbar_wait_(&rhbar[pb], (uint32_t)(s >> 1) & 1u);   // r ⊙ h of step s has landed

    // ---- product 2: candidate pre-activation over the gathered r ⊙ h
#pragma unroll
    for (int r = 0; r < R; ++r) pa[r] = pc[r] = nerdev::pk2(0.f, 0.f);
    if (ok) {
      const float4* g4 = reinterpret_cast<const float4*>(rhcur);
#pragma unroll 4
      for (int i = 0; i < N2; ++i) {
        const float4 w = W2[i * NT + tid];
        const int k4 = min(4 * i + k4b, H4 - 1);
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const float4 hv = g4[r * H4 + k4];
          pa[r] = nerdev::fma2(nerdev::pk2(w.x, w.y), nerdev::pk2(hv.x, hv.y), pa[r]);
          pc[r] = nerdev::fma2(nerdev::pk2(w.z, w.w), nerdev::pk2(hv.z, hv.w), pc[r]);
        }
      }
    }
    float zc[RC];
#pragma unroll
    for (int rr = 0; rr < RC; ++rr) zc[rr] = 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float z0, z1, z2, z3;
      nerdev::upk2(pa[r], z0, z1);
      nerdev::upk2(pc[r], z2, z3);
      float z = (z0 + z1) + (z2 + z3);
      z += __shfl_xor_sync(0xffffffffu, z, 1);
      z += __shfl_xor_sync(0xffffffffu, z, 2);
      if (q == (r & 3)) zc[r >> 2] = z;
    }
#pragma unroll
    for (int rr = 0; rr < RC; ++rr) {
      const int row = q + 4 * rr;
      const bool cell_ok = ok && row < R;
      const int len = lenr[rr];
      const int b = b0 + row;
      const bool live = s < len;
      const int pos = dir == 0 ? s : len - 1 - s;
      float h_out = 0.f, h_state = 0.f, c_a = 0.f;
      if (live) {
        c_a = rnn::act_fast<ACT>(zc[rr] + xc[rr]);
        h_out = h_state = u_s[rr] * hown[rr] + (1.f - u_s[rr]) * c_a;
        if (keep_prob < 1.f)   // (for GRUCell the whole state is h)
          rnn::dropout_out_state(h_out, h_state, seed_lo, seed_hi, thr, inv_keep, b, L, pos, H, dir, ug);
        hown[rr] = h_state;
      }
      // (h of a finished row is never read again — its own recurrence has stopped — so 0 is as good as the carried value)
      if (cell_ok) rnn::publish_all(nerdev::smem_u32(hnxt + row * H + ug), nerdev::smem_u32(&hbar[pb ^ 1]), h_state, C);
      if (live) {
        const size_t o = ((size_t)b * L + pos) * 2 * H + (size_t)dir * H + ug;
        out[o] = h_out;
        if (gates_out != nullptr) {   // saved for back-propagation through time (bigru_bwd.cu)
          const size_t gi = ((size_t)b * L + pos) * 6 * H + (size_t)dir * 3 * H + ug;
          gates_out[gi] = r_s[rr];
          gates_out[gi + H] = u_s[rr];
          gates_out[gi + 2 * H] = c_a;
          hstate_out[o] = h_state;
          rh_out[o] = rh[rr];
        }
      } else if (cell_ok && b < B) {
        out[((size_t)b * L + s) * 2 * H + (size_t)dir * H + ug] = 0.f;   // past this row's end: dynamic_rnn emits zeros
      }
    }
  }
  cluster.sync();   // nobody exits while a peer may still be sending into its shared memory

  // positions past the longest row of this cluster: zeros
  for (int idx = tid; idx < R * HU; idx += blockDim.x) {
    const int r = idx / HU, uu = idx - r * HU;
    const int b = b0 + r;
    if (b < B)
      for (int s = maxlen; s < L; ++s) out[((size_t)b * L + s) * 2 * H + (size_t)dir * H + rank * HU + uu] = 0.f;
  }
}

template <int R, int ACT>
int launch_rec(const float* xproj, const float* wh_fw, const float* wh_bw, const int32_t* seq_len, float* out, int B,
               int L, int H, int ldx, int C, const int32_t* cu_seqlens, float* gates_out, float* hstate_out, float* rh_out,
               float keep_prob, uint64_t seed, cudaStream_t st) {
  return rnn::launch_cluster(bigru_rec_kernel<R, ACT>, B, R, C, (4 * (H / C) + 31) / 32 * 32, rnn::gru_smem_bytes(H, C, R),
                             st, xproj, wh_fw, wh_bw, seq_len, out, B, L, H, ldx, C, cu_seqlens, gates_out, hstate_out,
                             rh_out, keep_prob, (uint32_t)seed, (uint32_t)(seed >> 32));
}

}  // namespace

extern "C" int ner_bigru_recurrence(const float* xproj, const float* wh_fw, const float* wh_bw, const int32_t* seq_len,
                                    float* out, int B, int L, int H, int ld_xproj, int activation,
                                    const int32_t* cu_seqlens,
                                    float* gates_out, float* hstate_out, float* rh_out, float keep_prob, uint64_t seed,
                                    ner_stream_t stream) {
  if (B < 0 || L < 1 || H < 1 || ld_xproj < 6 * H) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!xproj || !wh_fw || !wh_bw || !seq_len || !out) return NER_ERR_INVALID_ARG;
  if ((gates_out == nullptr) != (hstate_out == nullptr) || (gates_out == nullptr) != (rh_out == nullptr))
    return NER_ERR_INVALID_ARG;
  if (!(keep_prob > 0.f) || keep_prob > 1.f) return NER_ERR_INVALID_ARG;
  if (activation != 0 && activation != 1) return NER_ERR_INVALID_ARG;
  int R, C;
  const int status = ner_rnn_plan(NER_RNN_GRU_FWD, B, H, 0, ner_num_sms(), &R, &C, nullptr);
  if (status != NER_OK) return status;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define GO(RR)                                                                                                         \
  return activation == 1                                                                                               \
             ? launch_rec<RR, 1>(xproj, wh_fw, wh_bw, seq_len, out, B, L, H, ld_xproj, C, cu_seqlens, gates_out, hstate_out,     \
                                 rh_out, keep_prob, seed, st)                                                          \
             : launch_rec<RR, 0>(xproj, wh_fw, wh_bw, seq_len, out, B, L, H, ld_xproj, C, cu_seqlens, gates_out, hstate_out,     \
                                 rh_out, keep_prob, seed, st)
  if (R == 4) GO(4);
  if (R == 2) GO(2);
  GO(1);
#undef GO
}
