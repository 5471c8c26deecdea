// Back-propagation through time of the bidirectional GRU recurrence (sm_90a), the gradient the reference obtains from
// tf.gradients through bidirectional_dynamic_rnn(GRUCell) (reference tools/train_utils.py:383 over tools/layer.py:27-41).
//
// Same decomposition as the forward kernel (bigru.cu): a cluster of C CTAs owns R batch rows of one direction, each CTA
// owns H/C hidden units k and keeps the rows kernel[D + k, :] of both recurrent matrices resident in shared memory, four
// lanes per unit.  Walking the steps in reverse order of the forward pass, per step and owned unit (dh is the gradient
// of the cell's new h, the emitted output's and the carried state's through their dropout masks):
//   du = dh ⊙ (h_prev − c),  da_c = dh ⊙ (1 − u) ⊙ act'(c),  da_u = du ⊙ u(1 − u)
//   exchange da_c;  d(rh) = da_c · W_c^hᵀ  (owned rows k)
//   da_r = d(rh) ⊙ h_prev ⊙ r(1 − r)
//   exchange [da_r | da_u];  dh_prev = dh ⊙ u + d(rh) ⊙ r + [da_r | da_u] · W_g^hᵀ
// [da_r | da_u | da_c] is written to d_xproj, the gradient of the hoisted input projection.  dW_x, dW_h and the bias
// gradients stay GEMMs / column sums over d_xproj done by the caller.
#include <cooperative_groups.h>

#include "common.cuh"
#include "rnn_cluster.cuh"

namespace cg = cooperative_groups;

namespace {

template <int R, int ACT>
__global__ void __launch_bounds__(512, 1)
bigru_bwd_kernel(const float* __restrict__ d_out, const float* __restrict__ gates, const float* __restrict__ hstate,
                 const float* __restrict__ wh_fw, const float* __restrict__ wh_bw, const int32_t* __restrict__ seq_len,
                 float* __restrict__ d_xproj, int B, int L, int H, int C, float keep_prob, uint32_t seed_lo,
                 uint32_t seed_hi) {
  cg::cluster_group cluster = cg::this_cluster();
  const int HU = H / C, NT = 4 * HU, H4 = H / 4;
  const int M1 = (H4 + 3) / 4, M2 = (H4 + 1) / 2;   // float4 steps of the W_c^hᵀ and W_g^hᵀ products per lane
  const rnn::RowGroup grp = rnn::row_group(C, B, R);
  const int rank = grp.rank, dir = grp.dir, b0 = grp.b0;
  const int tid = threadIdx.x;

  extern __shared__ __align__(16) float smem[];
  float4* V1 = reinterpret_cast<float4*>(smem);                   // [M1][NT] rows of W_c^h
  float4* V2 = V1 + (size_t)M1 * NT;                              // [M2][NT] rows of W_g^h
  float* dcbuf = reinterpret_cast<float*>(V2 + (size_t)M2 * NT);  // [2][R][H]  da_c
  float* dgbuf = dcbuf + 2 * R * H;                               // [2][R][2H] [da_r | da_u]
  int* s_len = reinterpret_cast<int*>(dgbuf + 4 * R * H);         // [R] (8 ints reserved)
  uint64_t* dcbar = reinterpret_cast<uint64_t*>(s_len + 8);       // [2]
  uint64_t* dgbar = dcbar + 2;                                    // [2]

  const float* wh = dir == 0 ? wh_fw : wh_bw;                     // [H][3H], columns (r, u, c) x H
  for (int idx = tid; idx < M1 * NT; idx += blockDim.x) {
    const int i = idx / NT, t = idx - i * NT;
    const int j4 = 4 * i + (t & 3);
    float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
    if (j4 < H4) w = *reinterpret_cast<const float4*>(wh + (size_t)(rank * HU + (t >> 2)) * 3 * H + 2 * H + 4 * j4);
    V1[idx] = w;
  }
  for (int idx = tid; idx < M2 * NT; idx += blockDim.x) {
    const int i = idx / NT, t = idx - i * NT;
    const int j4 = 4 * i + (t & 3);
    float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
    if (j4 < 2 * H4) w = *reinterpret_cast<const float4*>(wh + (size_t)(rank * HU + (t >> 2)) * 3 * H + 4 * j4);
    V2[idx] = w;
  }
  for (int idx = tid; idx < 6 * R * H; idx += blockDim.x) dcbuf[idx] = 0.f;   // dcbuf and dgbuf
  if (tid == 0) {
    for (int k = 0; k < 4; ++k) rnn::mbar_init_(&dcbar[k], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  const int maxlen = rnn::load_lengths<R>(s_len, seq_len, b0, B, L);
  cluster.sync();
  rnn::zero_unvisited<3>(d_xproj, s_len, R, b0, B, L, H, dir, rank, HU);

  const bool ok = tid < NT;
  const int q = tid & 3, ug = rank * HU + (tid >> 2);
  constexpr int RC = (R + 3) / 4;
  int lenr[RC];
  float dhrec[RC];   // gradient reaching the carried state of (row, unit ug) from the later steps
  // saved operands of the next step to walk, fetched one step ahead so their latency overlaps the current step
  float n_r[RC], n_u[RC], n_c[RC], n_hp[RC], n_do[RC];
#pragma unroll
  for (int rr = 0; rr < RC; ++rr) {
    lenr[rr] = (ok && q + 4 * rr < R) ? s_len[q + 4 * rr] : 0;
    dhrec[rr] = 0.f;
  }
  auto fetch = [&](int s) {
#pragma unroll
    for (int rr = 0; rr < RC; ++rr) {
      n_r[rr] = n_u[rr] = n_c[rr] = n_hp[rr] = n_do[rr] = 0.f;
      const int len = lenr[rr];
      if (s >= 0 && s < len) {
        const size_t b = (size_t)(b0 + q + 4 * rr);
        const int pos = dir == 0 ? s : len - 1 - s;
        const float* g = gates + (b * L + pos) * 6 * H + (size_t)dir * 3 * H + ug;
        n_r[rr] = g[0];
        n_u[rr] = g[H];
        n_c[rr] = g[2 * H];
        if (s > 0) {
          const int ppos = dir == 0 ? s - 1 : len - s;   // position of forward step s-1
          n_hp[rr] = hstate[(b * L + ppos) * 2 * H + (size_t)dir * H + ug];
        }
        n_do[rr] = d_out[(b * L + pos) * 2 * H + (size_t)dir * H + ug];
      }
    }
  };
  fetch(maxlen - 1);
  const uint32_t thr = nerdev::keep_threshold(keep_prob);
  const float inv_keep = 1.f / keep_prob;
  const uint32_t c_bytes = (uint32_t)(R * H * 4), g_bytes = 2 * c_bytes;

  for (int s = maxlen - 1, n = 0; s >= 0; --s, ++n) {
    const int pb = n & 1;
    float* dccur = dcbuf + pb * R * H;
    float* dgcur = dgbuf + pb * 2 * R * H;
    if (tid == 0) {
      rnn::mbar_arrive_expect_tx_(&dcbar[pb], c_bytes);
      rnn::mbar_arrive_expect_tx_(&dgbar[pb], g_bytes);
    }
    float r_s[RC], u_s[RC], hp[RC], dh[RC], dau[RC], dac[RC];
    size_t gi[RC];
#pragma unroll
    for (int rr = 0; rr < RC; ++rr) {
      const int row = q + 4 * rr;
      const int len = lenr[rr];
      const bool live = s < len;
      const int b = b0 + row;
      const int pos = dir == 0 ? s : len - 1 - s;
      r_s[rr] = n_r[rr];
      u_s[rr] = n_u[rr];
      hp[rr] = n_hp[rr];
      const float c_a = n_c[rr];
      float dh_o = n_do[rr], dh_s = dhrec[rr];
      dh[rr] = dau[rr] = dac[rr] = 0.f;
      gi[rr] = ((size_t)b * L + pos) * 6 * H + (size_t)dir * 3 * H + ug;
      if (live) {
        if (keep_prob < 1.f)   // the forward's DropoutWrapper masks (output / state)
          rnn::dropout_out_state(dh_o, dh_s, seed_lo, seed_hi, thr, inv_keep, b, L, pos, H, dir, ug);
        dh[rr] = dh_o + dh_s;
        dac[rr] = dh[rr] * (1.f - u_s[rr]) * rnn::act_grad_from_output<ACT>(c_a);
        dau[rr] = dh[rr] * (hp[rr] - c_a) * u_s[rr] * (1.f - u_s[rr]);
      }
      if (ok && row < R) rnn::publish_all(nerdev::smem_u32(dccur + row * H + ug), nerdev::smem_u32(&dcbar[pb]), dac[rr], C);
      if (live) {
        d_xproj[gi[rr] + H] = dau[rr];
        d_xproj[gi[rr] + 2 * H] = dac[rr];
      }
    }
    fetch(s - 1);
    rnn::mbar_wait_(&dcbar[pb], (uint32_t)(n >> 1) & 1u);

    // ---- d(rh)[k] = sum_j da_c[j] W_c^h[k, j]
    nerdev::f32x2 pa[R], pc[R];
#pragma unroll
    for (int r = 0; r < R; ++r) pa[r] = pc[r] = nerdev::pk2(0.f, 0.f);
    if (ok) {
      const float4* d4 = reinterpret_cast<const float4*>(dccur);
#pragma unroll 4
      for (int i = 0; i < M1; ++i) {
        const int j4 = min(4 * i + q, H4 - 1);   // past H the weights are zero
        rnn::fma2_rows<R>(pa, pc, V1[i * NT + tid], d4, H4, j4);
      }
    }
    float drh[RC];
#pragma unroll
    for (int rr = 0; rr < RC; ++rr) drh[rr] = 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float z = rnn::sum_chains(pa[r], pc[r]);
      z += __shfl_xor_sync(0xffffffffu, z, 1);
      z += __shfl_xor_sync(0xffffffffu, z, 2);
      if (q == (r & 3)) drh[r >> 2] = z;
    }
    float part[RC];
#pragma unroll
    for (int rr = 0; rr < RC; ++rr) {
      const int row = q + 4 * rr;
      const bool live = s < lenr[rr];
      float dar = 0.f;
      part[rr] = 0.f;
      if (live) {
        dar = drh[rr] * hp[rr] * r_s[rr] * (1.f - r_s[rr]);
        part[rr] = dh[rr] * u_s[rr] + drh[rr] * r_s[rr];
        d_xproj[gi[rr]] = dar;
      }
      if (ok && row < R) {
        const uint32_t lb = nerdev::smem_u32(&dgbar[pb]);
        rnn::publish_all(nerdev::smem_u32(dgcur + row * 2 * H + ug), lb, dar, C);
        rnn::publish_all(nerdev::smem_u32(dgcur + row * 2 * H + H + ug), lb, dau[rr], C);
      }
    }
    rnn::mbar_wait_(&dgbar[pb], (uint32_t)(n >> 1) & 1u);

    // ---- dh_prev[k] = dh u + d(rh) r + sum_j [da_r | da_u][j] W_g^h[k, j]
#pragma unroll
    for (int r = 0; r < R; ++r) pa[r] = pc[r] = nerdev::pk2(0.f, 0.f);
    if (ok) {
      const float4* d4 = reinterpret_cast<const float4*>(dgcur);
#pragma unroll 4
      for (int i = 0; i < M2; ++i) {
        const int j4 = min(4 * i + q, 2 * H4 - 1);
        rnn::fma2_rows<R>(pa, pc, V2[i * NT + tid], d4, 2 * H4, j4);
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float z = rnn::sum_chains(pa[r], pc[r]);
      z += __shfl_xor_sync(0xffffffffu, z, 1);
      z += __shfl_xor_sync(0xffffffffu, z, 2);
      // a finished row carries the recurrent gradient through unchanged (dynamic_rnn copies its state)
      if (q == (r & 3) && s < lenr[r >> 2]) dhrec[r >> 2] = part[r >> 2] + z;
    }
  }
  cluster.sync();   // nobody exits while a peer may still be sending into its shared memory
}

template <int R, int ACT>
int launch_bwd(const float* d_out, const float* gates, const float* hstate, const float* wh_fw, const float* wh_bw,
               const int32_t* seq_len, float* d_xproj, int B, int L, int H, int C, float keep_prob, uint64_t seed,
               cudaStream_t st) {
  return rnn::launch_cluster(bigru_bwd_kernel<R, ACT>, B, R, C, (4 * (H / C) + 31) / 32 * 32, rnn::gru_smem_bytes(H, C, R),
                             st, d_out, gates, hstate, wh_fw, wh_bw, seq_len, d_xproj, B, L, H, C, keep_prob,
                             (uint32_t)seed, (uint32_t)(seed >> 32));
}

}  // namespace

extern "C" int ner_bigru_recurrence_bwd(const float* d_out, const float* gates, const float* hstate, const float* wh_fw,
                                        const float* wh_bw, const int32_t* seq_len, float* d_xproj, int B, int L, int H,
                                        int activation, float keep_prob, uint64_t seed, ner_stream_t stream) {
  if (B < 0 || L < 1 || H < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!d_out || !gates || !hstate || !wh_fw || !wh_bw || !seq_len || !d_xproj) return NER_ERR_INVALID_ARG;
  if (!(keep_prob > 0.f) || keep_prob > 1.f) return NER_ERR_INVALID_ARG;
  if (activation != 0 && activation != 1) return NER_ERR_INVALID_ARG;
  int R, C;
  const int status = ner_rnn_plan(NER_RNN_GRU_BWD, B, H, 0, ner_num_sms(), &R, &C, nullptr);
  if (status != NER_OK) return status;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define GO(RR)                                                                                                       \
  return activation == 1 ? launch_bwd<RR, 1>(d_out, gates, hstate, wh_fw, wh_bw, seq_len, d_xproj, B, L, H, C,      \
                                             keep_prob, seed, st)                                                    \
                         : launch_bwd<RR, 0>(d_out, gates, hstate, wh_fw, wh_bw, seq_len, d_xproj, B, L, H, C,      \
                                             keep_prob, seed, st)
  if (R == 4) GO(4);
  if (R == 2) GO(2);
  GO(1);
#undef GO
}
