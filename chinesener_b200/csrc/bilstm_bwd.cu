// Back-propagation-through-time of the BiLSTM recurrence (sm_90a), the gradient the reference
// obtains from tf.gradients through bidirectional_dynamic_rnn (reference tools/train_utils.py:383
// over tools/layer.py:27-41).
//
// Same decomposition as the forward kernel (bilstm.cu): a cluster of C CTAs owns R batch rows of
// one direction; each CTA owns H/C hidden units (all four gates of them) and keeps the rows
// kernel[D + k, :] of the recurrent matrix for ITS units k resident (fp32, registers for H = 128,
// shared memory otherwise).  Walking the steps in reverse order of the forward pass, per step:
//   1. gate gradients dz (4 per owned unit) from d_out + the recurrent dh, the carried dc and the
//      gate activations / cell states saved by the forward pass; dz is written to d_xproj (the
//      gradient of the hoisted input projection: dW_x, dx and the bias gradient are plain GEMMs /
//      reductions over it) and broadcast to every CTA of the cluster through DSMEM;
//   2. dh_prev[k] = sum_col dz[col] * kernel[D + k, col] for the owned units k.
// dW_h = sum_t h_{t-1}^T dz_t is NOT accumulated here: it is one tensor-core GEMM over
// (h_prev [B*L, H], d_xproj [B*L, 4H]) done by the caller.
#include <cooperative_groups.h>

#include "common.cuh"
#include "rnn_cluster.cuh"

namespace cg = cooperative_groups;

namespace {

// exact tanhf, not the forward kernel's ex2.approx form (rnn::act_fast)
template <int ACT>
__device__ __forceinline__ float actf(float x) {
  if (ACT == 1) return fmaxf(x, 0.f);
  return tanhf(x);
}

// gates: [B, L, 2, 4H] post-activation (sigmoid(i), act(j), sigmoid(f + forget_bias), sigmoid(o));
// cstate: [B, L, 2, H] cell state after the step; both indexed by the ORIGINAL position of the step.
// WR > 0 (H = 128): the recurrent matrix slice lives in REGISTERS — thread (k, part) = (tid / 4, tid % 4) keeps
// kernel[D + rank*HU + k, part*WR .. part*WR + WR) and forms dh_prev[r][k] for all R rows from float4 reads of the gathered
// gate gradients (one address per `part` in a warp -> broadcasts; the per-part padding of 4 floats keeps the four parts on
// different banks).  The shared-memory walk it replaces issued two LDS per FMA.
template <int R, int ACT, int WR>
__global__ void __launch_bounds__(WR > 0 ? 256 : 512, 1)
bilstm_bwd_kernel(const float* __restrict__ d_out, const float* __restrict__ gates, const float* __restrict__ cstate,
                  const float* __restrict__ wh_fw, const float* __restrict__ wh_bw, const int32_t* __restrict__ seq_len,
                  float* __restrict__ d_xproj, int B, int L, int H, int C, float keep_prob, uint32_t seed_lo,
                  uint32_t seed_hi) {
  cg::cluster_group cluster = cg::this_cluster();
  const int HU = H / C, G4 = 4 * H;
  const rnn::RowGroup grp = rnn::row_group(C, B, R);
  const int rank = grp.rank, dir = grp.dir, b0 = grp.b0;
  const int tid = threadIdx.x;

  extern __shared__ __align__(16) float smem[];
  float* Wt = smem;                          // [4H][HU+1]: Wt[col][k] = kernel[D + rank*HU + k, col]   (WR == 0 only)
  const int WP = HU + 1;
  const int G4P = WR > 0 ? G4 + 4 * (G4 / (WR > 0 ? WR : 1)) : G4;     // padded row of the gathered dz (WR path)
  float* dzbuf = Wt + (WR > 0 ? (size_t)0 : (size_t)G4 * WP);           // [2][R][G4P] all-gathered gate gradients
  float* dhbuf = dzbuf + 2 * R * G4P;        // [R][HU]      recurrent dh for the owned units
  auto dzi_of = [&](int col) -> int { return WR > 0 ? col + 4 * (col / (WR > 0 ? WR : 1)) : col; };
  int* s_len = reinterpret_cast<int*>(dhbuf + R * HU);

  const float* wh = dir == 0 ? wh_fw : wh_bw;  // [H][4H]
  float wreg[WR > 0 ? WR : 1];
  if (WR > 0) {
    const int k = tid >> 2, part = tid & 3;
    if (k < HU) {
#pragma unroll
      for (int c = 0; c < (WR > 0 ? WR : 1); c += 4) {
        const float4 v = *reinterpret_cast<const float4*>(wh + (size_t)(rank * HU + k) * G4 + part * WR + c);
        wreg[c] = v.x; wreg[c + 1] = v.y; wreg[c + 2] = v.z; wreg[c + 3] = v.w;
      }
    }
  } else {
    for (int idx = tid; idx < HU * G4; idx += blockDim.x) {
      const int k = idx / G4, col = idx - k * G4;
      Wt[col * WP + k] = wh[(size_t)(rank * HU + k) * G4 + col];
    }
  }
  for (int idx = tid; idx < 2 * R * G4P; idx += blockDim.x) dzbuf[idx] = 0.f;
  for (int idx = tid; idx < R * HU; idx += blockDim.x) dhbuf[idx] = 0.f;
  const int maxlen = rnn::load_lengths<R>(s_len, seq_len, b0, B, L);
  cluster.sync();

  // cell role: thread (r, u) for tid < R*HU
  const bool cell_ok = tid < R * HU;
  const int cr = cell_ok ? tid / HU : 0, cu = cell_ok ? tid - cr * HU : 0;
  float dc_carry = 0.f;

  rnn::zero_unvisited<4>(d_xproj, s_len, R, b0, B, L, H, dir, rank, HU);

  // Per-step operands (saved gates, cell states, upstream gradient) do not depend on the recurrence: they are
  // fetched one step ahead so their L2/HBM latency overlaps the previous step instead of heading its chain.
  const int my_len = cell_ok ? s_len[cr] : 0;
  const int my_b = b0 + cr;
  const int ug = rank * HU + cu;
  float n_i = 0.f, n_j = 0.f, n_f = 0.f, n_o = 0.f, n_c = 0.f, n_cp = 0.f, n_dho = 0.f;
  auto fetch = [&](int s) {
    if (cell_ok && s >= 0 && s < my_len) {
      const int pos = dir == 0 ? s : my_len - 1 - s;
      const size_t gi = ((size_t)my_b * L + pos) * 2 * G4 + (size_t)dir * G4;
      n_i = gates[gi + 0 * H + ug];
      n_j = gates[gi + 1 * H + ug];
      n_f = gates[gi + 2 * H + ug];
      n_o = gates[gi + 3 * H + ug];
      n_c = cstate[((size_t)my_b * L + pos) * 2 * H + (size_t)dir * H + ug];
      n_cp = 0.f;
      if (s > 0) {
        const int ppos = dir == 0 ? s - 1 : my_len - s;  // position of forward step s-1
        n_cp = cstate[((size_t)my_b * L + ppos) * 2 * H + (size_t)dir * H + ug];
      }
      n_dho = d_out[((size_t)my_b * L + pos) * 2 * H + (size_t)dir * H + ug];
    }
  };
  fetch(maxlen - 1);

  for (int s = maxlen - 1; s >= 0; --s) {
    float* dzcur = dzbuf + (s & 1) * R * G4P;
    float dzi = 0.f, dzj = 0.f, dzf = 0.f, dzo = 0.f;
    const bool live = cell_ok && s < my_len;
    const float i_s = n_i, j_a = n_j, f_s = n_f, o_s = n_o, c_t = n_c, c_prev = n_cp;
    float dh_o = n_dho;
    fetch(s - 1);
    const int pos = dir == 0 ? s : my_len - 1 - s;
    const size_t gi = ((size_t)my_b * L + pos) * 2 * G4 + (size_t)dir * G4;
    if (live) {
      float dh_s = dhbuf[cr * HU + cu];
      if (keep_prob < 1.f)   // the forward's DropoutWrapper masks (output / state)
        rnn::dropout_out_state(dh_o, dh_s, seed_lo, seed_hi, nerdev::keep_threshold(keep_prob), 1.f / keep_prob, my_b, L,
                               pos, H, dir, ug);
      const float dh = dh_o + dh_s;
      const float ac = actf<ACT>(c_t);
      const float d_o = dh * ac;
      const float dc = dh * o_s * rnn::act_grad_from_output<ACT>(ac) + dc_carry;
      dzi = dc * j_a * i_s * (1.f - i_s);
      dzj = dc * i_s * rnn::act_grad_from_output<ACT>(j_a);
      dzf = dc * c_prev * f_s * (1.f - f_s);
      dzo = d_o * o_s * (1.f - o_s);
      dc_carry = dc * f_s;
    }
    if (cell_ok) {
      // broadcast this unit's four gate gradients to every CTA (global column order g*H + ug)
      for (int dst = 0; dst < C; ++dst) {
        float* remote = cluster.map_shared_rank(dzcur, dst);
        remote[cr * G4P + dzi_of(0 * H + ug)] = dzi;
        remote[cr * G4P + dzi_of(1 * H + ug)] = dzj;
        remote[cr * G4P + dzi_of(2 * H + ug)] = dzf;
        remote[cr * G4P + dzi_of(3 * H + ug)] = dzo;
      }
    }
    // arrive before this step's global stores: the barrier's release fence then does not wait for them
    cluster.barrier_arrive();
    if (live) {
      d_xproj[gi + 0 * H + ug] = dzi;
      d_xproj[gi + 1 * H + ug] = dzj;
      d_xproj[gi + 2 * H + ug] = dzf;
      d_xproj[gi + 3 * H + ug] = dzo;
    }
    cluster.barrier_wait();
    // dh_prev[r][k] for owned k
    if (WR > 0) {
      const int k = tid >> 2, part = tid & 3;
      float acc[R];
#pragma unroll
      for (int r = 0; r < R; ++r) acc[r] = 0.f;
      if (k < HU) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const float4* dz4 = reinterpret_cast<const float4*>(dzcur + r * G4P + part * ((WR > 0 ? WR : 1) + 4));
#pragma unroll
          for (int c4 = 0; c4 < (WR > 0 ? WR : 4) / 4; ++c4) {
            const float4 v = dz4[c4];
            acc[r] = fmaf(v.x, wreg[4 * c4], acc[r]);
            acc[r] = fmaf(v.y, wreg[4 * c4 + 1], acc[r]);
            acc[r] = fmaf(v.z, wreg[4 * c4 + 2], acc[r]);
            acc[r] = fmaf(v.w, wreg[4 * c4 + 3], acc[r]);
          }
        }
      }
#pragma unroll
      for (int r = 0; r < R; ++r) {
        acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], 1);
        acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], 2);
      }
      __syncthreads();  // everyone done reading dhbuf of this step
      if (k < HU && part == 0) {
#pragma unroll
        for (int r = 0; r < R; ++r)
          if (s < s_len[r]) dhbuf[r * HU + k] = acc[r];   // inactive rows carry the recurrent gradient through unchanged
      }
    } else {
      // split the 4H columns over the threads of a (r,k) team
      const int teams = R * HU;
      const int tpt = blockDim.x / teams > 0 ? blockDim.x / teams : 1;  // threads per team
      const int team = tid / tpt, part = tid - team * tpt;
      float partial = 0.f;
      if (team < teams) {
        const int r = team / HU, k = team - r * HU;
        const float* dz = dzcur + r * G4;
        for (int col = part; col < G4; col += tpt) partial = fmaf(dz[col], Wt[col * WP + k], partial);
      }
      // reduce within the team (tpt is a power of two <= 32 by construction of the launch)
      for (int o = tpt >> 1; o > 0; o >>= 1) partial += __shfl_down_sync(0xffffffffu, partial, o, tpt);
      __syncthreads();  // everyone done reading dhbuf of this step
      if (team < teams && part == 0) {
        const int r = team / HU, k = team - r * HU;
        // inactive rows carry the recurrent gradient through unchanged (state was copied through)
        const bool active = s < s_len[r];
        if (active) dhbuf[r * HU + k] = partial;
      }
    }
    __syncthreads();
  }
}

template <int R, int ACT, int WR>
int launch_bwd(const float* d_out, const float* gates, const float* cstate, const float* wh_fw, const float* wh_bw,
               const int32_t* seq_len, float* d_xproj, int B, int L, int H, int C, float keep_prob, uint64_t seed,
               cudaStream_t st) {
  const int HU = H / C;
  const size_t smem = WR > 0 ? ((size_t)2 * R * (4 * H + 16) + (size_t)R * HU + 32) * 4
                            : ((size_t)4 * H * (HU + 1) + 2 * R * 4 * H + (size_t)R * HU + 32) * 4;
  // threads: R*HU teams x tpt threads, tpt = largest power of two with R*HU*tpt <= 512 (and <= 32)
  int tpt = 1;
  while (tpt < 32 && R * HU * tpt * 2 <= 512) tpt *= 2;
  int threads = ((R * HU * tpt + 31) / 32) * 32;
  if (WR > 0) threads = ((max(HU * 4, R * HU) + 31) / 32) * 32;      // (k, part) GEMV threads; the first R*HU also run the cells
  return rnn::launch_cluster(bilstm_bwd_kernel<R, ACT, WR>, B, R, C, threads, smem, st, d_out, gates, cstate, wh_fw, wh_bw,
                             seq_len, d_xproj, B, L, H, C, keep_prob, (uint32_t)seed, (uint32_t)(seed >> 32));
}

}  // namespace

extern "C" int ner_bilstm_recurrence_bwd(const float* d_out, const float* gates, const float* cstate,
                                         const float* wh_fw, const float* wh_bw, const int32_t* seq_len,
                                         float* d_xproj, int B, int L, int H, int activation, float keep_prob,
                                         uint64_t seed, ner_stream_t stream) {
  if (B < 0 || L < 1 || H < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!d_out || !gates || !cstate || !wh_fw || !wh_bw || !seq_len || !d_xproj) return NER_ERR_INVALID_ARG;
  if (activation != 0 && activation != 1) return NER_ERR_INVALID_ARG;
  int R, C, resident;
  const int status = ner_rnn_plan(NER_RNN_LSTM_BWD, B, H, 0, ner_num_sms(), &R, &C, &resident);
  if (status != NER_OK) return status;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define GO(RR, WRR)                                                                                                \
  return activation == 1 ? launch_bwd<RR, 1, WRR>(d_out, gates, cstate, wh_fw, wh_bw, seq_len, d_xproj, B, L, H, C, keep_prob, seed, st) \
                         : launch_bwd<RR, 0, WRR>(d_out, gates, cstate, wh_fw, wh_bw, seq_len, d_xproj, B, L, H, C, keep_prob, seed, st)
  if (resident) {   // register-resident recurrent matrix (H = 128, C = 2): 4H / 4 = 128 columns per thread
    if (R == 2) GO(2, 128);
    GO(1, 128);
  }
  if (R == 2) GO(2, 0);
  GO(1, 0);
#undef GO
}
