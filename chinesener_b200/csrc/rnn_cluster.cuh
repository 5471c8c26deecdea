// What the persistent thread-block-cluster recurrences share (bilstm.cu, bilstm_bwd.cu, bigru.cu, bigru_bwd.cu,
// lattice.cu).  Every one splits the batch the same way: a cluster of C CTAs owns R batch rows of one direction for all
// time steps, and CTA `rank` of the cluster owns the hidden units [rank * H/C, (rank + 1) * H/C).  The grid is
// 2 directions x ceil(B / R) row groups x C CTAs.  Each kernel keeps its own shared-memory layout and step math.
#pragma once
#include <cooperative_groups.h>
#include <stddef.h>
#include <stdint.h>

#include "common.cuh"

namespace rnn {

// ---- Distributed-shared-memory signalling.  A value is published to a peer CTA of the cluster with a remote 4-byte
// store that completes transaction bytes on the DESTINATION CTA's mbarrier (st.async), so a publish needs no fence over
// the thread's earlier global stores and the wait no L1 invalidate (barrier.cluster costs both every step).

__device__ __forceinline__ uint32_t mapa_u32(uint32_t local_smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_async_f32(uint32_t remote_addr, float v, uint32_t remote_bar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(remote_addr),
               "r"(__float_as_uint(v)), "r"(remote_bar)
               : "memory");
}
__device__ __forceinline__ void mbar_init_(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(nerdev::smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx_(uint64_t* bar, uint32_t tx_bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(nerdev::smem_u32(bar)), "r"(tx_bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait_(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(nerdev::smem_u32(bar)), "r"(parity)
        : "memory");
  }
}
// Publish v at the same shared-memory location (local address `la`, mbarrier `lb`) in every CTA of a C-CTA cluster.
__device__ __forceinline__ void publish_all(uint32_t la, uint32_t lb, float v, int C) {
  for (int dst = 0; dst < C; ++dst) st_async_f32(mapa_u32(la, (uint32_t)dst), v, mapa_u32(lb, (uint32_t)dst));
}

// ---- Row-group geometry

struct RowGroup {
  int rank;   // this CTA's rank in its cluster
  int dir;    // 0 forward, 1 backward
  int b0;     // first batch row of the cluster
};
__device__ __forceinline__ RowGroup row_group(int C, int B, int R) {
  const int ngroups = (B + R - 1) / R;
  const int cid = blockIdx.x / C;
  return RowGroup{(int)cooperative_groups::this_cluster().block_rank(), cid / ngroups, (cid % ngroups) * R};
}

// Fills s_len[0, R) with the row group's lengths clamped to [0, L] (0 for rows past the batch), waits for the CTA and
// returns the longest.
template <int R>
__device__ __forceinline__ int load_lengths(int* s_len, const int32_t* __restrict__ seq_len, int b0, int B, int L) {
  const int tid = threadIdx.x;
  if (tid < R) s_len[tid] = (b0 + tid < B) ? min(max(seq_len[b0 + tid], 0), L) : 0;
  __syncthreads();
  int maxlen = 0;
#pragma unroll
  for (int r = 0; r < R; ++r) maxlen = max(maxlen, s_len[r]);
  return maxlen;
}

// ---- Cell math

// ex2.approx-based forms (abs. error ~1e-7, far inside the 1e-4 parity bar of tests/test_bilstm_gpu.py): the activations
// sit on the per-step critical path of the forward recurrences.
__device__ __forceinline__ float sigmoid_fast(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }

template <int ACT>   // 0 tanh, 1 relu
__device__ __forceinline__ float act_fast(float x) {
  if (ACT == 1) return fmaxf(x, 0.f);
  return 1.f - __fdividef(2.f, 1.f + __expf(2.f * x));   // tanh(x); saturates correctly for |x| large
}

template <int ACT>
__device__ __forceinline__ float act_grad_from_output(float a) {   // d act(x)/dx expressed through a = act(x)
  if (ACT == 1) return a > 0.f ? 1.f : 0.f;
  return 1.f - a * a;
}

// DropoutWrapper(output_keep_prob, state_keep_prob): independent keep masks for the emitted output and for the h part of
// the carried state, fresh per step, drawn for element (b, pos, dir * H + u) of the [B, L, 2H] output.  Scales `out` and
// `state` in place: kept values by inv_keep, dropped ones to 0.  The forward kernels apply it to h and the backward
// kernels to the gradients of the same elements, so all four must draw the same masks; _rnn_masks in
// tests/test_rnn_cells_gpu.py restates the draw and is the test side of this format.
__device__ __forceinline__ void dropout_out_state(float& out, float& state, uint32_t seed_lo, uint32_t seed_hi,
                                                  uint32_t thr, float inv_keep, int b, int L, int pos, int H, int dir,
                                                  int u) {
  const uint32_t e = (uint32_t)(((size_t)b * L + pos) * 2 * H + (size_t)dir * H + u);
  out = nerdev::hash3(seed_lo, seed_hi, e) < thr ? out * inv_keep : 0.f;
  state = nerdev::hash3(seed_lo ^ 0x5bd1e995u, seed_hi, e) < thr ? state * inv_keep : 0.f;
}

// ---- Packed-FFMA2 dot products.  A lane holds one float4 of a weight column and accumulates R rows in two packed
// chains, (w.x, w.y) . (v.x, v.y) into a and (w.z, w.w) . (v.z, v.w) into b, where v is float4 k4 of row r of `v4`
// (row stride ld float4s).  Pairs halve the FMA issue slots of the dot products, the per-step throughput bound of the
// recurrences; two chains per row hide the FMA latency.  The caller chooses k4, so each kernel keeps its own mapping
// of lanes to float4s.
template <int R>
__device__ __forceinline__ void fma2_rows(nerdev::f32x2 (&a)[R], nerdev::f32x2 (&b)[R], float4 w, const float4* v4,
                                          int ld, int k4) {
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const float4 v = v4[r * ld + k4];
    a[r] = nerdev::fma2(nerdev::pk2(w.x, w.y), nerdev::pk2(v.x, v.y), a[r]);
    b[r] = nerdev::fma2(nerdev::pk2(w.z, w.w), nerdev::pk2(v.z, v.w), b[r]);
  }
}
// The lane's partial dot product of one row: (z0 + z1) + (z2 + z3) over the two chains.
__device__ __forceinline__ float sum_chains(nerdev::f32x2 a, nerdev::f32x2 b) {
  float z0, z1, z2, z3;
  nerdev::upk2(a, z0, z1);
  nerdev::upk2(b, z2, z3);
  return (z0 + z1) + (z2 + z3);
}

// ---- Tail writes

// out [B, L, 2H]: zeros at the positions [maxlen, L) past the longest row of the cluster, for this CTA's HU units.
__device__ __forceinline__ void zero_past_maxlen(float* out, int R, int b0, int B, int L, int H, int dir, int rank,
                                                 int HU, int maxlen) {
  for (int idx = threadIdx.x; idx < R * HU; idx += blockDim.x) {
    const int r = idx / HU, uu = idx - r * HU;
    const int b = b0 + r;
    if (b < B)
      for (int s = maxlen; s < L; ++s) out[((size_t)b * L + s) * 2 * H + (size_t)dir * H + rank * HU + uu] = 0.f;
  }
}

// d_xproj [B, L, 2 G H] (G gates per direction): zeros at the positions [s_len[r], L) that no step of row r visits, for
// this CTA's HU units of every gate.
template <int G>
__device__ __forceinline__ void zero_unvisited(float* d_xproj, const int* s_len, int R, int b0, int B, int L, int H,
                                               int dir, int rank, int HU) {
  for (int idx = threadIdx.x; idx < R * G * HU; idx += blockDim.x) {
    const int r = idx / (G * HU), c = idx - r * G * HU;
    const int g = c / HU, u = c - g * HU;
    const int b = b0 + r;
    if (b < B)
      for (int t = s_len[r]; t < L; ++t)
        d_xproj[((size_t)b * L + t) * 2 * G * H + (size_t)dir * G * H + g * H + rank * HU + u] = 0.f;
  }
}

// ---- Host side

// Launch kern over the 2 * ceil(B / R) * C CTAs of a recurrence, in clusters of C, with `threads` threads and `smem`
// bytes of dynamic shared memory per CTA.
template <typename K, typename... Args>
int launch_cluster(K kern, int B, int R, int C, int threads, size_t smem, cudaStream_t st, Args... args) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)(2 * ((B + R - 1) / R) * C));
  cfg.blockDim = dim3((unsigned)threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)C;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  e = cudaLaunchKernelEx(&cfg, kern, args...);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  return ner_launch_status();
}

// Rows per cluster of the BiLSTM and BiGRU recurrences: fill the num_sms SMs once when the batch is small, amortise the
// weight reads when it is large.
static inline int rows_per_cluster(int B, int C, int num_sms) {
  int R = 1;
  if ((long)2 * B * C > num_sms) R = 2;
  if ((long)2 * ((B + 1) / 2) * C > 2 * (long)num_sms) R = 4;
  return R;
}

// Smallest power-of-two cluster of the BiLSTM recurrence (bilstm.cu) whose W_h slice (H * 4H/C floats) fits ~190 KB
// and divides H; 0 if none.
static inline int lstm_pick_cluster(int H) {
  for (int C = 1; C <= 8; C *= 2) {
    if (H % C != 0) continue;
    const size_t bytes = (size_t)H * 4 * (H / C) * 4;
    if (bytes <= 190 * 1024 && 4 * (H / C) <= 512) return C;
  }
  return 0;
}

// The same for its back-propagation through time (bilstm_bwd.cu): a [4H][H/C + 1] transposed slice within 180 KB.
static inline int lstm_pick_cluster_bwd(int H) {
  for (int C = 1; C <= 8; C *= 2) {
    if (H % C != 0) continue;
    const size_t bytes = (size_t)4 * H * (H / C + 1) * 4;
    if (bytes <= 180 * 1024) return C;
  }
  return 0;
}

// The GRU recurrence (bigru.cu) and its back-propagation through time (bigru_bwd.cu) keep the same recurrent weights
// resident (three columns per owned unit, four lanes per unit) and exchange at most 3 R H floats per step through
// double-buffered DSMEM, so one cluster size and one shared-memory size serve both.
// float4 weight streams of four lanes per unit: ceil(H/8) for the 2H-wide gate columns, ceil(H/16) for the candidate.
static inline size_t gru_smem_bytes(int H, int C, int R) {
  const int NT = 4 * (H / C), H4 = H / 4;
  return (size_t)((H4 + 1) / 2 + (H4 + 3) / 4) * NT * 16 + (size_t)6 * R * H * 4 + 64;   // + s_len[8] + 4 mbarriers
}

// Smallest power-of-two cluster (<= 8, portable) whose GRU slice fits 200 KB at R = 4 with at most 512 threads; 0 if none.
static inline int gru_pick_cluster(int H) {
  for (int C = 1; C <= 8; C *= 2) {
    if (H % C != 0) continue;
    if (4 * (H / C) <= 512 && gru_smem_bytes(H, C, 4) <= 200 * 1024) return C;
  }
  return 0;
}

// Rows per cluster and cluster size of the Lattice LSTM kernels (lattice.cu, where their shared-memory layout lives):
// NER_OK, or the status ner_lattice_recurrence returns for the shape.
int lattice_config(int B, int H, int Kw, int num_sms, int* R, int* C);

}  // namespace rnn
