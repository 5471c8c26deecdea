// fp32 self-attention for small heads, with the TENER relative-position term (sm_90a, SIMT).
//
// Replaces reference tools/transformer/tener.py:12-119 (relative_attention + shift +
// normalize_attention + weighted value) for model/transformer_tener_crf_bichar.py:
//     scores[q,k] = (Q_q + u_h)·K_k + (Q_q + v_h)·R_{k-q+L}      (unscaled, K unprojected)
//     out_q = softmax_k(scores + (1-mask_k)·(-2^32+1)) · V
// R = sinusoidal table over positions -L..L-1 (tools/transformer/modules.py:177-197); the
// reference's zero-pad/reshape `shift` is the index identity BD'[q,k] = BD[q, k-q+L], so the
// [B,n,L,2L] BD tensor it materialises never exists here.  With rel == NULL the kernel is a
// plain scaled dot-product attention (used by the fp32-accurate BERT mode, head_dim 64).
//
// One CTA = one (batch row, head, tile of 32 queries); K, V and the needed R rows are staged in
// shared memory (row pitch DH+1 floats: conflict-free for lane-per-key access).  One warp per
// query at a time: lanes split the keys, scores stay in registers, softmax by warp shuffles.
// Masked keys (k >= seq_len) contribute exp(-4.29e9 - max) == 0 exactly in fp32, so skipping
// them is bit-equivalent for valid query rows; rows q >= seq_len are written as zeros (they never
// reach loss / pred_ids).  ~4 GFLOP per TENER forward: HBM/latency-bound, not tensor-core work.
#include "common.cuh"

namespace {

using namespace nerdev;

constexpr int QT = 32;      // queries per CTA
constexpr int NWARP = 4;
constexpr int MAXI = 16;    // keys per lane -> L <= 512

template <int DH, bool REL>
__global__ void __launch_bounds__(NWARP * 32)
attention_f32_kernel(const float* __restrict__ Q, int ldq, const float* __restrict__ K, int ldk,
                     const float* __restrict__ V, int ldv, const float* __restrict__ bias_u,
                     const float* __restrict__ bias_v, const float* __restrict__ rel,
                     const int32_t* __restrict__ seq_len, float scale, float* __restrict__ out_f32,
                     __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo, int L, int NH) {
  constexpr int P = DH + 1;
  extern __shared__ float sm[];
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * QT;
  const int len = min(max(seq_len[b], 0), L);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const size_t row0 = (size_t)b * L;
  const int HD = NH * DH;

  float* sK = sm;                    // [len][P]
  float* sV = sK + (size_t)L * P;    // [len][P]
  float* sR = sV + (size_t)L * P;    // [len + QT][P]   rows r = rbase .. rbase + len + QT - 1
  const int rbase = L - q0 - (QT - 1);  // smallest R row any query of this tile touches (k=0, q=q0+QT-1)

  if (q0 < len) {
    for (int idx = tid; idx < len * DH; idx += NWARP * 32) {
      const int k = idx / DH, d = idx - k * DH;
      sK[k * P + d] = K[(row0 + k) * ldk + h * DH + d];
      sV[k * P + d] = V[(row0 + k) * ldv + h * DH + d];
    }
    if (REL) {
      for (int idx = tid; idx < (len + QT) * DH; idx += NWARP * 32) {
        const int r = idx / DH, d = idx - r * DH;
        const int rr = rbase + r;
        sR[r * P + d] = (rr >= 0 && rr < 2 * L) ? rel[(size_t)rr * DH + d] : 0.f;
      }
    }
  }
  __syncthreads();

  for (int qi = warp; qi < QT; qi += NWARP) {
    const int q = q0 + qi;
    if (q >= L) break;
    float* orow = out_f32 ? out_f32 + (row0 + q) * HD + h * DH : nullptr;
    if (q >= len) {  // padded query row: zeros
      for (int d = lane; d < DH; d += 32) {
        if (orow) orow[d] = 0.f;
        if (out_hi) out_hi[(row0 + q) * HD + h * DH + d] = __float2bfloat16_rn(0.f);
        if (out_lo) out_lo[(row0 + q) * HD + h * DH + d] = __float2bfloat16_rn(0.f);
      }
      continue;
    }
    float qu[DH], qv[REL ? DH : 1];
#pragma unroll
    for (int d = 0; d < DH; ++d) {
      const float qd = Q[(row0 + q) * ldq + h * DH + d];
      qu[d] = qd + (bias_u ? bias_u[h * DH + d] : 0.f);
      if (REL) qv[d] = qd + bias_v[h * DH + d];
    }
    float s[MAXI];
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < MAXI; ++i) {
      const int k = lane + 32 * i;
      s[i] = -INFINITY;
      if (k < len) {
        const float* kr = sK + k * P;
        float acc = 0.f;
#pragma unroll
        for (int d = 0; d < DH; ++d) acc = fmaf(qu[d], kr[d], acc);
        if (REL) {
          const float* rr = sR + (k - q + L - rbase) * P;
          float acc2 = 0.f;
#pragma unroll
          for (int d = 0; d < DH; ++d) acc2 = fmaf(qv[d], rr[d], acc2);
          acc += acc2;
        }
        s[i] = acc * scale;
        mx = fmaxf(mx, s[i]);
      }
    }
    mx = warp_max(mx);
    float sum = 0.f;
    float o[DH];
#pragma unroll
    for (int d = 0; d < DH; ++d) o[d] = 0.f;
#pragma unroll
    for (int i = 0; i < MAXI; ++i) {
      const int k = lane + 32 * i;
      if (k < len) {
        const float p = expf(s[i] - mx);
        sum += p;
        const float* vr = sV + k * P;
#pragma unroll
        for (int d = 0; d < DH; ++d) o[d] = fmaf(p, vr[d], o[d]);
      }
    }
    sum = warp_sum(sum);
    const float inv = 1.f / sum;
#pragma unroll
    for (int d = 0; d < DH; ++d) o[d] = warp_sum(o[d]);
    // lane (d % 32) writes column d
#pragma unroll
    for (int base = 0; base < DH; base += 32) {
      float val = 0.f;
#pragma unroll
      for (int d = 0; d < DH; ++d)
        if (d >= base && d < base + 32 && (d - base) == lane) val = o[d];
      const int d = base + lane;
      if (d < DH) {
        const float r = val * inv;
        if (orow) orow[d] = r;
        if (out_hi) {
          const __nv_bfloat16 hi = __float2bfloat16_rn(r);
          out_hi[(row0 + q) * HD + h * DH + d] = hi;
          if (out_lo) out_lo[(row0 + q) * HD + h * DH + d] = __float2bfloat16_rn(r - __bfloat162float(hi));
        }
      }
    }
  }
}

template <int DH, bool REL>
int launch_attn(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv, const float* u,
                const float* v, const float* rel, const int32_t* seq_len, float scale, float* out_f32, void* out_hi,
                void* out_lo, int B, int L, int NH, cudaStream_t st) {
  const size_t smem = ((size_t)2 * L + (REL ? (L + QT) : 0)) * (DH + 1) * 4;
  if (smem > 227 * 1024) return NER_ERR_UNSUPPORTED;
  auto kern = attention_f32_kernel<DH, REL>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  dim3 grid((L + QT - 1) / QT, NH, B);
  kern<<<grid, NWARP * 32, smem, st>>>(Q, ldq, K, ldk, V, ldv, u, v, rel, seq_len, scale, out_f32,
                                        static_cast<__nv_bfloat16*>(out_hi), static_cast<__nv_bfloat16*>(out_lo), L, NH);
  return ner_launch_status();
}

}  // namespace

extern "C" int ner_attention_f32(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv,
                                 const float* bias_u, const float* bias_v, const float* rel_table,
                                 const int32_t* seq_len, float scale, float* out_f32, void* out_hi_bf16,
                                 void* out_lo_bf16, int B, int L, int num_heads, int head_dim, ner_stream_t stream) {
  if (B < 0 || L < 1 || num_heads < 1 || head_dim < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!Q || !K || !V || !seq_len || (!out_f32 && !out_hi_bf16)) return NER_ERR_INVALID_ARG;
  if (out_lo_bf16 && !out_hi_bf16) return NER_ERR_INVALID_ARG;
  if (rel_table && !bias_v) return NER_ERR_INVALID_ARG;
  if (L > 32 * MAXI) return NER_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define GO(DHV)                                                                                                   \
  return rel_table ? launch_attn<DHV, true>(Q, ldq, K, ldk, V, ldv, bias_u, bias_v, rel_table, seq_len, scale,    \
                                            out_f32, out_hi_bf16, out_lo_bf16, B, L, num_heads, st)               \
                   : launch_attn<DHV, false>(Q, ldq, K, ldk, V, ldv, bias_u, bias_v, rel_table, seq_len, scale,   \
                                             out_f32, out_hi_bf16, out_lo_bf16, B, L, num_heads, st)
  switch (head_dim) {
    case 20: GO(20);
    case 32: GO(32);
    case 40: GO(40);
    case 64: GO(64);
    default: return NER_ERR_UNSUPPORTED;
  }
#undef GO
}

// ---------------------------------------------------------------------------------------------
// Backward of the kernel above (TRAIN mode of the TENER plugin: tf.gradients through
// relative_multi_head_attention, reference tools/transformer/tener.py:12-119).  With
//   s_qk = scale * [(Q_q + u)·K_k + (Q_q + v)·R_{k-q+L}],  p = softmax_k(s),  O_q = sum_k p_qk V_k :
//   dV_k += p_qk dO_q                      dP_qk = dO_q · V_k          D_q = sum_k p_qk dP_qk
//   dS_qk = scale * p_qk (dP_qk - D_q)
//   dQ_q  = sum_k dS_qk (K_k + R_{k-q+L})  dK_k += dS_qk (Q_q + u)
//   du   += sum_qk dS_qk K_k               dv   += sum_qk dS_qk R_{k-q+L}
// Same decomposition as the forward: one CTA = (batch row, head, 32 queries), one warp per query, lanes split
// the keys; scores are recomputed (nothing L x L is stored).  dK / dV of the CTA's queries are accumulated
// in shared memory and leave with one global atomic per (key, d); du / dv with one per (CTA, d).
template <int DH, bool REL>
__global__ void __launch_bounds__(NWARP * 32)
attention_f32_bwd_kernel(const float* __restrict__ Q, int ldq, const float* __restrict__ K, int ldk,
                         const float* __restrict__ V, int ldv, const float* __restrict__ bias_u,
                         const float* __restrict__ bias_v, const float* __restrict__ rel,
                         const int32_t* __restrict__ seq_len, float scale, const float* __restrict__ dO, int lddo,
                         float* __restrict__ dQ, int lddq, float* __restrict__ dK, int lddk, float* __restrict__ dV,
                         int lddv, float* __restrict__ d_u, float* __restrict__ d_v, int L, int NH) {
  constexpr int P = DH + 1;
  extern __shared__ float sm[];
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * QT;
  const int len = min(max(seq_len[b], 0), L);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const size_t row0 = (size_t)b * L;

  float* sK = sm;                         // [L][P]
  float* sV = sK + (size_t)L * P;         // [L][P]
  float* sdK = sV + (size_t)L * P;        // [L][P]
  float* sdV = sdK + (size_t)L * P;       // [L][P]
  float* sR = sdV + (size_t)L * P;        // [L + QT][P]
  float* sdu = sR + (size_t)(REL ? (L + QT) : 0) * P;   // [2][DH]: du, dv partials of this CTA
  const int rbase = L - q0 - (QT - 1);

  // padded query rows of this tile: zero gradient
  for (int idx = tid; idx < QT * DH; idx += NWARP * 32) {
    const int q = q0 + idx / DH, d = idx % DH;
    if (q < L && q >= len) dQ[(row0 + q) * lddq + h * DH + d] = 0.f;
  }
  if (q0 >= len) return;
  for (int idx = tid; idx < len * DH; idx += NWARP * 32) {
    const int k = idx / DH, d = idx - k * DH;
    sK[k * P + d] = K[(row0 + k) * ldk + h * DH + d];
    sV[k * P + d] = V[(row0 + k) * ldv + h * DH + d];
    sdK[k * P + d] = 0.f;
    sdV[k * P + d] = 0.f;
  }
  if (REL) {
    for (int idx = tid; idx < (len + QT) * DH; idx += NWARP * 32) {
      const int r = idx / DH, d = idx - r * DH;
      const int rr = rbase + r;
      sR[r * P + d] = (rr >= 0 && rr < 2 * L) ? rel[(size_t)rr * DH + d] : 0.f;
    }
  }
  for (int idx = tid; idx < 2 * DH; idx += NWARP * 32) sdu[idx] = 0.f;
  __syncthreads();

  float du_acc[DH], dv_acc[REL ? DH : 1];   // per-lane partials over this warp's queries
#pragma unroll
  for (int d = 0; d < DH; ++d) du_acc[d] = 0.f;
  if (REL) {
#pragma unroll
    for (int d = 0; d < DH; ++d) dv_acc[d] = 0.f;
  }

  for (int qi = warp; qi < QT; qi += NWARP) {
    const int q = q0 + qi;
    if (q >= len) break;
    float qu[DH], qv[REL ? DH : 1], go[DH];
#pragma unroll
    for (int d = 0; d < DH; ++d) {
      const float qd = Q[(row0 + q) * ldq + h * DH + d];
      qu[d] = qd + (bias_u ? bias_u[h * DH + d] : 0.f);
      if (REL) qv[d] = qd + bias_v[h * DH + d];
      go[d] = dO[(row0 + q) * lddo + h * DH + d];
    }
    float s[MAXI], dp[MAXI];
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < MAXI; ++i) {
      const int k = lane + 32 * i;
      s[i] = -INFINITY;
      dp[i] = 0.f;
      if (k < len) {
        const float* kr = sK + k * P;
        const float* vr = sV + k * P;
        float acc = 0.f, g = 0.f;
#pragma unroll
        for (int d = 0; d < DH; ++d) {
          acc = fmaf(qu[d], kr[d], acc);
          g = fmaf(go[d], vr[d], g);
        }
        if (REL) {
          const float* rr = sR + (k - q + L - rbase) * P;
          float acc2 = 0.f;
#pragma unroll
          for (int d = 0; d < DH; ++d) acc2 = fmaf(qv[d], rr[d], acc2);
          acc += acc2;
        }
        s[i] = acc * scale;
        dp[i] = g;
        mx = fmaxf(mx, s[i]);
      }
    }
    mx = warp_max(mx);
    float sum = 0.f, dsum = 0.f;
#pragma unroll
    for (int i = 0; i < MAXI; ++i) {
      const int k = lane + 32 * i;
      if (k < len) {
        s[i] = expf(s[i] - mx);   // unnormalised p
        sum += s[i];
        dsum = fmaf(s[i], dp[i], dsum);
      }
    }
    sum = warp_sum(sum);
    dsum = warp_sum(dsum);
    const float inv = 1.f / sum;
    const float D = dsum * inv;
    float dq[DH];
#pragma unroll
    for (int d = 0; d < DH; ++d) dq[d] = 0.f;
#pragma unroll
    for (int i = 0; i < MAXI; ++i) {
      const int k = lane + 32 * i;
      if (k < len) {
        const float p = s[i] * inv;
        const float ds = scale * p * (dp[i] - D);
        const float* kr = sK + k * P;
        float* dkr = sdK + k * P;
        float* dvr = sdV + k * P;
        const float* rr = REL ? sR + (k - q + L - rbase) * P : nullptr;
#pragma unroll
        for (int d = 0; d < DH; ++d) {
          float t = kr[d];
          du_acc[d] = fmaf(ds, kr[d], du_acc[d]);
          if (REL) {
            t += rr[d];
            dv_acc[d] = fmaf(ds, rr[d], dv_acc[d]);
          }
          dq[d] = fmaf(ds, t, dq[d]);
          atomicAdd(dkr + d, ds * qu[d]);     // the four warps of the CTA share the keys
          atomicAdd(dvr + d, p * go[d]);
        }
      }
    }
#pragma unroll
    for (int d = 0; d < DH; ++d) dq[d] = warp_sum(dq[d]);
    if (lane == 0) {
#pragma unroll
      for (int d = 0; d < DH; ++d) dQ[(row0 + q) * lddq + h * DH + d] = dq[d];
    }
  }
#pragma unroll
  for (int d = 0; d < DH; ++d) {
    const float a = warp_sum(du_acc[d]);
    if (lane == 0) atomicAdd(sdu + d, a);
    if (REL) {
      const float c = warp_sum(dv_acc[d]);
      if (lane == 0) atomicAdd(sdu + DH + d, c);
    }
  }
  __syncthreads();
  for (int idx = tid; idx < len * DH; idx += NWARP * 32) {
    const int k = idx / DH, d = idx - k * DH;
    atomicAdd(dK + (row0 + k) * lddk + h * DH + d, sdK[k * P + d]);
    atomicAdd(dV + (row0 + k) * lddv + h * DH + d, sdV[k * P + d]);
  }
  for (int d = tid; d < DH; d += NWARP * 32) {
    if (d_u) atomicAdd(d_u + h * DH + d, sdu[d]);
    if (REL && d_v) atomicAdd(d_v + h * DH + d, sdu[DH + d]);
  }
}

namespace {
template <int DH, bool REL>
int launch_attn_bwd(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv, const float* u, const float* v,
                    const float* rel, const int32_t* seq_len, float scale, const float* dO, int lddo, float* dQ, int lddq,
                    float* dK, int lddk, float* dV, int lddv, float* d_u, float* d_v, int B, int L, int NH, cudaStream_t st) {
  const size_t smem = (((size_t)4 * L + (REL ? (L + QT) : 0)) * (DH + 1) + 2 * DH) * 4;
  if (smem > 227 * 1024) return NER_ERR_UNSUPPORTED;
  auto kern = attention_f32_bwd_kernel<DH, REL>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  dim3 grid((L + QT - 1) / QT, NH, B);
  kern<<<grid, NWARP * 32, smem, st>>>(Q, ldq, K, ldk, V, ldv, u, v, rel, seq_len, scale, dO, lddo, dQ, lddq, dK, lddk, dV, lddv,
                                        d_u, d_v, L, NH);
  return ner_launch_status();
}
}  // namespace

extern "C" int ner_attention_f32_bwd(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv,
                                     const float* bias_u, const float* bias_v, const float* rel_table,
                                     const int32_t* seq_len, float scale, const float* d_out, int ld_dout, float* dQ,
                                     int ld_dq, float* dK, int ld_dk, float* dV, int ld_dv, float* d_bias_u,
                                     float* d_bias_v, int B, int L, int num_heads, int head_dim, ner_stream_t stream) {
  if (B < 0 || L < 1 || num_heads < 1 || head_dim < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!Q || !K || !V || !seq_len || !d_out || !dQ || !dK || !dV) return NER_ERR_INVALID_ARG;
  if (rel_table && !bias_v) return NER_ERR_INVALID_ARG;
  if (L > 32 * MAXI) return NER_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define GOB(DHV)                                                                                                       \
  return rel_table ? launch_attn_bwd<DHV, true>(Q, ldq, K, ldk, V, ldv, bias_u, bias_v, rel_table, seq_len, scale, d_out,  \
                                                ld_dout, dQ, ld_dq, dK, ld_dk, dV, ld_dv, d_bias_u, d_bias_v, B, L,        \
                                                num_heads, st)                                                             \
                   : launch_attn_bwd<DHV, false>(Q, ldq, K, ldk, V, ldv, bias_u, bias_v, rel_table, seq_len, scale, d_out, \
                                                 ld_dout, dQ, ld_dq, dK, ld_dk, dV, ld_dv, d_bias_u, d_bias_v, B, L,       \
                                                 num_heads, st)
  switch (head_dim) {
    case 20: GOB(20);
    case 32: GOB(32);
    case 40: GOB(40);
    case 64: GOB(64);
    default: return NER_ERR_UNSUPPORTED;
  }
#undef GOB
}
