// Backward-pass HBM-bound kernels of the encoder (sm_90a): LayerNorm backward (with the residual
// recomputed from the saved operands), bf16 transposes for the weight-gradient GEMMs, bias
// gradients of bf16 tensors, GELU backward, and the embedding scatter-add.  Together with the
// wgmma GEMM (gemm_tc.cu) and attention_bwd.cu they are the gradient that tf.gradients produces
// for bert_base.bert.modeling.BertModel in the reference (tools/train_utils.py:314).
#include "common.cuh"

namespace {

using namespace nerdev;

constexpr int LN_MAXV = 8;

__device__ __forceinline__ float4 ld_bf16x4(const __nv_bfloat16* p) {
  const uint2 pk = *reinterpret_cast<const uint2*>(p);
  const __nv_bfloat162 lo = *reinterpret_cast<const __nv_bfloat162*>(&pk.x);
  const __nv_bfloat162 hi = *reinterpret_cast<const __nv_bfloat162*>(&pk.y);
  return make_float4(__low2float(lo), __high2float(lo), __low2float(hi), __high2float(hi));
}
__device__ __forceinline__ void st_bf16x4(__nv_bfloat16* p, float4 v) {
  __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
  uint2 pk;
  pk.x = *reinterpret_cast<uint32_t*>(&lo);
  pk.y = *reinterpret_cast<uint32_t*>(&hi);
  *reinterpret_cast<uint2*>(p) = pk;
}

// z = y(bf16|f32) + residual(f32) is recomputed; out = LN(z)*gamma + beta.
//   dz = rstd * (g*gamma - mean(g*gamma) - zhat * mean(g*gamma*zhat)),  dgamma += g*zhat,  dbeta += g
// dz is written as f32 (the residual-branch gradient) and as bf16 (A operand of the dgrad GEMM).
// DROP: the forward was ner_layernorm_dropout — z is rebuilt as dropout(y) + residual from the UNdropped y and
// the bf16 gradient (the dense-output branch) is masked the same way; dz_f32 (the residual branch) is not.
// NV = float4 per lane (ceil(H / 128)).  The column partials (dgamma, dbeta, dbias) of a warp live in the warp's OWN slab of
// shared memory — each lane read-modify-writes only its own columns, no atomics — instead of 3 * NV float4 registers: the
// register version needed 254 registers, i.e. one 8-warp CTA per SM, and ncu showed it latency-bound (81 % of the cycles
// without an eligible warp at 12 % DRAM throughput).  ~120 registers -> two CTAs per SM.
template <bool YBF16, bool DROP, int NV>
__global__ void __launch_bounds__(256, 2)
layernorm_bwd_kernel(const void* __restrict__ yv, const float* __restrict__ residual, const float* __restrict__ gamma,
                     const float* __restrict__ dout, float* __restrict__ dz_f32, __nv_bfloat16* __restrict__ dz_bf16,
                     float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ dbias, int M, int H, float eps,
                     float keep, uint32_t seed_lo, uint32_t seed_hi) {
  const uint32_t thr = keep_threshold(keep);
  const float inv_keep = 1.f / keep;
  extern __shared__ __align__(16) float s_acc[];  // [8 warps][3][H]: dgamma / dbeta / dbias partials of each warp
  for (int e = threadIdx.x; e < 8 * 3 * H; e += blockDim.x) s_acc[e] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* my = s_acc + (size_t)warp * 3 * H;
  const int nv4 = (H / 4 + 31) / 32;
  for (int row = blockIdx.x * (blockDim.x >> 5) + warp; row < M; row += gridDim.x * (blockDim.x >> 5)) {
    float4 z[NV], g[NV];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int e = (lane + 32 * k) * 4;
      if (k < nv4 && e < H) {
        if constexpr (YBF16) z[k] = ld_bf16x4(static_cast<const __nv_bfloat16*>(yv) + (size_t)row * H + e);
        else z[k] = *reinterpret_cast<const float4*>(static_cast<const float*>(yv) + (size_t)row * H + e);
        if constexpr (DROP) {
          const size_t i = (size_t)row * H + e;
          const uint32_t hi = seed_hi ^ (uint32_t)(i >> 32), lo = (uint32_t)i;
          z[k].x *= hash3(seed_lo, hi, lo) < thr ? inv_keep : 0.f;
          z[k].y *= hash3(seed_lo, hi, lo + 1) < thr ? inv_keep : 0.f;
          z[k].z *= hash3(seed_lo, hi, lo + 2) < thr ? inv_keep : 0.f;
          z[k].w *= hash3(seed_lo, hi, lo + 3) < thr ? inv_keep : 0.f;
        }
        if (residual != nullptr) {
          const float4 r = *reinterpret_cast<const float4*>(residual + (size_t)row * H + e);
          z[k].x += r.x; z[k].y += r.y; z[k].z += r.z; z[k].w += r.w;
        }
        g[k] = *reinterpret_cast<const float4*>(dout + (size_t)row * H + e);
        s += z[k].x + z[k].y + z[k].z + z[k].w;
      }
    }
    s = warp_sum(s);
    const float mean = s / (float)H;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int e = (lane + 32 * k) * 4;
      if (k < nv4 && e < H) {
        z[k].x -= mean; z[k].y -= mean; z[k].z -= mean; z[k].w -= mean;
        q += z[k].x * z[k].x + z[k].y * z[k].y + z[k].z * z[k].z + z[k].w * z[k].w;
      }
    }
    q = warp_sum(q);
    const float rstd = rsqrtf(q / (float)H + eps);
    float m1 = 0.f, m2 = 0.f;  // sum(g*gamma), sum(g*gamma*zhat)
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int e = (lane + 32 * k) * 4;
      if (k < nv4 && e < H) {
        const float4 gm = __ldg(reinterpret_cast<const float4*>(gamma + e));
        z[k].x *= rstd; z[k].y *= rstd; z[k].z *= rstd; z[k].w *= rstd;          // zhat
        float4 ag = *reinterpret_cast<float4*>(my + e), ab = *reinterpret_cast<float4*>(my + H + e);
        ag.x = fmaf(g[k].x, z[k].x, ag.x); ag.y = fmaf(g[k].y, z[k].y, ag.y);
        ag.z = fmaf(g[k].z, z[k].z, ag.z); ag.w = fmaf(g[k].w, z[k].w, ag.w);
        ab.x += g[k].x; ab.y += g[k].y; ab.z += g[k].z; ab.w += g[k].w;
        *reinterpret_cast<float4*>(my + e) = ag;
        *reinterpret_cast<float4*>(my + H + e) = ab;
        g[k].x *= gm.x; g[k].y *= gm.y; g[k].z *= gm.z; g[k].w *= gm.w;
        m1 += g[k].x + g[k].y + g[k].z + g[k].w;
        m2 += g[k].x * z[k].x + g[k].y * z[k].y + g[k].z * z[k].z + g[k].w * z[k].w;
      }
    }
    m1 = warp_sum(m1) / (float)H;
    m2 = warp_sum(m2) / (float)H;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int e = (lane + 32 * k) * 4;
      if (k < nv4 && e < H) {
        float4 d;
        d.x = rstd * (g[k].x - m1 - z[k].x * m2);
        d.y = rstd * (g[k].y - m1 - z[k].y * m2);
        d.z = rstd * (g[k].z - m1 - z[k].z * m2);
        d.w = rstd * (g[k].w - m1 - z[k].w * m2);
        if (dz_f32 != nullptr) *reinterpret_cast<float4*>(dz_f32 + (size_t)row * H + e) = d;
        if constexpr (DROP) {   // the mask is regenerated (it is not kept in registers across the row)
          const size_t i = (size_t)row * H + e;
          const uint32_t hi = seed_hi ^ (uint32_t)(i >> 32), lo = (uint32_t)i;
          d.x *= hash3(seed_lo, hi, lo) < thr ? inv_keep : 0.f;
          d.y *= hash3(seed_lo, hi, lo + 1) < thr ? inv_keep : 0.f;
          d.z *= hash3(seed_lo, hi, lo + 2) < thr ? inv_keep : 0.f;
          d.w *= hash3(seed_lo, hi, lo + 3) < thr ? inv_keep : 0.f;
        }
        if (dz_bf16 != nullptr) st_bf16x4(dz_bf16 + (size_t)row * H + e, d);
        if (dbias != nullptr) {
          float4 ad = *reinterpret_cast<float4*>(my + 2 * H + e);
          ad.x += d.x; ad.y += d.y; ad.z += d.z; ad.w += d.w;
          *reinterpret_cast<float4*>(my + 2 * H + e) = ad;
        }
      }
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < H; e += blockDim.x) {
    float a = 0.f, b = 0.f, c = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      a += s_acc[(size_t)w * 3 * H + e];
      b += s_acc[(size_t)w * 3 * H + H + e];
      c += s_acc[(size_t)w * 3 * H + 2 * H + e];
    }
    atomicAdd(dgamma + e, a);
    atomicAdd(dbeta + e, b);
    if (dbias != nullptr) atomicAdd(dbias + e, c);
  }
}

// bf16 [M,N] -> bf16 [N,Mp] (zero padded), 64x64 tiles through smem — 2-byte accesses, any N (fallback)
__global__ void __launch_bounds__(256)
transpose_bf16_scalar_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst, int M, int N, int Mp) {
  __shared__ __nv_bfloat16 tile[64][66];
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;  // 64 x 4
  for (int i = ty; i < 64; i += 4) {
    const int m = m0 + i, n = n0 + tx;
    tile[i][tx] = (m < M && n < N) ? src[(size_t)m * N + n] : __float2bfloat16_rn(0.f);
  }
  __syncthreads();
  for (int i = ty; i < 64; i += 4) {
    const int n = n0 + i, m = m0 + tx;
    if (n < N && m < Mp) dst[(size_t)n * Mp + m] = tile[tx][i];
  }
}

// Same for even N: 2x2 sub-blocks.  A thread loads the words (m, n..n+1) and (m+1, n..n+1), re-pairs them with two
// PRMTs into (n; m..m+1) and (n+1; m..m+1) and parks those in a [64 n][32 m-pair] word tile (pitch 33: the 16-byte
// output reads are conflict-free, the parking stores 2-way); output rows leave as 16-byte stores.  Half the
// memory instructions of the scalar kernel and 4x wider ones on the store side.
__global__ void __launch_bounds__(256)
transpose_bf16_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst, int M, int N, int Mp) {
  __shared__ uint32_t t[64][33];
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = n0 + 2 * lane;
#pragma unroll
  for (int rp = warp; rp < 32; rp += 8) {
    const int m = m0 + 2 * rp;
    uint32_t a = 0u, b = 0u;
    if (n < N) {
      if (m < M) a = *reinterpret_cast<const uint32_t*>(src + (size_t)m * N + n);
      if (m + 1 < M) b = *reinterpret_cast<const uint32_t*>(src + (size_t)(m + 1) * N + n);
    }
    t[2 * lane][rp] = __byte_perm(a, b, 0x5410);      // column n   : (row m, row m+1)
    t[2 * lane + 1][rp] = __byte_perm(a, b, 0x7632);  // column n+1 : (row m, row m+1)
  }
  __syncthreads();
#pragma unroll
  for (int c = threadIdx.x; c < 512; c += 256) {
    const int nr = c >> 3, ch = c & 7;
    if (n0 + nr < N && m0 + 8 * ch < Mp) {
      const uint4 v = make_uint4(t[nr][4 * ch], t[nr][4 * ch + 1], t[nr][4 * ch + 2], t[nr][4 * ch + 3]);
      *reinterpret_cast<uint4*>(dst + (size_t)(n0 + nr) * Mp + m0 + 8 * ch) = v;
    }
  }
}

// out[n] += sum_m x[m,n] for bf16 x (bias gradients of bf16 dense-output gradients)
__global__ void __launch_bounds__(256)
colsum_bf16_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ out, int M, int N) {
  const int n = blockIdx.x * 32 + (threadIdx.x & 31);
  const int ty = threadIdx.x >> 5;
  __shared__ float part[8][33];
  float acc = 0.f;
  if (n < N)
    for (int m = blockIdx.y * 8 + ty; m < M; m += gridDim.y * 8) acc += __bfloat162float(x[(size_t)m * N + n]);
  part[ty][threadIdx.x & 31] = acc;
  __syncthreads();
  if (ty == 0 && n < N) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += part[i][threadIdx.x & 31];
    atomicAdd(out + n, s);
  }
}

// Same for N % 8 == 0: a thread owns 8 adjacent columns (one 16-byte load per row), a warp 256 columns,
// the 8 warps of a CTA stride over rows; shared-memory reduction over the warps, one atomic per column per CTA.
__global__ void __launch_bounds__(256)
colsum_bf16_v8_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ out, int M, int N) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c0 = blockIdx.x * 256 + lane * 8;
  __shared__ float part[8][256 + 8];
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (c0 < N) {
    for (int m = blockIdx.y * 8 + warp; m < M; m += gridDim.y * 8) {
      const uint4 v = *reinterpret_cast<const uint4*>(x + (size_t)m * N + c0);
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __bfloat1622float2(h[j]);
        acc[2 * j] += f.x;
        acc[2 * j + 1] += f.y;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) part[warp][lane * 8 + j] = acc[j];
  __syncthreads();
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c < N) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += part[w][threadIdx.x];
    atomicAdd(out + c, s);
  }
}

// gelu'(v), tanh approximation or erf.  Every operation is an explicitly rounded intrinsic, so the compiler cannot contract
// it differently in the two kernels below: the fused-bias kernel must reproduce ner_gelu_bwd_bf16 bit for bit.
__device__ __forceinline__ float gelu_grad(float v, int erf_variant) {
  if (erf_variant) {
    const float cdf = __fmul_rn(0.5f, __fadd_rn(1.f, erff(__fmul_rn(v, 0.7071067811865476f))));
    const float pdf = __expf(__fmul_rn(__fmul_rn(-0.5f, v), v));
    return __fadd_rn(cdf, __fmul_rn(__fmul_rn(v, 0.3989422804014327f), pdf));
  }
  const float v2 = __fmul_rn(v, v);
  const float u = __fmul_rn(0.7978845608028654f, __fadd_rn(v, __fmul_rn(__fmul_rn(0.044715f, v2), v)));
  const float t = tanhf(u);
  const float du = __fmul_rn(0.7978845608028654f, __fadd_rn(1.f, __fmul_rn(3.f * 0.044715f, v2)));
  return __fadd_rn(__fmul_rn(0.5f, __fadd_rn(1.f, t)), __fmul_rn(__fmul_rn(__fmul_rn(0.5f, v), __fsub_rn(1.f, __fmul_rn(t, t))), du));
}

// d_pre = d_act * gelu'(pre)   (tanh approximation or erf), all bf16
__global__ void __launch_bounds__(256)
gelu_bwd_kernel(const __nv_bfloat16* __restrict__ pre, const __nv_bfloat16* __restrict__ dact,
                __nv_bfloat16* __restrict__ dpre, size_t n4, int erf_variant) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 x = ld_bf16x4(pre + 4 * i), g = ld_bf16x4(dact + 4 * i);
    float xs[4] = {x.x, x.y, x.z, x.w}, gs[4] = {g.x, g.y, g.z, g.w}, o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) o[k] = gs[k] * gelu_grad(xs[k], erf_variant);
    st_bf16x4(dpre + 4 * i, make_float4(o[0], o[1], o[2], o[3]));
  }
}

// The same with the bias gradient of the dense layer in front of the GELU fused in: d_bias[c] += sum over rows of d_pre[:, c]
// (2-D tiling of colsum_bf16_v8_kernel: a lane owns 8 consecutive columns, the CTA's 8 warps stride over rows).
__global__ void __launch_bounds__(256)
gelu_bwd_bias_kernel(const __nv_bfloat16* __restrict__ pre, const __nv_bfloat16* __restrict__ dact,
                     __nv_bfloat16* __restrict__ dpre, float* __restrict__ dbias, int M, int N, int erf_variant) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c0 = blockIdx.x * 256 + lane * 8;
  __shared__ float part[8][256 + 8];
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (c0 < N) {
    for (int m = blockIdx.y * 8 + warp; m < M; m += gridDim.y * 8) {
      const size_t o = (size_t)m * N + c0;
      const float4 x0 = ld_bf16x4(pre + o), x1 = ld_bf16x4(pre + o + 4), g0 = ld_bf16x4(dact + o), g1 = ld_bf16x4(dact + o + 4);
      float4 d0, d1;
      d0.x = g0.x * gelu_grad(x0.x, erf_variant); d0.y = g0.y * gelu_grad(x0.y, erf_variant);
      d0.z = g0.z * gelu_grad(x0.z, erf_variant); d0.w = g0.w * gelu_grad(x0.w, erf_variant);
      d1.x = g1.x * gelu_grad(x1.x, erf_variant); d1.y = g1.y * gelu_grad(x1.y, erf_variant);
      d1.z = g1.z * gelu_grad(x1.z, erf_variant); d1.w = g1.w * gelu_grad(x1.w, erf_variant);
      st_bf16x4(dpre + o, d0);
      st_bf16x4(dpre + o + 4, d1);
      // the separate column-sum pass read the bf16-rounded d_pre: sum the rounded values here too
      auto rb = [](float v) { return __bfloat162float(__float2bfloat16_rn(v)); };
      acc[0] += rb(d0.x); acc[1] += rb(d0.y); acc[2] += rb(d0.z); acc[3] += rb(d0.w);
      acc[4] += rb(d1.x); acc[5] += rb(d1.y); acc[6] += rb(d1.z); acc[7] += rb(d1.w);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) part[warp][lane * 8 + j] = acc[j];
  __syncthreads();
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c < N) {
    float sum = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) sum += part[w][threadIdx.x];
    atomicAdd(dbias + c, sum);
  }
}

// gelu forward on a bf16 pre-activation (training keeps `pre` for the backward pass)
__global__ void __launch_bounds__(256)
gelu_fwd_kernel(const __nv_bfloat16* __restrict__ pre, __nv_bfloat16* __restrict__ act, size_t n4, int erf_variant) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 x = ld_bf16x4(pre + 4 * i);
    float xs[4] = {x.x, x.y, x.z, x.w}, o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float v = xs[k];
      if (erf_variant) o[k] = 0.5f * v * (1.f + erff(v * 0.7071067811865476f));
      else o[k] = 0.5f * v * (1.f + tanhf(0.7978845608028654f * (v + 0.044715f * v * v * v)));
    }
    st_bf16x4(act + 4 * i, make_float4(o[0], o[1], o[2], o[3]));
  }
}

// embedding backward: d_word[ids[tok]] += dx[tok], d_type[seg[tok]] += dx[tok], d_pos[tok % L] += dx[tok]
__global__ void __launch_bounds__(256)
bert_embed_bwd_kernel(const float* __restrict__ dx, const int32_t* __restrict__ ids, const int32_t* __restrict__ seg,
                      float* __restrict__ d_word, float* __restrict__ d_type, float* __restrict__ d_pos, int n_tok, int L,
                      int H, int V, int n_type) {
  const int lane = threadIdx.x & 31;
  for (int tok = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); tok < n_tok; tok += gridDim.x * (blockDim.x >> 5)) {
    const int id = min(max(ids[tok], 0), V - 1);
    const int sg = seg ? min(max(seg[tok], 0), n_type - 1) : 0;
    const int pos = tok % L;
    const float* g = dx + (size_t)tok * H;
    for (int e = lane; e < H; e += 32) {
      const float v = g[e];
      atomicAdd(d_word + (size_t)id * H + e, v);
      atomicAdd(d_type + (size_t)sg * H + e, v);
      atomicAdd(d_pos + (size_t)pos * H + e, v);
    }
  }
}

int rows_grid(int rows, int per_block) {
  long g = ((long)rows + per_block - 1) / per_block;
  if (g > (long)ner_num_sms() * 8) g = (long)ner_num_sms() * 8;
  if (g < 1) g = 1;
  return (int)g;
}
int flat_grid(size_t n) {
  size_t g = (n + 255) / 256;
  if (g > ner_num_sms() * 16) g = ner_num_sms() * 16;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace

extern "C" int ner_layernorm_dropout_bwd_bias(const void* y, int y_is_bf16, const float* residual, const float* gamma,
                                              const float* d_out, float* dz_f32, void* dz_bf16, float* d_gamma, float* d_beta,
                                              float* d_bias, int M, int H, float eps, float keep_prob, uint64_t seed,
                                              ner_stream_t stream);

extern "C" int ner_layernorm_dropout_bwd(const void* y, int y_is_bf16, const float* residual, const float* gamma,
                                         const float* d_out, float* dz_f32, void* dz_bf16, float* d_gamma, float* d_beta,
                                         int M, int H, float eps, float keep_prob, uint64_t seed, ner_stream_t stream) {
  return ner_layernorm_dropout_bwd_bias(y, y_is_bf16, residual, gamma, d_out, dz_f32, dz_bf16, d_gamma, d_beta, nullptr, M, H, eps,
                                        keep_prob, seed, stream);
}

extern "C" int ner_layernorm_dropout_bwd_bias(const void* y, int y_is_bf16, const float* residual, const float* gamma,
                                              const float* d_out, float* dz_f32, void* dz_bf16, float* d_gamma, float* d_beta,
                                              float* d_bias, int M, int H, float eps, float keep_prob, uint64_t seed,
                                              ner_stream_t stream) {
  if (M < 0 || H < 4) return NER_ERR_INVALID_ARG;
  if (M == 0) return NER_OK;
  if (!y || !gamma || !d_out || !d_gamma || !d_beta || (!dz_f32 && !dz_bf16)) return NER_ERR_INVALID_ARG;
  if (!(keep_prob > 0.f) || keep_prob > 1.f) return NER_ERR_INVALID_ARG;
  if (H % 4 != 0 || H > 128 * LN_MAXV) return NER_ERR_UNSUPPORTED;
  const size_t smem = (size_t)8 * 3 * H * 4;   // per-warp column partials
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // two CTAs per SM: rows per CTA sized so that the grid covers 2 x #SMs CTA slots once
  int per_block = ((M + 2 * ner_num_sms() - 1) / (2 * ner_num_sms()) + 7) / 8 * 8;
  per_block = per_block < 8 ? 8 : (per_block > 64 ? 64 : per_block);
  const int grid = rows_grid(M, per_block);
  const bool drop = keep_prob < 1.f;
  const int nv = (H / 4 + 31) / 32;
  using KernT = void (*)(const void*, const float*, const float*, const float*, float*, __nv_bfloat16*, float*, float*, float*, int,
                         int, float, float, uint32_t, uint32_t);
  KernT kern = nullptr;
#define LN_PICK(NVV)                                                                                                   \
  kern = y_is_bf16 ? (drop ? (KernT)layernorm_bwd_kernel<true, true, NVV> : (KernT)layernorm_bwd_kernel<true, false, NVV>)  \
                   : (drop ? (KernT)layernorm_bwd_kernel<false, true, NVV> : (KernT)layernorm_bwd_kernel<false, false, NVV>)
  if (nv <= 2) { LN_PICK(2); } else if (nv <= 4) { LN_PICK(4); } else if (nv <= 6) { LN_PICK(6); } else { LN_PICK(8); }
#undef LN_PICK
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  kern<<<grid, 256, smem, st>>>(y, residual, gamma, d_out, dz_f32, static_cast<__nv_bfloat16*>(dz_bf16), d_gamma, d_beta, d_bias, M,
                                H, eps, keep_prob, (uint32_t)seed, (uint32_t)(seed >> 32));
  return ner_launch_status();
}

extern "C" int ner_layernorm_bwd(const void* y, int y_is_bf16, const float* residual, const float* gamma,
                                 const float* d_out, float* dz_f32, void* dz_bf16, float* d_gamma, float* d_beta, int M,
                                 int H, float eps, ner_stream_t stream) {
  return ner_layernorm_dropout_bwd(y, y_is_bf16, residual, gamma, d_out, dz_f32, dz_bf16, d_gamma, d_beta, M, H, eps, 1.0f, 0,
                                   stream);
}

extern "C" int ner_transpose_bf16(const void* src_bf16, void* dst_bf16, int M, int N, int Mp, ner_stream_t stream) {
  if (M < 1 || N < 1 || Mp < M || !src_bf16 || !dst_bf16) return NER_ERR_INVALID_ARG;
  dim3 grid((N + 63) / 64, (Mp + 63) / 64);
  const bool vec = (N % 2 == 0) && (Mp % 8 == 0) && ((reinterpret_cast<uintptr_t>(src_bf16) & 3) == 0) &&
                   ((reinterpret_cast<uintptr_t>(dst_bf16) & 15) == 0);
  if (vec)
    transpose_bf16_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(src_bf16), static_cast<__nv_bfloat16*>(dst_bf16), M, N, Mp);
  else
    transpose_bf16_scalar_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(src_bf16), static_cast<__nv_bfloat16*>(dst_bf16), M, N, Mp);
  return ner_launch_status();
}

extern "C" int ner_colsum_bf16_add(const void* x_bf16, float* out, int M, int N, ner_stream_t stream) {
  if (M < 0 || N < 1 || !x_bf16 || !out) return NER_ERR_INVALID_ARG;
  if (M == 0) return NER_OK;
  if (N % 8 == 0 && (reinterpret_cast<uintptr_t>(x_bf16) & 15) == 0) {
    const int cb = (N + 255) / 256;
    int gy = (2 * ner_num_sms() + cb - 1) / cb;          // ~2 CTAs per SM in total
    if (gy > (M + 7) / 8) gy = (M + 7) / 8;
    colsum_bf16_v8_kernel<<<dim3(cb, gy), 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const __nv_bfloat16*>(x_bf16),
                                                                                        out, M, N);
    return ner_launch_status();
  }
  dim3 grid((N + 31) / 32, M >= 4096 ? 32 : (M >= 256 ? 8 : 1));
  colsum_bf16_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const __nv_bfloat16*>(x_bf16), out, M, N);
  return ner_launch_status();
}

// GELU on f32 activations (the fp32-accurate BERT mode keeps the FFN intermediate in f32)
__global__ void __launch_bounds__(256) gelu_f32_kernel(const float* __restrict__ x, float* __restrict__ y, size_t n, int erf_variant) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float v = x[i];
    if (erf_variant)
      y[i] = 0.5f * v * (1.f + erff(v * 0.7071067811865476f));
    else
      y[i] = 0.5f * v * (1.f + tanhf(0.7978845608028654f * (v + 0.044715f * v * v * v)));
  }
}

extern "C" int ner_gelu_f32(const float* x, float* y, size_t n, int erf_variant, ner_stream_t stream) {
  if (!x || !y) return n == 0 ? NER_OK : NER_ERR_INVALID_ARG;
  if (n == 0) return NER_OK;
  gelu_f32_kernel<<<flat_grid(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, y, n, erf_variant);
  return ner_launch_status();
}

extern "C" int ner_gelu_bf16(const void* pre_bf16, void* act_bf16, size_t n, int erf_variant, ner_stream_t stream) {
  if (!pre_bf16 || !act_bf16 || (n % 4) != 0) return n == 0 ? NER_OK : NER_ERR_INVALID_ARG;
  if (n == 0) return NER_OK;
  gelu_fwd_kernel<<<flat_grid(n / 4), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(pre_bf16), static_cast<__nv_bfloat16*>(act_bf16), n / 4, erf_variant);
  return ner_launch_status();
}

extern "C" int ner_gelu_bwd_bf16(const void* pre_bf16, const void* dact_bf16, void* dpre_bf16, size_t n, int erf_variant,
                                 ner_stream_t stream) {
  if (!pre_bf16 || !dact_bf16 || !dpre_bf16 || (n % 4) != 0) return n == 0 ? NER_OK : NER_ERR_INVALID_ARG;
  if (n == 0) return NER_OK;
  gelu_bwd_kernel<<<flat_grid(n / 4), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(pre_bf16), static_cast<const __nv_bfloat16*>(dact_bf16),
      static_cast<__nv_bfloat16*>(dpre_bf16), n / 4, erf_variant);
  return ner_launch_status();
}

extern "C" int ner_gelu_bwd_bias_bf16(const void* pre_bf16, const void* dact_bf16, void* dpre_bf16, float* d_bias, int M, int N,
                                      int erf_variant, ner_stream_t stream) {
  if (M < 0 || N < 1) return NER_ERR_INVALID_ARG;
  if (M == 0) return NER_OK;
  if (!pre_bf16 || !dact_bf16 || !dpre_bf16 || !d_bias) return NER_ERR_INVALID_ARG;
  if (N % 8 != 0 || ((reinterpret_cast<uintptr_t>(pre_bf16) | reinterpret_cast<uintptr_t>(dact_bf16) |
                      reinterpret_cast<uintptr_t>(dpre_bf16)) & 15) != 0)
    return NER_ERR_UNSUPPORTED;
  const int cb = (N + 255) / 256;
  int gy = (4 * ner_num_sms() + cb - 1) / cb;
  if (gy > (M + 7) / 8) gy = (M + 7) / 8;
  gelu_bwd_bias_kernel<<<dim3(cb, gy), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(pre_bf16), static_cast<const __nv_bfloat16*>(dact_bf16),
      static_cast<__nv_bfloat16*>(dpre_bf16), d_bias, M, N, erf_variant);
  return ner_launch_status();
}

extern "C" int ner_bert_embed_bwd(const float* dx, const int32_t* ids, const int32_t* seg, float* d_word, float* d_type,
                                  float* d_pos, int B, int L, int H, int vocab, int n_type, ner_stream_t stream) {
  if (B < 0 || L < 1 || H < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!dx || !ids || !d_word || !d_type || !d_pos) return NER_ERR_INVALID_ARG;
  bert_embed_bwd_kernel<<<rows_grid(B * L, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(dx, ids, seg, d_word, d_type,
                                                                                          d_pos, B * L, L, H, vocab, n_type);
  return ner_launch_status();
}
