// HBM-bound glue kernels of the encoder path (sm_90a): embedding-sum + LayerNorm, LayerNorm,
// weight packing / casts, and the small-N (label_size) dense projection.
//
// Reference call sites: bert_base.bert.modeling (embedding_postprocessor, layer_norm) executed
// from tools/layer.py:68-77; tf.layers.dense(units=label_size) at model/bert_bilstm_crf.py:26
// and model/bert_crf.py:20; tools/transformer/modules.py:40-65 (layer_norm, eps = fp32 eps).
#include "common.cuh"

namespace {

using namespace nerdev;

constexpr int LN_MAXV = 8;  // float4 per lane -> H <= 1024

// Row LayerNorm over registers: v holds this lane's float4s (nv4 valid), H = row length.
// Matches tf.contrib.layers.layer_norm / tf.nn.moments: biased variance of (x - mean).
// Q: also write the row as e4m3 (out_q) with one scale per 128 columns (out_s).  Needs H % 128 == 0: float4 k of every lane
// is then valid and the 32 lanes' float4 k are exactly columns [128k, 128k + 128), so a block's amax is one warp_max.
template <bool Q = false>
__device__ __forceinline__ void ln_row(float4 (&v)[LN_MAXV], int nv4, int H, int lane, float eps,
                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                       float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_bf16,
                                       uint8_t* __restrict__ out_q = nullptr, float* __restrict__ out_s = nullptr) {
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < LN_MAXV; ++k)
    if (k < nv4 && (lane + 32 * k) * 4 < H) s += v[k].x + v[k].y + v[k].z + v[k].w;
  s = warp_sum(s);
  const float mean = s / (float)H;
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < LN_MAXV; ++k)
    if (k < nv4 && (lane + 32 * k) * 4 < H) {
      const float a = v[k].x - mean, b = v[k].y - mean, c = v[k].z - mean, d = v[k].w - mean;
      q += a * a + b * b + c * c + d * d;
    }
  q = warp_sum(q);
  const float rstd = rsqrtf(q / (float)H + eps);
#pragma unroll
  for (int k = 0; k < LN_MAXV; ++k) {
    const int e = (lane + 32 * k) * 4;
    if (k < nv4 && e < H) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + e));
      const float4 b = __ldg(reinterpret_cast<const float4*>(beta + e));
      float4 o;
      o.x = (v[k].x - mean) * rstd * g.x + b.x;
      o.y = (v[k].y - mean) * rstd * g.y + b.y;
      o.z = (v[k].z - mean) * rstd * g.z + b.z;
      o.w = (v[k].w - mean) * rstd * g.w + b.w;
      if (out_f32 != nullptr) *reinterpret_cast<float4*>(out_f32 + e) = o;
      if (out_bf16 != nullptr) {
        __nv_bfloat162 lo = __floats2bfloat162_rn(o.x, o.y), hi = __floats2bfloat162_rn(o.z, o.w);
        uint2 pk;
        pk.x = *reinterpret_cast<uint32_t*>(&lo);
        pk.y = *reinterpret_cast<uint32_t*>(&hi);
        *reinterpret_cast<uint2*>(out_bf16 + e) = pk;
      }
      if constexpr (Q) {
        const float s = e4m3_scale(warp_max(fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w)))));
        const uint32_t lo = cvt_e4m3x2(__fdiv_rn(o.x, s), __fdiv_rn(o.y, s)), hi = cvt_e4m3x2(__fdiv_rn(o.z, s), __fdiv_rn(o.w, s));
        *reinterpret_cast<uint32_t*>(out_q + e) = lo | (hi << 16);
        if (lane == 0) out_s[k] = s;
      }
    }
  }
}

// one warp per token; Q: also the e4m3 + block-scale copy (out_q [n_tok, H], out_s [n_tok, H/128])
template <bool Q>
__global__ void __launch_bounds__(256)
bert_embed_ln_kernel(const float* __restrict__ word_emb, const float* __restrict__ type_emb,
                     const float* __restrict__ pos_emb, const float* __restrict__ gamma,
                     const float* __restrict__ beta, const int32_t* __restrict__ ids,
                     const int32_t* __restrict__ seg, float* __restrict__ out_f32,
                     __nv_bfloat16* __restrict__ out_bf16, int n_tok, int L, int H, int V, int n_type, float eps,
                     const int32_t* __restrict__ tok_src, uint8_t* __restrict__ out_q, float* __restrict__ out_s) {
  const int lane = threadIdx.x & 31;
  const int nv4 = (H / 4 + 31) / 32;
  for (int tok = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); tok < n_tok; tok += gridDim.x * (blockDim.x >> 5)) {
    const int src = tok_src ? tok_src[tok] : tok;  // packed row -> padded (b*L + pos) index
    int id = ids[src];
    id = min(max(id, 0), V - 1);
    int sg = (seg != nullptr) ? seg[src] : 0;
    sg = min(max(sg, 0), n_type - 1);
    const int pos = src % L;
    const float* w = word_emb + (size_t)id * H;
    const float* ty = type_emb + (size_t)sg * H;
    const float* po = pos_emb + (size_t)pos * H;
    float4 v[LN_MAXV];
#pragma unroll
    for (int k = 0; k < LN_MAXV; ++k) {
      const int e = (lane + 32 * k) * 4;
      if (k < nv4 && e < H) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(w + e));
        const float4 b = __ldg(reinterpret_cast<const float4*>(ty + e));
        const float4 c = __ldg(reinterpret_cast<const float4*>(po + e));
        v[k] = make_float4(a.x + b.x + c.x, a.y + b.y + c.y, a.z + b.z + c.z, a.w + b.w + c.w);
      }
    }
    ln_row<Q>(v, nv4, H, lane, eps, gamma, beta, out_f32 ? out_f32 + (size_t)tok * H : nullptr,
              out_bf16 ? out_bf16 + (size_t)tok * H : nullptr, Q ? out_q + (size_t)tok * H : nullptr,
              Q ? out_s + (size_t)tok * (H / 128) : nullptr);
  }
}

// word + token_type + position, no LayerNorm (the pre-LN sum the embedding LayerNorm backward needs)
__global__ void __launch_bounds__(256)
bert_embed_sum_kernel(const float* __restrict__ word_emb, const float* __restrict__ type_emb,
                      const float* __restrict__ pos_emb, const int32_t* __restrict__ ids, const int32_t* __restrict__ seg,
                      float* __restrict__ out, int n_tok, int L, int H, int V, int n_type) {
  const int lane = threadIdx.x & 31;
  for (int tok = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); tok < n_tok; tok += gridDim.x * (blockDim.x >> 5)) {
    const int id = min(max(ids[tok], 0), V - 1);
    const int sg = min(max(seg != nullptr ? seg[tok] : 0, 0), n_type - 1);
    const float* w = word_emb + (size_t)id * H;
    const float* ty = type_emb + (size_t)sg * H;
    const float* po = pos_emb + (size_t)(tok % L) * H;
    for (int e = lane * 4; e < H; e += 128) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(w + e));
      const float4 b = __ldg(reinterpret_cast<const float4*>(ty + e));
      const float4 c = __ldg(reinterpret_cast<const float4*>(po + e));
      *reinterpret_cast<float4*>(out + (size_t)tok * H + e) = make_float4(a.x + b.x + c.x, a.y + b.y + c.y, a.z + b.z + c.z, a.w + b.w + c.w);
    }
  }
}

// y (+ optional residual) -> LayerNorm -> fp32 and/or bf16.  y is fp32 or (YBF16) bf16.
// DROP: y is first passed through dropout (counter-based mask of ner_dropout: element index row*H + col) —
// BertModel's hidden dropout in front of the residual add, fused so the dropped tensor is never written.
// Q: also the e4m3 + block-scale copy (out_q [M, H], out_s [M, H/128]).
template <bool YBF16, bool DROP, bool Q>
__global__ void __launch_bounds__(256)
layernorm_kernel(const void* __restrict__ yv, const float* __restrict__ residual, const float* __restrict__ gamma,
                 const float* __restrict__ beta, float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_bf16,
                 int M, int H, float eps, float keep, uint32_t seed_lo, uint32_t seed_hi, uint8_t* __restrict__ out_q,
                 float* __restrict__ out_s) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int nv4 = (H / 4 + 31) / 32;
  const uint32_t thr = keep_threshold(keep);
  const float inv_keep = 1.f / keep;
  for (int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < M; row += gridDim.x * (blockDim.x >> 5)) {
    const float* r = residual ? residual + (size_t)row * H : nullptr;
    float4 v[LN_MAXV];
#pragma unroll
    for (int k = 0; k < LN_MAXV; ++k) {
      const int e = (lane + 32 * k) * 4;
      if (k < nv4 && e < H) {
        if constexpr (YBF16) {
          const uint2 pk = *reinterpret_cast<const uint2*>(static_cast<const __nv_bfloat16*>(yv) + (size_t)row * H + e);
          const __nv_bfloat162 lo = *reinterpret_cast<const __nv_bfloat162*>(&pk.x);
          const __nv_bfloat162 hi = *reinterpret_cast<const __nv_bfloat162*>(&pk.y);
          v[k] = make_float4(__low2float(lo), __high2float(lo), __low2float(hi), __high2float(hi));
        } else {
          v[k] = *reinterpret_cast<const float4*>(static_cast<const float*>(yv) + (size_t)row * H + e);
        }
        if constexpr (DROP) {
          const size_t i = (size_t)row * H + e;
          const uint32_t hi = seed_hi ^ (uint32_t)(i >> 32), lo = (uint32_t)i;
          v[k].x = hash3(seed_lo, hi, lo) < thr ? v[k].x * inv_keep : 0.f;
          v[k].y = hash3(seed_lo, hi, lo + 1) < thr ? v[k].y * inv_keep : 0.f;
          v[k].z = hash3(seed_lo, hi, lo + 2) < thr ? v[k].z * inv_keep : 0.f;
          v[k].w = hash3(seed_lo, hi, lo + 3) < thr ? v[k].w * inv_keep : 0.f;
        }
        if (r != nullptr) {
          const float4 b = *reinterpret_cast<const float4*>(r + e);
          v[k].x += b.x;
          v[k].y += b.y;
          v[k].z += b.z;
          v[k].w += b.w;
        }
      }
    }
    ln_row<Q>(v, nv4, H, lane, eps, gamma, beta, out_f32 ? out_f32 + (size_t)row * H : nullptr,
              out_bf16 ? out_bf16 + (size_t)row * H : nullptr, Q ? out_q + (size_t)row * H : nullptr,
              Q ? out_s + (size_t)row * (H / 128) : nullptr);
  }
}

// TF dense kernel [K,N] fp32  ->  bf16 [N,K] (K contiguous) through a 32x33 smem tile
__global__ void __launch_bounds__(256)
pack_weight_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int K, int N) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8) {
    const int k = k0 + i, n = n0 + tx;
    tile[i][tx] = (k < K && n < N) ? src[(size_t)k * N + n] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int n = n0 + i, k = k0 + tx;
    if (n < N && k < K) dst[(size_t)n * K + k] = __float2bfloat16_rn(tile[tx][i]);
  }
}

// Every bf16 copy of a group of dense kernels in ONE launch (TRAIN re-packs all weights after each optimizer step): per
// 64 x 64 tile of a TF-layout fp32 kernel [K, N] write (a) the bf16 cast in the same layout into dst_kn (+ column offset through
// ld_kn: the fused [H, 3H] Q|K|V operand of the data-gradient GEMM) and (b) the transposed bf16 [N, K] pack into dst_nk (K
// contiguous: the B operand of the forward GEMMs; stacking the Q, K, V packs gives the fused [3H, H] operand).  One read of
// the fp32 weights, both writes coalesced (the transpose goes through shared memory).
__global__ void __launch_bounds__(256)
pack_group_kernel(const ner_pack_entry* __restrict__ entries, const int32_t* __restrict__ tile_start, int count) {
  __shared__ __nv_bfloat16 tile[64][66];
  int e = 0;
  {
    int lo = 0, hi = count;                 // last entry whose first tile is <= blockIdx.x
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (tile_start[mid] <= (int)blockIdx.x) lo = mid; else hi = mid;
    }
    e = lo;
  }
  const ner_pack_entry en = entries[e];
  const int t = blockIdx.x - tile_start[e], tn = (en.N + 63) / 64;
  const int k0 = (t / tn) * 64, n0 = (t % tn) * 64;
  const int c4 = (threadIdx.x & 15) * 4, r = threadIdx.x >> 4;
  __nv_bfloat16* kn = static_cast<__nv_bfloat16*>(en.dst_kn_bf16);
  __nv_bfloat16* nk = static_cast<__nv_bfloat16*>(en.dst_nk_bf16);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int k = k0 + r + 16 * i, n = n0 + c4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k < en.K) {
      if (n + 3 < en.N && (en.N & 3) == 0) v = *reinterpret_cast<const float4*>(en.src + (size_t)k * en.N + n);
      else {
        if (n < en.N) v.x = en.src[(size_t)k * en.N + n];
        if (n + 1 < en.N) v.y = en.src[(size_t)k * en.N + n + 1];
        if (n + 2 < en.N) v.z = en.src[(size_t)k * en.N + n + 2];
        if (n + 3 < en.N) v.w = en.src[(size_t)k * en.N + n + 3];
      }
    }
    const __nv_bfloat16 b0 = __float2bfloat16_rn(v.x), b1 = __float2bfloat16_rn(v.y), b2 = __float2bfloat16_rn(v.z),
                        b3 = __float2bfloat16_rn(v.w);
    tile[r + 16 * i][c4] = b0; tile[r + 16 * i][c4 + 1] = b1; tile[r + 16 * i][c4 + 2] = b2; tile[r + 16 * i][c4 + 3] = b3;
    if (kn != nullptr && k < en.K) {
      __nv_bfloat16* d = kn + (size_t)k * en.ld_kn + n;
      if (n + 3 < en.N && (en.ld_kn & 3) == 0 && (reinterpret_cast<uintptr_t>(kn) & 7) == 0) {
        __nv_bfloat162 lo = __halves2bfloat162(b0, b1), hi = __halves2bfloat162(b2, b3);
        *reinterpret_cast<uint2*>(d) = make_uint2(*reinterpret_cast<uint32_t*>(&lo), *reinterpret_cast<uint32_t*>(&hi));
      } else {
        if (n < en.N) d[0] = b0;
        if (n + 1 < en.N) d[1] = b1;
        if (n + 2 < en.N) d[2] = b2;
        if (n + 3 < en.N) d[3] = b3;
      }
    }
  }
  __syncthreads();
  if (nk != nullptr) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int n = n0 + r + 16 * i, k = k0 + c4;
      if (n < en.N) {
        __nv_bfloat16* d = nk + (size_t)n * en.ld_nk + k;
        const __nv_bfloat16 b0 = tile[c4][r + 16 * i], b1 = tile[c4 + 1][r + 16 * i], b2 = tile[c4 + 2][r + 16 * i],
                            b3 = tile[c4 + 3][r + 16 * i];
        if (k + 3 < en.K && (en.ld_nk & 3) == 0 && (reinterpret_cast<uintptr_t>(nk) & 7) == 0) {
          __nv_bfloat162 lo = __halves2bfloat162(b0, b1), hi = __halves2bfloat162(b2, b3);
          *reinterpret_cast<uint2*>(d) = make_uint2(*reinterpret_cast<uint32_t*>(&lo), *reinterpret_cast<uint32_t*>(&hi));
        } else {
          if (k < en.K) d[0] = b0;
          if (k + 1 < en.K) d[1] = b1;
          if (k + 2 < en.K) d[2] = b2;
          if (k + 3 < en.K) d[3] = b3;
        }
      }
    }
  }
}

// TF dense kernel [K,N] fp32 -> e4m3 [N,K] (K contiguous) with one scale per output channel n (= column of src).  One CTA per
// 32 channels: the column amax over K, then the scaled, transposed pack through a 32 x 33 smem tile.
__global__ void __launch_bounds__(256)
quantize_weight_e4m3_kernel(const float* __restrict__ src, uint8_t* __restrict__ dst, float* __restrict__ scale, int K, int N) {
  __shared__ float tile[32][33];
  __shared__ float red[8][32];
  const int n0 = blockIdx.x * 32, tx = threadIdx.x & 31, ty = threadIdx.x >> 5, n = n0 + tx;
  float m = 0.f;
  if (n < N)
    for (int k = ty; k < K; k += 8) m = fmaxf(m, fabsf(src[(size_t)k * N + n]));
  red[ty][tx] = m;
  __syncthreads();
  if (ty == 0) {
    for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i][tx]);
    const float s = e4m3_scale(m);
    red[0][tx] = s;
    if (n < N) scale[n] = s;
  }
  __syncthreads();
  for (int k0 = 0; k0 < K; k0 += 32) {
    for (int i = ty; i < 32; i += 8) {
      const int k = k0 + i;
      tile[i][tx] = (k < K && n < N) ? src[(size_t)k * N + n] : 0.f;
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
      const int nn = n0 + i, k = k0 + tx;
      if (nn < N && k < K) dst[(size_t)nn * K + k] = (uint8_t)(cvt_e4m3x2(__fdiv_rn(tile[tx][i], red[0][i]), 0.f) & 0xffu);
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256)
cast_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dst[i] = __float2bfloat16_rn(src[i]);
}

// out[M,N] = x[M,F] · W[F,N] + b[N], N <= 32 (label_size).  W staged in smem; one warp per row,
// lanes split F, N partial sums reduced with shuffles.  x is fp32 or bf16.
template <typename XT, int NMAX>
__global__ void __launch_bounds__(256)
dense_small_n_kernel(const XT* __restrict__ x, const float* __restrict__ W, const float* __restrict__ bias,
                     float* __restrict__ out, int M, int F, int N, const int32_t* __restrict__ row_map) {
  extern __shared__ float s_w[];  // [F][N]
  for (int e = threadIdx.x; e < F * N; e += blockDim.x) s_w[e] = W[e];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < M; row += gridDim.x * (blockDim.x >> 5)) {
    float acc[NMAX];
#pragma unroll
    for (int n = 0; n < NMAX; ++n) acc[n] = 0.f;
    const XT* xr = x + (size_t)row * F;
    for (int f = lane; f < F; f += 32) {
      float xv;
      if constexpr (sizeof(XT) == 2) xv = __bfloat162float(xr[f]);
      else xv = xr[f];
      const float* wr = s_w + f * N;
#pragma unroll
      for (int n = 0; n < NMAX; ++n)
        if (n < N) acc[n] = fmaf(xv, wr[n], acc[n]);
    }
#pragma unroll
    for (int n = 0; n < NMAX; ++n) acc[n] = warp_sum(acc[n]);
    if (lane < N) {
      float v = 0.f;
#pragma unroll
      for (int n = 0; n < NMAX; ++n)
        if (n == lane) v = acc[n];
      const size_t orow = row_map ? (size_t)row_map[row] : (size_t)row;
      out[orow * N + lane] = v + (bias ? bias[lane] : 0.f);
    }
  }
}


// out[tok, 0:E] (row stride ld_out) = table[ids[tok], :]   (tf.nn.embedding_lookup)
__global__ void __launch_bounds__(256)
embedding_lookup_kernel(const float* __restrict__ table, const int32_t* __restrict__ ids, float* __restrict__ out,
                        int n_tok, int E, int V, int ld_out) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int tok = blockIdx.x * wpb + (threadIdx.x >> 5); tok < n_tok; tok += gridDim.x * wpb) {
    const int id = min(max(ids[tok], 0), V - 1);
    const float* row = table + (size_t)id * E;
    float* o = out + (size_t)tok * ld_out;
    for (int e = lane; e < E; e += 32) o[e] = __ldg(row + e);
  }
}

// f32 [M,D] (row stride ld_src) -> bf16 [M,Dp], zero padded columns D..Dp-1
__global__ void __launch_bounds__(256)
cast_pad_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int M, int D, int Dp, int ld_src) {
  const size_t total = (size_t)M * Dp;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const size_t r = i / Dp;
    const int c = (int)(i - r * Dp);
    dst[i] = __float2bfloat16_rn(c < D ? src[r * ld_src + c] : 0.f);
  }
}

// Sequence-packing plan from a prefix mask [B,L]: len_b = sum(mask[b,:]); cu[b] = exclusive prefix
// sum; tok_src[cu[b] + t] = b*L + t.  One CTA (B <= 1024 rows handled by loops).
__global__ void __launch_bounds__(1024)
seq_pack_plan_kernel(const int32_t* __restrict__ mask, int32_t* __restrict__ cu, int32_t* __restrict__ tok_src, int B, int L) {
  extern __shared__ int s_plan[];  // [B+1]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int b = warp; b < B; b += nw) {
    int c = 0;
    for (int t = lane; t < L; t += 32) c += (mask[(size_t)b * L + t] != 0);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) s_plan[b + 1] = c;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    s_plan[0] = 0;
    for (int b = 0; b < B; ++b) s_plan[b + 1] += s_plan[b];
  }
  __syncthreads();
  for (int b = threadIdx.x; b <= B; b += blockDim.x) cu[b] = s_plan[b];
  for (int b = warp; b < B; b += nw) {
    const int o = s_plan[b], n = s_plan[b + 1] - o;
    for (int t = lane; t < n; t += 32) tok_src[o + t] = b * L + t;
  }
}

// f32 [M,D] (row stride ld_src) -> (hi, lo) bf16 [M,Dp]: hi = bf16(x), lo = bf16(x - hi); zero padded.
// hi + lo carries ~16 mantissa bits: three bf16 tensor-core products (hi*hi + hi*lo + lo*hi)
// reproduce an fp32 product to ~2^-17 (the fp32-accurate dense mode).
__global__ void __launch_bounds__(256)
split_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int M,
                  int D, int Dp, int ld_src) {
  const size_t total = (size_t)M * Dp;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const size_t r = i / Dp;
    const int c = (int)(i - r * Dp);
    const float x = c < D ? src[r * ld_src + c] : 0.f;
    const __nv_bfloat16 h = __float2bfloat16_rn(x);
    hi[i] = h;
    lo[i] = __float2bfloat16_rn(x - __bfloat162float(h));
  }
}

int grid_for_rows(int rows, int rows_per_block) {
  long g = ((long)rows + rows_per_block - 1) / rows_per_block;
  if (g > (long)ner_num_sms() * 16) g = (long)ner_num_sms() * 16;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace

extern "C" int ner_bert_embed_ln(const float* word_emb, const float* type_emb, const float* pos_emb,
                                 const float* gamma, const float* beta, const int32_t* ids, const int32_t* seg,
                                 float* out_f32, void* out_bf16, int B, int L, int H, int vocab, int n_type,
                                 int max_pos, float eps, const int32_t* tok_src, int n_packed, ner_stream_t stream) {
  if (B < 0 || L < 1 || H < 4 || vocab < 1 || n_type < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!word_emb || !type_emb || !pos_emb || !gamma || !beta || !ids || (!out_f32 && !out_bf16)) return NER_ERR_INVALID_ARG;
  if (H % 4 != 0 || H > 128 * LN_MAXV || L > max_pos) return NER_ERR_UNSUPPORTED;
  const int n_tok = tok_src ? n_packed : B * L;
  if (n_tok < 0 || n_tok > B * L) return NER_ERR_INVALID_ARG;
  if (n_tok == 0) return NER_OK;
  bert_embed_ln_kernel<false><<<grid_for_rows(n_tok, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      word_emb, type_emb, pos_emb, gamma, beta, ids, seg, out_f32, static_cast<__nv_bfloat16*>(out_bf16), n_tok, L, H,
      vocab, n_type, eps, tok_src, nullptr, nullptr);
  return ner_launch_status();
}

extern "C" int ner_bert_embed_sum(const float* word_emb, const float* type_emb, const float* pos_emb, const int32_t* ids,
                                  const int32_t* seg, float* out, int B, int L, int H, int vocab, int n_type, int max_pos,
                                  ner_stream_t stream) {
  if (B < 0 || L < 1 || H < 4 || H % 4 != 0) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!word_emb || !type_emb || !pos_emb || !ids || !out || L > max_pos) return NER_ERR_INVALID_ARG;
  bert_embed_sum_kernel<<<grid_for_rows(B * L, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(word_emb, type_emb, pos_emb, ids,
                                                                                             seg, out, B * L, L, H, vocab, n_type);
  return ner_launch_status();
}

extern "C" int ner_layernorm_dropout(const void* y, int y_is_bf16, const float* residual, const float* gamma,
                                     const float* beta, float* out_f32, void* out_bf16, int M, int H, float eps,
                                     float keep_prob, uint64_t seed, ner_stream_t stream) {
  if (M < 0 || H < 4) return NER_ERR_INVALID_ARG;
  if (M == 0) return NER_OK;
  if (!y || !gamma || !beta || (!out_f32 && !out_bf16)) return NER_ERR_INVALID_ARG;
  if (!(keep_prob > 0.f) || keep_prob > 1.f) return NER_ERR_INVALID_ARG;
  if (H % 4 != 0 || H > 128 * LN_MAXV) return NER_ERR_UNSUPPORTED;
  const bool drop = keep_prob < 1.f;
  auto kern = y_is_bf16 ? (drop ? layernorm_kernel<true, true, false> : layernorm_kernel<true, false, false>)
                        : (drop ? layernorm_kernel<false, true, false> : layernorm_kernel<false, false, false>);
  cudaError_t e = ner_launch_pdl(kern, dim3(grid_for_rows(M, 8)), dim3(256), 0, static_cast<cudaStream_t>(stream), y, residual,
                                 gamma, beta, out_f32, static_cast<__nv_bfloat16*>(out_bf16), M, H, eps, keep_prob,
                                 (uint32_t)seed, (uint32_t)(seed >> 32), (uint8_t*)nullptr, (float*)nullptr);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  return ner_launch_status();
}

extern "C" int ner_layernorm(const void* y, int y_is_bf16, const float* residual, const float* gamma,
                             const float* beta, float* out_f32, void* out_bf16, int M, int H, float eps,
                             ner_stream_t stream) {
  return ner_layernorm_dropout(y, y_is_bf16, residual, gamma, beta, out_f32, out_bf16, M, H, eps, 1.0f, 0, stream);
}

extern "C" int ner_pack_weight_bf16(const float* w_kn, void* wt_nk_bf16, int K, int N, ner_stream_t stream) {
  if (K < 1 || N < 1 || !w_kn || !wt_nk_bf16) return NER_ERR_INVALID_ARG;
  dim3 grid((N + 31) / 32, (K + 31) / 32);
  pack_weight_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(w_kn, static_cast<__nv_bfloat16*>(wt_nk_bf16), K, N);
  return ner_launch_status();
}

extern "C" int ner_pack_weights_group_bf16(const ner_pack_entry* entries_device, const int32_t* tile_start_device, int count,
                                           int total_tiles, ner_stream_t stream) {
  if (count < 0 || total_tiles < 0) return NER_ERR_INVALID_ARG;
  if (count == 0 || total_tiles == 0) return NER_OK;
  if (!entries_device || !tile_start_device) return NER_ERR_INVALID_ARG;
  pack_group_kernel<<<total_tiles, 256, 0, static_cast<cudaStream_t>(stream)>>>(entries_device, tile_start_device, count);
  return ner_launch_status();
}

extern "C" int ner_cast_bf16(const float* src, void* dst_bf16, size_t n, ner_stream_t stream) {
  if (!src || !dst_bf16) return n == 0 ? NER_OK : NER_ERR_INVALID_ARG;
  if (n == 0) return NER_OK;
  size_t g = (n + 255) / 256;
  if (g > ner_num_sms() * 32) g = ner_num_sms() * 32;
  cast_bf16_kernel<<<(int)g, 256, 0, static_cast<cudaStream_t>(stream)>>>(src, static_cast<__nv_bfloat16*>(dst_bf16), n);
  return ner_launch_status();
}

extern "C" int ner_dense_small_n(const void* x, int x_is_bf16, const float* W, const float* bias, float* out, int M,
                                 int F, int N, const int32_t* row_map, ner_stream_t stream) {
  if (M < 0 || F < 1 || N < 1) return NER_ERR_INVALID_ARG;
  if (M == 0) return NER_OK;
  if (!x || !W || !out) return NER_ERR_INVALID_ARG;
  if (N > 32 || (size_t)F * N * 4 > 200 * 1024) return NER_ERR_UNSUPPORTED;
  const size_t smem = (size_t)F * N * 4;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int grid = grid_for_rows(M, 8 * 4);
  cudaError_t e;
#define LAUNCH(XT, NM)                                                                                   \
  {                                                                                                      \
    auto kern = dense_small_n_kernel<XT, NM>;                                                            \
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);              \
    if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;                                             \
    kern<<<grid, 256, smem, st>>>(static_cast<const XT*>(x), W, bias, out, M, F, N, row_map);                     \
  }
  if (x_is_bf16) {
    if (N <= 16) LAUNCH(__nv_bfloat16, 16) else LAUNCH(__nv_bfloat16, 32)
  } else {
    if (N <= 16) LAUNCH(float, 16) else LAUNCH(float, 32)
  }
#undef LAUNCH
  return ner_launch_status();
}

extern "C" int ner_embedding_lookup(const float* table, const int32_t* ids, float* out, int n_tok, int E, int V,
                                    int ld_out, ner_stream_t stream) {
  if (n_tok < 0 || E < 1 || V < 1 || ld_out < E) return NER_ERR_INVALID_ARG;
  if (n_tok == 0) return NER_OK;
  if (!table || !ids || !out) return NER_ERR_INVALID_ARG;
  embedding_lookup_kernel<<<grid_for_rows(n_tok, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(table, ids, out, n_tok,
                                                                                               E, V, ld_out);
  return ner_launch_status();
}

extern "C" int ner_cast_pad_bf16(const float* src, void* dst_bf16, int M, int D, int Dp, int ld_src,
                                 ner_stream_t stream) {
  if (M < 0 || D < 1 || Dp < D || ld_src < D) return NER_ERR_INVALID_ARG;
  if (M == 0) return NER_OK;
  if (!src || !dst_bf16) return NER_ERR_INVALID_ARG;
  size_t g = ((size_t)M * Dp + 255) / 256;
  if (g > ner_num_sms() * 32) g = ner_num_sms() * 32;
  cast_pad_bf16_kernel<<<(int)g, 256, 0, static_cast<cudaStream_t>(stream)>>>(src, static_cast<__nv_bfloat16*>(dst_bf16), M,
                                                                              D, Dp, ld_src);
  return ner_launch_status();
}

extern "C" int ner_seq_pack_plan(const int32_t* mask, int32_t* cu_seqlens, int32_t* tok_src, int B, int L,
                                 ner_stream_t stream) {
  if (B < 0 || L < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!mask || !cu_seqlens || !tok_src) return NER_ERR_INVALID_ARG;
  if ((size_t)(B + 1) * 4 > 200 * 1024) return NER_ERR_UNSUPPORTED;
  const size_t smem = (size_t)(B + 1) * 4;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(seq_pack_plan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  }
  seq_pack_plan_kernel<<<1, 1024, smem, static_cast<cudaStream_t>(stream)>>>(mask, cu_seqlens, tok_src, B, L);
  return ner_launch_status();
}

extern "C" int ner_split_bf16(const float* src, void* hi_bf16, void* lo_bf16, int M, int D, int Dp, int ld_src,
                              ner_stream_t stream) {
  if (M < 0 || D < 1 || Dp < D || ld_src < D) return NER_ERR_INVALID_ARG;
  if (M == 0) return NER_OK;
  if (!src || !hi_bf16 || !lo_bf16) return NER_ERR_INVALID_ARG;
  size_t g = ((size_t)M * Dp + 255) / 256;
  if (g > ner_num_sms() * 32) g = ner_num_sms() * 32;
  split_bf16_kernel<<<(int)g, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      src, static_cast<__nv_bfloat16*>(hi_bf16), static_cast<__nv_bfloat16*>(lo_bf16), M, D, Dp, ld_src);
  return ner_launch_status();
}

extern "C" int ner_bert_embed_ln_e4m3(const float* word_emb, const float* type_emb, const float* pos_emb, const float* gamma,
                                      const float* beta, const int32_t* ids, const int32_t* seg, float* out_f32, void* out_bf16,
                                      void* out_e4m3, float* out_scale, int B, int L, int H, int vocab, int n_type, int max_pos,
                                      float eps, const int32_t* tok_src, int n_packed, ner_stream_t stream) {
  if (B < 0 || L < 1 || H < 4 || vocab < 1 || n_type < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!word_emb || !type_emb || !pos_emb || !gamma || !beta || !ids || !out_e4m3 || !out_scale) return NER_ERR_INVALID_ARG;
  if (H % 128 != 0 || H > 128 * LN_MAXV || L > max_pos) return NER_ERR_UNSUPPORTED;
  const int n_tok = tok_src ? n_packed : B * L;
  if (n_tok < 0 || n_tok > B * L) return NER_ERR_INVALID_ARG;
  if (n_tok == 0) return NER_OK;
  bert_embed_ln_kernel<true><<<grid_for_rows(n_tok, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      word_emb, type_emb, pos_emb, gamma, beta, ids, seg, out_f32, static_cast<__nv_bfloat16*>(out_bf16), n_tok, L, H,
      vocab, n_type, eps, tok_src, static_cast<uint8_t*>(out_e4m3), out_scale);
  return ner_launch_status();
}

extern "C" int ner_layernorm_e4m3(const void* y, int y_is_bf16, const float* residual, const float* gamma, const float* beta,
                                  float* out_f32, void* out_bf16, void* out_e4m3, float* out_scale, int M, int H, float eps,
                                  ner_stream_t stream) {
  if (M < 0 || H < 4) return NER_ERR_INVALID_ARG;
  if (M == 0) return NER_OK;
  if (!y || !gamma || !beta || !out_e4m3 || !out_scale) return NER_ERR_INVALID_ARG;
  if (H % 128 != 0 || H > 128 * LN_MAXV) return NER_ERR_UNSUPPORTED;
  auto kern = y_is_bf16 ? layernorm_kernel<true, false, true> : layernorm_kernel<false, false, true>;
  cudaError_t e = ner_launch_pdl(kern, dim3(grid_for_rows(M, 8)), dim3(256), 0, static_cast<cudaStream_t>(stream), y, residual,
                                 gamma, beta, out_f32, static_cast<__nv_bfloat16*>(out_bf16), M, H, eps, 1.0f, 0u, 0u,
                                 static_cast<uint8_t*>(out_e4m3), out_scale);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  return ner_launch_status();
}

extern "C" int ner_quantize_weight_e4m3(const float* w_kn, void* wt_nk_e4m3, float* w_scale, int K, int N, ner_stream_t stream) {
  if (K < 1 || N < 1 || !w_kn || !wt_nk_e4m3 || !w_scale) return NER_ERR_INVALID_ARG;
  quantize_weight_e4m3_kernel<<<(N + 31) / 32, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      w_kn, static_cast<uint8_t*>(wt_nk_e4m3), w_scale, K, N);
  return ner_launch_status();
}
