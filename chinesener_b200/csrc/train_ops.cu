// Training-side HBM-bound kernels (sm_90a): operand transposes for the weight-gradient GEMMs,
// bias gradients, label-projection backward, dropout, and the two optimizer steps of the reference
// (tools/train_utils.py:246-390): AdamWeightDecayOptimizer (no bias correction, decoupled weight
// decay, global-norm clipping) and tf.train.AdamOptimizer (bias-corrected, clip-by-value).
#include "common.cuh"

namespace {

using namespace nerdev;

// src f32 [M,N] (row stride ld) -> dst bf16 [N, Mp] (Mp >= M, zero padded): the K-major operand of a
// weight-gradient GEMM  dW[K,N] = X^T dY  (reduction over the M rows).
__global__ void __launch_bounds__(256)
transpose_cast_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int M, int N, int Mp, int ld) {
  __shared__ float tile[32][33];
  const int m0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8) {
    const int m = m0 + i, n = n0 + tx;
    tile[i][tx] = (m < M && n < N) ? src[(size_t)m * ld + n] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int n = n0 + i, m = m0 + tx;
    if (n < N && m < Mp) dst[(size_t)n * Mp + m] = __float2bfloat16_rn(tile[tx][i]);
  }
}

// out[n] (+)= scale * sum_m x[m, n]   (bias gradients)
__global__ void __launch_bounds__(256)
colsum_kernel(const float* __restrict__ x, float* __restrict__ out, int M, int N, int ld, float scale) {
  const int n = blockIdx.x * 32 + (threadIdx.x & 31);
  const int ty = threadIdx.x >> 5;
  __shared__ float part[8][33];
  float acc = 0.f;
  if (n < N)
    for (int m = blockIdx.y * 8 + ty; m < M; m += gridDim.y * 8) acc += x[(size_t)m * ld + n];
  part[ty][threadIdx.x & 31] = acc;
  __syncthreads();
  if (ty == 0 && n < N) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += part[i][threadIdx.x & 31];
    atomicAdd(out + n, scale * s);
  }
}

// label projection backward:  dW[F,N] += x^T dy,  db[N] += colsum(dy),  dx[M,F] = dy W^T   (N <= 32)
template <int NMAX>
__global__ void __launch_bounds__(256)
dense_small_n_bwd_kernel(const float* __restrict__ x, const float* __restrict__ W, const float* __restrict__ dy,
                         float* __restrict__ dW, float* __restrict__ db, float* __restrict__ dx, int M, int F, int N) {
  extern __shared__ float sm[];
  float* s_w = sm;            // [F][N]
  float* s_dw = sm + F * N;   // [F][N] CTA partial
  for (int e = threadIdx.x; e < F * N; e += blockDim.x) {
    s_w[e] = W[e];
    s_dw[e] = 0.f;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float dbacc = 0.f;  // lane n accumulates db[n]
  for (int row = blockIdx.x * nw + warp; row < M; row += gridDim.x * nw) {
    float g[NMAX];
#pragma unroll
    for (int n = 0; n < NMAX; ++n) g[n] = (n < N) ? dy[(size_t)row * N + n] : 0.f;
    if (lane < N) dbacc += dy[(size_t)row * N + lane];
    for (int f = lane; f < F; f += 32) {
      const float xv = x[(size_t)row * F + f];
      float d = 0.f;
#pragma unroll
      for (int n = 0; n < NMAX; ++n)
        if (n < N) {
          d = fmaf(g[n], s_w[f * N + n], d);
          atomicAdd(&s_dw[f * N + n], xv * g[n]);
        }
      if (dx != nullptr) dx[(size_t)row * F + f] = d;
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < F * N; e += blockDim.x) {
    const float v = s_dw[e];
    if (v != 0.f) atomicAdd(dW + e, v);
  }
  if (db != nullptr && lane < N && dbacc != 0.f) atomicAdd(db + lane, dbacc);
}

// Counter-based dropout (Philox-like integer hash of (seed, element index)): the same (seed, i)
// gives the same keep decision in forward and backward, so no mask tensor is stored.
__global__ void __launch_bounds__(256)
dropout_kernel(const float* __restrict__ x, float* __restrict__ y, size_t n, float keep, uint32_t seed_lo, uint32_t seed_hi) {
  const float inv = 1.f / keep;
  const uint32_t thr = keep_threshold(keep);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t r = hash3(seed_lo, seed_hi ^ (uint32_t)(i >> 32), (uint32_t)i);
    y[i] = (r < thr) ? x[i] * inv : 0.f;
  }
}

__global__ void __launch_bounds__(256)
dropout_bf16_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, size_t n, float keep, uint32_t seed_lo,
                    uint32_t seed_hi) {
  const float inv = 1.f / keep;
  const uint32_t thr = keep_threshold(keep);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t r = hash3(seed_lo, seed_hi ^ (uint32_t)(i >> 32), (uint32_t)i);
    y[i] = (r < thr) ? __float2bfloat16(__bfloat162float(x[i]) * inv) : __float2bfloat16(0.f);
  }
}

// sum of squares of a flat buffer, for clip_by_global_norm.  Deterministic: every CTA writes its partial sum (fixed
// element -> thread map, fixed shuffle order) to partials[blockIdx.x]; the second kernel adds them in index order.  (An atomicAdd
// per CTA made the norm — and through the clip factor every weight — depend on CTA arrival order: data-parallel replicas that
// start identical drifted apart by an ulp per step.)
__global__ void __launch_bounds__(256)
sumsq_partial_kernel(const float* __restrict__ g, size_t n, float* __restrict__ partials) {
  float acc = 0.f;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t n4 = (reinterpret_cast<uintptr_t>(g) & 15) == 0 ? n / 4 : 0;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 x = g4[i];
    acc = fmaf(x.x, x.x, acc);
    acc = fmaf(x.y, x.y, acc);
    acc = fmaf(x.z, x.z, acc);
    acc = fmaf(x.w, x.w, acc);
  }
  for (size_t i = 4 * n4 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) acc = fmaf(g[i], g[i], acc);
  acc = warp_sum(acc);
  __shared__ float part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < 8; ++i) s += part[i];
    partials[blockIdx.x] = s;
  }
}
__global__ void __launch_bounds__(256)
sumsq_final_kernel(const float* __restrict__ partials, int n, float* __restrict__ out) {
  __shared__ double part[256];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) acc += (double)partials[i];
  part[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) part[threadIdx.x] += part[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] += (float)part[0];
}

// mode 0: AdamWeightDecayOptimizer (bert optimization.py): m,v update, upd = m/(sqrt(v)+eps) (+ wd*p), p -= lr*upd.
//         gradient pre-scaled by clip = clip_norm / max(global_norm, clip_norm) read from gnorm_sq.
// mode 1: tf.train.AdamOptimizer: g clipped to [-clip_value, clip_value], bias-corrected step size `lr`
//         (caller passes lr_t = lr*sqrt(1-b2^t)/(1-b1^t)), p -= lr_t * m / (sqrt(v) + eps).
__global__ void __launch_bounds__(256)
adam_step_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                 size_t n, float lr, float b1, float b2, float eps, float wd, int mode, float clip,
                 const float* __restrict__ gnorm_sq, float grad_scale) {
  float gs = grad_scale;
  if (mode == 0 && gnorm_sq != nullptr && clip > 0.f) {
    const float gn = sqrtf(*gnorm_sq) * grad_scale;
    gs *= clip / fmaxf(gn, clip);
  }
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  auto one = [&](float& pi, float gin, float& mi_io, float& vi_io) {
    float gi = gin * gs;
    if (mode == 1 && clip > 0.f) gi = fminf(fmaxf(gi, -clip), clip);
    const float mi = b1 * mi_io + (1.f - b1) * gi;
    const float vi = b2 * vi_io + (1.f - b2) * gi * gi;
    mi_io = mi;
    vi_io = vi;
    float upd = mi / (sqrtf(vi) + eps);
    if (mode == 0) upd += wd * pi;
    pi -= lr * upd;
  };
  // 16-byte accesses when the four buffers allow it (the flat optimizer state: 256-byte aligned ranges): 28 B per parameter
  // of HBM traffic is the whole cost of this kernel
  const bool vec = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                     reinterpret_cast<uintptr_t>(v)) & 15) == 0;
  const size_t n4 = vec ? n / 4 : 0;
  float4* p4 = reinterpret_cast<float4*>(p);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  float4* m4 = reinterpret_cast<float4*>(m);
  float4* v4 = reinterpret_cast<float4*>(v);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 pp = p4[i], mm = m4[i], vv = v4[i];
    const float4 gg = g4[i];
    one(pp.x, gg.x, mm.x, vv.x);
    one(pp.y, gg.y, mm.y, vv.y);
    one(pp.z, gg.z, mm.z, vv.z);
    one(pp.w, gg.w, mm.w, vv.w);
    p4[i] = pp;
    m4[i] = mm;
    v4[i] = vv;
  }
  for (size_t i = 4 * n4 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) one(p[i], g[i], m[i], v[i]);
}



// tf.reduce_max(x[B,L,C], axis=1) -> y[B,C]: one thread per (b, c), a warp reads 32 consecutive c per step
__global__ void __launch_bounds__(256)
reduce_max_time_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int L, int C) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * C) return;
  const int b = i / C, c = i - b * C;
  const float* p = x + (size_t)b * L * C + c;
  float m = p[0];
  for (int t = 1; t < L; ++t) m = fmaxf(m, p[(size_t)t * C]);
  y[i] = m;
}

// its gradient as TF defines it (math_grad._MinOrMaxGrad): every position that equals the max gets dy / #ties.
// dx[b,t,c] += scale * dy[b,c] / ties   (scale folds the gradient flip of the adversarial plugin)
__global__ void __launch_bounds__(256)
reduce_max_time_bwd_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dy,
                           float* __restrict__ dx, int B, int L, int C, float scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * C) return;
  const int b = i / C, c = i - b * C;
  const float* p = x + (size_t)b * L * C + c;
  float* q = dx + (size_t)b * L * C + c;
  const float m = y[i];
  int ties = 0;
  for (int t = 0; t < L; ++t) ties += (p[(size_t)t * C] == m);
  const float g = scale * dy[i] / (float)ties;
  for (int t = 0; t < L; ++t)
    if (p[(size_t)t * C] == m) q[(size_t)t * C] += g;
}

// tf.nn.sparse_softmax_cross_entropy_with_logits on [B, N<=32] rows: loss[b] = logsumexp(z_b) - z_b[label_b];
// dz (optional) = scale * (softmax(z_b) - onehot(label_b))
__global__ void __launch_bounds__(128)
softmax_xent_kernel(const float* __restrict__ z, const int* __restrict__ labels, float* __restrict__ loss,
                    float* __restrict__ dz, int B, int N, float scale) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float* r = z + (size_t)b * N;
  float m = r[0];
  for (int n = 1; n < N; ++n) m = fmaxf(m, r[n]);
  float s = 0.f;
  for (int n = 0; n < N; ++n) s += expf(r[n] - m);
  const int lab = labels[b];
  loss[b] = (m + logf(s)) - r[lab];
  if (dz != nullptr) {
    const float inv = 1.f / s;
    for (int n = 0; n < N; ++n) dz[(size_t)b * N + n] = scale * (expf(r[n] - m) * inv - (n == lab ? 1.f : 0.f));
  }
}

// Row moves between the padded [B*L, .] and the packed [n, .] layouts (rows are multiples of 16 bytes):
// gather: dst row r = src row idx[r];  scatter: dst row idx[r] = src row r.
template <bool SCATTER>
__global__ void __launch_bounds__(256)
move_rows_kernel(const uint4* __restrict__ src, const int32_t* __restrict__ idx, uint4* __restrict__ dst, int n, int vpr) {
  const size_t total = (size_t)n * vpr, stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const size_t r = i / vpr, c = i - r * vpr;
    const size_t j = (size_t)idx[r] * vpr + c;
    if (SCATTER) dst[j] = src[i];
    else dst[i] = src[j];
  }
}

int flat_grid(size_t n) {
  size_t g = (n + 255) / 256;
  if (g > ner_num_sms() * 16) g = ner_num_sms() * 16;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace

extern "C" int ner_transpose_cast_bf16(const float* src, void* dst_bf16, int M, int N, int Mp, int ld_src,
                                       ner_stream_t stream) {
  if (M < 1 || N < 1 || Mp < M || ld_src < N || !src || !dst_bf16) return NER_ERR_INVALID_ARG;
  dim3 grid((N + 31) / 32, (Mp + 31) / 32);
  transpose_cast_bf16_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      src, static_cast<__nv_bfloat16*>(dst_bf16), M, N, Mp, ld_src);
  return ner_launch_status();
}

extern "C" int ner_colsum_add(const float* x, float* out, int M, int N, int ld, float scale, ner_stream_t stream) {
  if (M < 0 || N < 1 || ld < N || !x || !out) return NER_ERR_INVALID_ARG;
  if (M == 0) return NER_OK;
  dim3 grid((N + 31) / 32, M >= 4096 ? 32 : (M >= 256 ? 8 : 1));
  colsum_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, out, M, N, ld, scale);
  return ner_launch_status();
}

extern "C" int ner_dense_small_n_bwd(const float* x, const float* W, const float* dy, float* dW, float* db, float* dx,
                                     int M, int F, int N, ner_stream_t stream) {
  if (M < 0 || F < 1 || N < 1) return NER_ERR_INVALID_ARG;
  if (M == 0) return NER_OK;
  if (!x || !W || !dy || !dW) return NER_ERR_INVALID_ARG;
  if (N > 32 || (size_t)2 * F * N * 4 > 200 * 1024) return NER_ERR_UNSUPPORTED;
  const size_t smem = (size_t)2 * F * N * 4;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  long g = ((long)M + 63) / 64;
  if (g > ner_num_sms() * 2) g = ner_num_sms() * 2;
  cudaError_t e;
  if (N <= 16) {
    auto kern = dense_small_n_bwd_kernel<16>;
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
    kern<<<(int)g, 256, smem, st>>>(x, W, dy, dW, db, dx, M, F, N);
  } else {
    auto kern = dense_small_n_bwd_kernel<32>;
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
    kern<<<(int)g, 256, smem, st>>>(x, W, dy, dW, db, dx, M, F, N);
  }
  return ner_launch_status();
}

__global__ void __launch_bounds__(256) axpy_kernel(float* __restrict__ dst, const float* __restrict__ src, size_t n, float a) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dst[i] = fmaf(a, src[i], dst[i]);
}

// d_pre = d_act where act > 0 else 0   (tf.nn.relu gradient, all f32)
__global__ void __launch_bounds__(256)
relu_bwd_kernel(const float* __restrict__ act, const float* __restrict__ dact, float* __restrict__ dpre, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dpre[i] = act[i] > 0.f ? dact[i] : 0.f;
}

__global__ void __launch_bounds__(256) relu_kernel(const float* __restrict__ x, float* __restrict__ y, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) y[i] = fmaxf(x[i], 0.f);
}

extern "C" int ner_relu_f32(const float* x, float* y, size_t n, ner_stream_t stream) {
  if (!x || !y) return n == 0 ? NER_OK : NER_ERR_INVALID_ARG;
  if (n == 0) return NER_OK;
  relu_kernel<<<flat_grid(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, y, n);
  return ner_launch_status();
}

extern "C" int ner_relu_bwd_f32(const float* act, const float* dact, float* dpre, size_t n, ner_stream_t stream) {
  if (!act || !dact || !dpre) return n == 0 ? NER_OK : NER_ERR_INVALID_ARG;
  if (n == 0) return NER_OK;
  relu_bwd_kernel<<<flat_grid(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(act, dact, dpre, n);
  return ner_launch_status();
}

extern "C" int ner_axpy_f32(float* dst, const float* src, size_t n, float a, ner_stream_t stream) {
  if (!dst || !src) return n == 0 ? NER_OK : NER_ERR_INVALID_ARG;
  if (n == 0) return NER_OK;
  axpy_kernel<<<flat_grid(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(dst, src, n, a);
  return ner_launch_status();
}

extern "C" int ner_dropout_bf16(const void* x, void* y, size_t n, float keep_prob, uint64_t seed, ner_stream_t stream) {
  if (!x || !y) return n == 0 ? NER_OK : NER_ERR_INVALID_ARG;
  if (!(keep_prob > 0.f) || keep_prob > 1.f) return NER_ERR_INVALID_ARG;
  if (n == 0) return NER_OK;
  dropout_bf16_kernel<<<flat_grid(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), n, keep_prob, (uint32_t)seed, (uint32_t)(seed >> 32));
  return ner_launch_status();
}

extern "C" int ner_dropout(const float* x, float* y, size_t n, float keep_prob, uint64_t seed, ner_stream_t stream) {
  if (!x || !y) return n == 0 ? NER_OK : NER_ERR_INVALID_ARG;
  if (!(keep_prob > 0.f) || keep_prob > 1.f) return NER_ERR_INVALID_ARG;
  if (n == 0) return NER_OK;
  dropout_kernel<<<flat_grid(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, y, n, keep_prob, (uint32_t)seed,
                                                                             (uint32_t)(seed >> 32));
  return ner_launch_status();
}

extern "C" size_t ner_sumsq_scratch_floats(void) { return (size_t)ner_num_sms() * 16; }

extern "C" int ner_sumsq_add(const float* g, size_t n, float* out, float* scratch, ner_stream_t stream) {
  if (!g || !out || !scratch) return n == 0 ? NER_OK : NER_ERR_INVALID_ARG;
  if (n == 0) return NER_OK;
  const int grid = flat_grid(n);
  sumsq_partial_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(g, n, scratch);
  sumsq_final_kernel<<<1, 256, 0, static_cast<cudaStream_t>(stream)>>>(scratch, grid, out);
  return ner_launch_status();
}

extern "C" int ner_adam_step(float* p, const float* g, float* m, float* v, size_t n, float lr, float beta1,
                             float beta2, float eps, float weight_decay, int mode, float clip,
                             const float* gnorm_sq, float grad_scale, ner_stream_t stream) {
  if (!p || !g || !m || !v) return n == 0 ? NER_OK : NER_ERR_INVALID_ARG;
  if (mode != 0 && mode != 1) return NER_ERR_INVALID_ARG;
  if (n == 0) return NER_OK;
  adam_step_kernel<<<flat_grid(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(p, g, m, v, n, lr, beta1, beta2, eps,
                                                                               weight_decay, mode, clip, gnorm_sq,
                                                                               grad_scale);
  return ner_launch_status();
}

extern "C" int ner_reduce_max_time(const float* x, float* y, int B, int L, int C, ner_stream_t stream) {
  if (B < 0 || L < 1 || C < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!x || !y) return NER_ERR_INVALID_ARG;
  reduce_max_time_kernel<<<(B * C + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, y, B, L, C);
  return ner_launch_status();
}

extern "C" int ner_reduce_max_time_bwd(const float* x, const float* y, const float* dy, float* dx, int B, int L, int C,
                                       float scale, ner_stream_t stream) {
  if (B < 0 || L < 1 || C < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!x || !y || !dy || !dx) return NER_ERR_INVALID_ARG;
  reduce_max_time_bwd_kernel<<<(B * C + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, y, dy, dx, B, L, C, scale);
  return ner_launch_status();
}

extern "C" int ner_softmax_xent(const float* logits, const int32_t* labels, float* loss, float* dlogits, int B, int N,
                                float scale, ner_stream_t stream) {
  if (B < 0 || N < 1) return NER_ERR_INVALID_ARG;
  if (N > 32) return NER_ERR_UNSUPPORTED;
  if (B == 0) return NER_OK;
  if (!logits || !labels || !loss) return NER_ERR_INVALID_ARG;
  softmax_xent_kernel<<<(B + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(logits, labels, loss, dlogits, B, N, scale);
  return ner_launch_status();
}

extern "C" int ner_gather_rows(const void* src, const int32_t* idx, void* dst, int n, int row_bytes, ner_stream_t stream) {
  if (n < 0 || row_bytes < 16 || row_bytes % 16 != 0) return NER_ERR_INVALID_ARG;
  if (n == 0) return NER_OK;
  if (!src || !idx || !dst) return NER_ERR_INVALID_ARG;
  const int vpr = row_bytes / 16;
  move_rows_kernel<false><<<flat_grid((size_t)n * vpr), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(src), idx, static_cast<uint4*>(dst), n, vpr);
  return ner_launch_status();
}

extern "C" int ner_scatter_rows(const void* src, const int32_t* idx, void* dst, int n, int row_bytes, ner_stream_t stream) {
  if (n < 0 || row_bytes < 16 || row_bytes % 16 != 0) return NER_ERR_INVALID_ARG;
  if (n == 0) return NER_OK;
  if (!src || !idx || !dst) return NER_ERR_INVALID_ARG;
  const int vpr = row_bytes / 16;
  move_rows_kernel<true><<<flat_grid((size_t)n * vpr), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(src), idx, static_cast<uint4*>(dst), n, vpr);
  return ner_launch_status();
}
