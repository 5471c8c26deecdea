// Shared device/host helpers for the ner_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include "../../include/ner_b200.h"

#define NER_MAX_TAGS 32

// SMs of the current device (132 on an H100 SXM, 114 on an H100 PCIe): grid caps, small-batch / big-batch thresholds and
// the scratch sized by them are in units of it.  Queried once per device ordinal.
static inline int ner_num_sms() {
  static int cache[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
    (void)cudaGetLastError();
    return 132;
  }
  if (cache[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
      (void)cudaGetLastError();
      n = 132;
    }
    cache[dev] = n;
  }
  return cache[dev];
}

// Map the last CUDA launch error onto the C-ABI status space.
static inline int ner_launch_status() {
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) return NER_OK;
  return NER_ERR_CUDA_BASE - (int)e;
}

// Launch with programmatic dependent launch (PDL): the grid may be scheduled while the previous
// kernel of the stream is still draining, runs its prologue, and blocks in pdl_wait() until that
// kernel has completed and flushed.  Kernels launched this way call pdl_launch_dependents() at
// entry and pdl_wait() before their first global-memory access.
template <typename... KArgs, typename... Args>
static inline cudaError_t ner_launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                         Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

namespace nerdev {

__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(smem_u32(smem)), "l"(gmem));
}
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(smem_u32(smem)), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_lg2(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// fp32 pairs.  Hopper has no packed fp32 instructions, so each pair op is two scalar ops with the same
// rounding (fma.rn / mul.rn / add.rn per lane); the kernels keep the pair form for their data layout.
struct f32x2 {
  float lo, hi;
};
__device__ __forceinline__ f32x2 pk2(float lo, float hi) { return f32x2{lo, hi}; }
__device__ __forceinline__ void upk2(f32x2 v, float& lo, float& hi) {
  lo = v.lo;
  hi = v.hi;
}
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) {
  return f32x2{__fmaf_rn(a.lo, b.lo, c.lo), __fmaf_rn(a.hi, b.hi, c.hi)};
}
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) { return f32x2{__fmul_rn(a.lo, b.lo), __fmul_rn(a.hi, b.hi)}; }
__device__ __forceinline__ f32x2 add2(f32x2 a, f32x2 b) { return f32x2{__fadd_rn(a.lo, b.lo), __fadd_rn(a.hi, b.hi)}; }
__device__ __forceinline__ float max3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Counter-based keep decision shared by every dropout site (forward and backward regenerate it).
__device__ __forceinline__ uint32_t hash3(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t x = a * 0x9E3779B1u ^ (b + 0x7F4A7C15u) * 0x85EBCA77u ^ (c + 0x165667B1u) * 0xC2B2AE3Du;
  x ^= x >> 16;
  x *= 0x7FEB352Du;
  x ^= x >> 15;
  x *= 0x846CA68Bu;
  x ^= x >> 16;
  return x;
}
__device__ __forceinline__ uint32_t keep_threshold(float keep) {
  return (uint32_t)fminf(keep * 4294967296.f, 4294967295.f);
}

// OCP e4m3 ("fn", max 448) block scaling of the FP8 encoder: scale = amax / 448 in fp32, 1 when amax == 0;
// q = e4m3(x / scale), round to nearest even, saturating.
constexpr float kE4m3Max = 448.f;
__device__ __forceinline__ float e4m3_scale(float amax) { return amax > 0.f ? __fdiv_rn(amax, kE4m3Max) : 1.f; }
// two floats -> packed e4m3 pair: `lo` in the low byte (the lower address)
__device__ __forceinline__ uint16_t cvt_e4m3x2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}

}  // namespace nerdev
