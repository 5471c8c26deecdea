// Stand-alone timing harness for ner_crf_viterbi at the roofline shape (no Python start-up: the whole run is seconds).
//   nvcc -O3 -o vit_harness vit_harness.cu -I../../include -L../../chinesener_b200 -lner_b200 -Xlinker -rpath -Xlinker '$ORIGIN/../../chinesener_b200'
// Prints the kernel plan (NER_VIT_* of ner_b200.h), ms, algorithmic GB/s and a checksum of the tags (equal across builds).
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
#include "ner_b200.h"

__global__ void fill(float* x, size_t n, uint32_t seed) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t h = (uint32_t)i * 2654435761u + seed;
    h ^= h >> 16; h *= 2246822519u; h ^= h >> 13; h *= 3266489917u; h ^= h >> 16;
    x[i] = ((float)(h & 0xFFFFFF) / 8388608.0f - 1.0f) * 3.0f;
  }
}
__global__ void checksum(const int32_t* t, size_t n, unsigned long long* out) {
  unsigned long long acc = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    acc += (unsigned long long)(t[i] + 1) * (unsigned long long)((i % 1000003) + 1);
  atomicAdd(out, acc);
}

int main(int argc, char** argv) {
  const int B = argc > 1 ? atoi(argv[1]) : 262144, L = argc > 2 ? atoi(argv[2]) : 128, K = argc > 3 ? atoi(argv[3]) : 10;
  const int ragged = argc > 4 ? atoi(argv[4]) : 0;
  float *x, *tr, *best;
  int32_t *lens, *tags;
  unsigned long long* cs;
  const size_t n = (size_t)B * L * K;
  cudaMalloc(&x, n * 4); cudaMalloc(&tr, K * K * 4); cudaMalloc(&best, B * 4); cudaMalloc(&lens, B * 4);
  cudaMalloc(&tags, (size_t)B * L * 4); cudaMalloc(&cs, 8);
  fill<<<1184, 256>>>(x, n, 12345u);
  fill<<<1, 128>>>(tr, K * K, 777u);
  int32_t* hl = (int32_t*)malloc(B * 4);
  for (int i = 0; i < B; ++i) hl[i] = ragged ? 1 + (int)(((uint32_t)i * 2654435761u >> 8) % L) : L;
  cudaMemcpy(lens, hl, B * 4, cudaMemcpyHostToDevice);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int w = 0; w < 3; ++w) {
    int rc = ner_crf_viterbi(x, lens, tr, tags, best, B, L, K, nullptr);
    if (rc) { printf("rc=%d %s\n", rc, ner_strerror(rc)); return 1; }
  }
  float best_ms = 1e9f, sum = 0;
  const int R = 20;
  for (int r = 0; r < R; ++r) {
    cudaEventRecord(e0);
    ner_crf_viterbi(x, lens, tr, tags, best, B, L, K, nullptr);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    sum += ms; if (ms < best_ms) best_ms = ms;
  }
  cudaMemset(cs, 0, 8);
  checksum<<<1184, 256>>>(tags, (size_t)B * L, cs);
  unsigned long long h; cudaMemcpy(&h, cs, 8, cudaMemcpyDeviceToHost);
  const double bytes = (double)B * L * 4 * K + 4.0 * B + 4.0 * K * K + (double)B * L * 4 + 4.0 * B;
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  printf("plan=%d B=%d L=%d K=%d ragged=%d  mean %.4f ms  best %.4f ms  %.0f GB/s  checksum %llu  %s\n",
         ner_crf_viterbi_plan(B, L, K, ((uintptr_t)x & 15) == 0, prop.multiProcessorCount),
         B, L, K, ragged, sum / R, best_ms, bytes / (sum / R) / 1e6, h, cudaGetErrorString(cudaGetLastError()));
  return 0;
}
