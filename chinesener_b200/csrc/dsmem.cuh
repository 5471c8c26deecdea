// Distributed-shared-memory signalling of the persistent recurrence kernels (bilstm.cu, bigru.cu, bigru_bwd.cu).
//
// A value is published to a peer CTA of the cluster with a remote 4-byte store that completes transaction bytes on the
// DESTINATION CTA's mbarrier (st.async), so a publish needs no fence over the thread's earlier global stores and the
// wait no L1 invalidate (barrier.cluster costs both every step).
#pragma once
#include <stdint.h>

#include "common.cuh"

static __device__ __forceinline__ uint32_t mapa_u32(uint32_t local_smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(rank));
  return r;
}
static __device__ __forceinline__ void st_async_f32(uint32_t remote_addr, float v, uint32_t remote_bar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(remote_addr),
               "r"(__float_as_uint(v)), "r"(remote_bar)
               : "memory");
}
static __device__ __forceinline__ void mbar_init_(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(nerdev::smem_u32(bar)), "r"(count) : "memory");
}
static __device__ __forceinline__ void mbar_arrive_expect_tx_(uint64_t* bar, uint32_t tx_bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(nerdev::smem_u32(bar)), "r"(tx_bytes) : "memory");
}
static __device__ __forceinline__ void mbar_wait_(uint64_t* bar, uint32_t parity) {
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
static __device__ __forceinline__ void publish_all(uint32_t la, uint32_t lb, float v, int C) {
  for (int dst = 0; dst < C; ++dst) st_async_f32(mapa_u32(la, (uint32_t)dst), v, mapa_u32(lb, (uint32_t)dst));
}
