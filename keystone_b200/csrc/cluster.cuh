// Thread-block cluster primitives (sm_90): the CTA's rank in its cluster, the cluster-wide barrier and distributed shared
// memory addresses.  Shared by the clustered Cholesky solve (solve_kernels.cu) and the CTA pairs of the split-operand tensor-core
// kernels (tc_kernels.cu).
#pragma once
#include <stdint.h>

namespace ks {

__device__ __forceinline__ uint32_t cl_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cl_nctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
  return r;
}
// every thread of every CTA of the cluster; orders the memory operations before it (release) against those after it (acquire)
__device__ __forceinline__ void cl_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of the variable at shared::cta address `local_addr` in the CTA of rank `rank`
__device__ __forceinline__ uint32_t cl_map_shared(uint32_t local_addr, uint32_t rank) {
  uint32_t ra;
  asm("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local_addr), "r"(rank));
  return ra;
}

}  // namespace ks
