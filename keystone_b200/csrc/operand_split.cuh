// Element-wise formats of the MMA operands that the packing kernels write (aux_kernels.cu, lbfgs.cu): one definition of each, so
// the kernels that produce the same operand cannot drift apart.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace ks {

// fp32 -> tf32 with round-to-nearest (ties away), kept in fp32 (the MMA itself would truncate)
__device__ __forceinline__ float round_tf32_rna(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
// tf32 pair of v: hi = tf32(v), lo = tf32(v - hi) (the rounding error, itself exact in fp32); hi + lo carries 21+ bits of v
__device__ __forceinline__ void tf32_pair(float v, float& hi, float& lo) {
  hi = round_tf32_rna(v);
  lo = round_tf32_rna(v - hi);
}
// fp16 pairs of two adjacent values o0, o1 (already scaled into fp16's range), packed two per 32-bit word as the operand rows store
// them: hi = fp16(o) (f16_hi2), lo = fp16(o - hi) (f16_lo2, from the hi word)
__device__ __forceinline__ __half2 f16_hi2(float o0, float o1) { return __floats2half2_rn(o0, o1); }
__device__ __forceinline__ __half2 f16_lo2(float o0, float o1, __half2 hi) {
  const float2 f = __half22float2(hi);
  return __floats2half2_rn(o0 - f.x, o1 - f.y);
}

}  // namespace ks
