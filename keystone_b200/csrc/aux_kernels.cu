// HBM-bound helper kernels of the block least-squares path: conversions, column sums
// (StandardScaler, K/nodes/stats/StandardScaler.scala:45-59; MatrixUtils.computeMean,
// K/utils/MatrixUtils.scala:137-146), residual initialisation, the fp64 assembly of the reduced
// normal equations and operand packing.  All matrices are row-major fp32 with ld % 32 == 0
// unless stated; fp64 matrices are column-major exactly as Breeze stores DenseMatrix[Double].
#include <cuda_fp16.h>

#include "kernels.h"
#include "operand_split.cuh"

namespace ks {

static inline unsigned grid_for(int64_t n, int threads, int64_t cap = 132 * 16) {
  int64_t g = (n + threads - 1) / threads;
  if (g < 1) g = 1;
  if (g > cap) g = cap;
  return static_cast<unsigned>(g);
}

// ------------------------------------------------------------------ conversions
__global__ void f64_to_f32_rows_kernel(const double* __restrict__ src, int64_t src_ld, float* __restrict__ dst,
                                       int64_t dst_ld, int64_t rows, int64_t cols) {
  const int64_t total = rows * dst_ld;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / dst_ld, c = i - r * dst_ld;
    dst[i] = c < cols ? static_cast<float>(src[r * src_ld + c]) : 0.f;
  }
}
void launch_f64_to_f32_rows(const double* src, int64_t src_ld, float* dst, int64_t dst_ld, int64_t rows, int64_t cols,
                            cudaStream_t st) {
  if (rows * dst_ld == 0) return;
  f64_to_f32_rows_kernel<<<grid_for(rows * dst_ld, 256), 256, 0, st>>>(src, src_ld, dst, dst_ld, rows, cols);
}

// dense host-order rows -> pitched matrix rows, padding columns zeroed (the upload path stages contiguous H2D copies: a 1-D copy
// runs at the link rate, a pitched 2-D copy of 1760-byte rows at a third of it)
__global__ void f32_repitch_rows_kernel(const float* __restrict__ src, int64_t src_ld, float* __restrict__ dst, int64_t dst_ld,
                                        int64_t rows, int64_t cols) {
  const int64_t total = rows * dst_ld;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / dst_ld, c = i - r * dst_ld;
    dst[i] = c < cols ? src[r * src_ld + c] : 0.f;
  }
}
void launch_f32_repitch_rows(const float* src, int64_t src_ld, float* dst, int64_t dst_ld, int64_t rows, int64_t cols,
                             cudaStream_t st) {
  if (rows * dst_ld == 0) return;
  f32_repitch_rows_kernel<<<grid_for(rows * dst_ld, 256), 256, 0, st>>>(src, src_ld, dst, dst_ld, rows, cols);
}

__global__ void f32_to_f64_rows_kernel(const float* __restrict__ src, int64_t src_ld, double* __restrict__ dst,
                                       int64_t dst_ld, int64_t rows, int64_t cols) {
  const int64_t total = rows * cols;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / cols, c = i - r * cols;
    dst[r * dst_ld + c] = static_cast<double>(src[r * src_ld + c]);
  }
}
void launch_f32_to_f64_rows(const float* src, int64_t src_ld, double* dst, int64_t dst_ld, int64_t rows, int64_t cols,
                            cudaStream_t st) {
  if (rows * cols == 0) return;
  f32_to_f64_rows_kernel<<<grid_for(rows * cols, 256), 256, 0, st>>>(src, src_ld, dst, dst_ld, rows, cols);
}

__global__ void f64_to_f32_vec_kernel(const double* __restrict__ src, float* __restrict__ dst, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    dst[i] = static_cast<float>(src[i]);
}
void launch_f64_to_f32_vec(const double* src, float* dst, int64_t n, cudaStream_t st) {
  if (n == 0) return;
  f64_to_f32_vec_kernel<<<grid_for(n, 256), 256, 0, st>>>(src, dst, n);
}

// ClassLabelIndicatorsFromIntLabels (K/nodes/util/ClassLabelIndicators.scala:15-29): +1 at the class, -1 elsewhere
__global__ void labels_from_classes_kernel(const int32_t* __restrict__ cls, float* __restrict__ dst, int64_t ld,
                                           int64_t rows, int k) {
  const int64_t total = rows * ld;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / ld;
    const int c = static_cast<int>(i - r * ld);
    dst[i] = c < k ? (c == cls[r] ? 1.f : -1.f) : 0.f;
  }
}
void launch_labels_from_classes(const int32_t* cls, float* dst, int64_t ld, int64_t rows, int k, cudaStream_t st) {
  if (rows == 0) return;
  labels_from_classes_kernel<<<grid_for(rows * ld, 256), 256, 0, st>>>(cls, dst, ld, rows, k);
}

__global__ void fill_kernel(float* p, int64_t n, float v) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    p[i] = v;
}
void launch_fill_f32(float* p, int64_t n, float v, cudaStream_t st) {
  if (n == 0) return;
  fill_kernel<<<grid_for(n, 256), 256, 0, st>>>(p, n, v);
}

// ------------------------------------------------------------------ synthetic N(mean, std) (benchmarks)
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__global__ void normal_kernel(float* __restrict__ dst, int64_t ld, int64_t rows, int cols, uint64_t seed,
                              int64_t row_offset, float mean, float stddev) {
  const int64_t total = rows * ld;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / ld;
    const int c = static_cast<int>(i - r * ld);
    float v = 0.f;
    if (c < cols) {
      const uint64_t h = splitmix64(seed ^ splitmix64(static_cast<uint64_t>((row_offset + r) * cols + c)));
      const float u1 = (static_cast<float>(h >> 40) + 0.5f) * (1.0f / 16777216.0f);
      const float u2 = (static_cast<float>((h >> 16) & 0xFFFFFF) + 0.5f) * (1.0f / 16777216.0f);
      v = mean + stddev * sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
    }
    dst[i] = v;
  }
}
void launch_normal_f32(float* dst, int64_t ld, int64_t rows, int cols, uint64_t seed, int64_t row_offset, float mean,
                       float stddev, cudaStream_t st) {
  if (rows == 0) return;
  normal_kernel<<<grid_for(rows * ld, 256), 256, 0, st>>>(dst, ld, rows, cols, seed, row_offset, mean, stddev);
}

// ------------------------------------------------------------------ column sums
// block (32, 8): each thread owns 4 consecutive columns (float4), rows strided by 8; one fp64 atomic per column
// per block.  Coalesced 512 B per warp-row.
__global__ void colsum_kernel(const float* __restrict__ hi, const float* __restrict__ lo, int64_t ld, int64_t rows,
                              int cols, double* __restrict__ sums, int64_t rows_per_block) {
  __shared__ double red[8][128];
  const int c4 = (blockIdx.x * 32 + threadIdx.x) * 4;
  const int64_t r_begin = blockIdx.y * rows_per_block;
  const int64_t r_end = min(rows, r_begin + rows_per_block);
  double a0 = 0, a1 = 0, a2 = 0, a3 = 0;
  if (c4 < ld) {
    for (int64_t r = r_begin + threadIdx.y; r < r_end; r += 8) {
      float4 v = *reinterpret_cast<const float4*>(hi + r * ld + c4);
      if (lo) {
        const float4 w = *reinterpret_cast<const float4*>(lo + r * ld + c4);
        a0 += static_cast<double>(v.x) + w.x; a1 += static_cast<double>(v.y) + w.y;
        a2 += static_cast<double>(v.z) + w.z; a3 += static_cast<double>(v.w) + w.w;
      } else {
        a0 += v.x; a1 += v.y; a2 += v.z; a3 += v.w;
      }
    }
  }
  red[threadIdx.y][threadIdx.x * 4 + 0] = a0;
  red[threadIdx.y][threadIdx.x * 4 + 1] = a1;
  red[threadIdx.y][threadIdx.x * 4 + 2] = a2;
  red[threadIdx.y][threadIdx.x * 4 + 3] = a3;
  __syncthreads();
  const int t = threadIdx.y * 32 + threadIdx.x;
  if (t < 128) {
    double s = 0;
#pragma unroll
    for (int y = 0; y < 8; ++y) s += red[y][t];
    const int c = blockIdx.x * 128 + t;
    if (c < cols) atomicAdd(sums + c, s);
  }
}
void launch_colsum(const float* hi, const float* lo, int64_t ld, int64_t rows, int cols, double* sums, cudaStream_t st) {
  if (rows == 0 || cols == 0) return;
  const int64_t rpb = 1024;
  dim3 grid(static_cast<unsigned>((cols + 127) / 128), static_cast<unsigned>((rows + rpb - 1) / rpb));
  colsum_kernel<<<grid, dim3(32, 8), 0, st>>>(hi, lo, ld, rows, cols, sums, rpb);
}

// ------------------------------------------------------------------ residual init / slab from materialised features
__global__ void init_residual_kernel(const float* __restrict__ Y, int64_t ldy, const double* __restrict__ ymean,
                                     float* __restrict__ R, int64_t ldr, int64_t rows, int k) {
  const int64_t total = rows * ldr;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / ldr;
    const int c = static_cast<int>(i - r * ldr);
    R[i] = c < k ? static_cast<float>(static_cast<double>(Y[r * ldy + c]) - ymean[c]) : 0.f;
  }
}
void launch_init_residual(const float* Y, int64_t ldy, const double* ymean, float* R, int64_t ldr, int64_t rows, int k,
                          cudaStream_t st) {
  if (rows == 0) return;
  init_residual_kernel<<<grid_for(rows * ldr, 256), 256, 0, st>>>(Y, ldy, ymean, R, ldr, rows, k);
}

// block (32, 8), 4 columns per thread: same access pattern as colsum_kernel, plus the rounded copy.
__global__ void round_colsum_kernel(const float* __restrict__ R, float* __restrict__ Rr, int64_t ld, int64_t rows, int k,
                                    double* __restrict__ sums, int64_t rows_per_block, float* __restrict__ Rlo) {
  __shared__ double red[8][128];
  const int c4 = (blockIdx.x * 32 + threadIdx.x) * 4;
  const int64_t r_begin = blockIdx.y * rows_per_block;
  const int64_t r_end = min(rows, r_begin + rows_per_block);
  double a[4] = {0, 0, 0, 0};
  if (c4 < ld) {
    for (int64_t r = r_begin + threadIdx.y; r < r_end; r += 8) {
      const float4 v = *reinterpret_cast<const float4*>(R + r * ld + c4);
      const float in[4] = {v.x, v.y, v.z, v.w};
      float o[4], l[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = c4 + j;
        if (c < k) {
          a[j] += in[j];
          tf32_pair(in[j], o[j], l[j]);  // l: the split-operand mode's lo plane
        } else {
          o[j] = 0.f;
          l[j] = 0.f;
        }
      }
      *reinterpret_cast<float4*>(Rr + r * ld + c4) = make_float4(o[0], o[1], o[2], o[3]);
      if (Rlo) *reinterpret_cast<float4*>(Rlo + r * ld + c4) = make_float4(l[0], l[1], l[2], l[3]);
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) red[threadIdx.y][threadIdx.x * 4 + j] = a[j];
  __syncthreads();
  const int t = threadIdx.y * 32 + threadIdx.x;
  if (t < 128) {
    double s = 0;
#pragma unroll
    for (int y = 0; y < 8; ++y) s += red[y][t];
    const int c = blockIdx.x * 128 + t;
    if (c < k) atomicAdd(sums + c, s);
  }
}
void launch_round_colsum(const float* R, float* Rr, int64_t ld, int64_t rows, int k, double* sums, cudaStream_t st, float* Rlo) {
  if (rows == 0) return;
  const int64_t rpb = 1024;
  dim3 grid(static_cast<unsigned>((ld + 127) / 128), static_cast<unsigned>((rows + rpb - 1) / rpb));
  round_colsum_kernel<<<grid, dim3(32, 8), 0, st>>>(R, Rr, ld, rows, k, sums, rpb, Rlo);
}

// block (32, 8), 4 columns per thread, rows strided by 8 (coalesced 512 B per warp-row); optional column sums
__global__ void center_round_kernel(const float* __restrict__ F, int64_t ldf, int c0, const float* __restrict__ shift,
                                    float* __restrict__ slab, float* __restrict__ colsum, int64_t lds, int64_t rows, int cols,
                                    int64_t rows_per_block, float* __restrict__ slab_lo) {
  __shared__ float red[8][128];
  const int c4 = (blockIdx.x * 32 + threadIdx.x) * 4;
  const int64_t r_begin = blockIdx.y * rows_per_block;
  const int64_t r_end = min(rows, r_begin + rows_per_block);
  float a[4] = {0.f, 0.f, 0.f, 0.f};
  if (c4 < lds) {
    float sh[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) sh[j] = (c4 + j < cols) ? shift[c4 + j] : 0.f;
    for (int64_t r = r_begin + threadIdx.y; r < r_end; r += 8) {
      float o[4], l[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float v = (c4 + j < cols) ? F[r * ldf + c0 + c4 + j] - sh[j] : 0.f;  // c0 may be unaligned: scalar loads
        o[j] = round_tf32_rna(v);
        l[j] = slab_lo ? round_tf32_rna(v - o[j]) : 0.f;  // split-operand mode: hi + lo carries 21 bits of v
        a[j] += o[j] + l[j];
      }
      *reinterpret_cast<float4*>(slab + r * lds + c4) = make_float4(o[0], o[1], o[2], o[3]);
      if (slab_lo) *reinterpret_cast<float4*>(slab_lo + r * lds + c4) = make_float4(l[0], l[1], l[2], l[3]);
    }
  }
  if (colsum == nullptr) return;
#pragma unroll
  for (int j = 0; j < 4; ++j) red[threadIdx.y][threadIdx.x * 4 + j] = a[j];
  __syncthreads();
  const int t = threadIdx.y * 32 + threadIdx.x;
  if (t < 128) {
    float s = 0;
#pragma unroll
    for (int y = 0; y < 8; ++y) s += red[y][t];
    const int c = blockIdx.x * 128 + t;
    if (c < cols) atomicAdd(colsum + c, s);
  }
}
void launch_center_round(const float* F, int64_t ldf, int c0, const float* shift, float* slab, float* colsum, int64_t lds,
                         int64_t rows, int cols, cudaStream_t st, float* slab_lo) {
  if (rows == 0) return;
  const int64_t rpb = 256;
  dim3 grid(static_cast<unsigned>((lds + 127) / 128), static_cast<unsigned>((rows + rpb - 1) / rpb));
  center_round_kernel<<<grid, dim3(32, 8), 0, st>>>(F, ldf, c0, shift, slab, colsum, lds, rows, cols, rpb, slab_lo);
}

__global__ void divide_by_count_kernel(const double* __restrict__ sums, const double* __restrict__ count, float* out,
                                       double* out64, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const double v = sums[i] / fmax(*count, 1.0);
    if (out) out[i] = static_cast<float>(v);
    if (out64) out64[i] = v;
  }
}
void launch_divide_by_count(const double* sums, const double* count, float* out, double* out64, int n, cudaStream_t st) {
  if (n == 0) return;
  divide_by_count_kernel<<<(n + 255) / 256, 256, 0, st>>>(sums, count, out, out64, n);
}

__global__ void delta_mean_kernel(const float* __restrict__ ssum, const float* __restrict__ shift, double n_total,
                                  double* __restrict__ delta, double* __restrict__ mean, int b) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < b) {
    const double d = static_cast<double>(ssum[i]) / n_total;
    delta[i] = d;
    if (mean) mean[i] = static_cast<double>(shift[i]) + d;
  }
}
void launch_delta_mean(const float* ssum, const float* shift, double n_total, double* delta, double* mean, int b, cudaStream_t st) {
  if (b == 0) return;
  delta_mean_kernel<<<(b + 255) / 256, 256, 0, st>>>(ssum, shift, n_total, delta, mean, b);
}

// ------------------------------------------------------------------ exact Gram diagonal of a split slab
// out[c] += sum_r (hi[r][c] + lo[r][c])^2 in fp64 (out must be zeroed).  The tensor core's fp32 accumulation does not round
// every product to nearest: entries whose products all have one sign -- the diagonal of S^T S -- are biased along the
// accumulation chain, zero-mean entries are not (tools/trunc_probe.py measures it).
// The split-operand mode therefore takes the diagonal from this reduction instead of from the tensor core.
template <class T2>
__device__ __forceinline__ float2 pair_to_float2(T2 v);
template <>
__device__ __forceinline__ float2 pair_to_float2<__half2>(__half2 v) { return __half22float2(v); }
template <>
__device__ __forceinline__ float2 pair_to_float2<float2>(float2 v) { return v; }

template <class T2>
__global__ void colsumsq_pair_kernel(const T2* __restrict__ hi, const T2* __restrict__ lo, int64_t ld2, int64_t rows, int cols,
                                     double* __restrict__ out, int64_t rows_per_block) {
  const int c2 = blockIdx.x * blockDim.x + threadIdx.x;  // column pair 2 c2, 2 c2 + 1: coalesced along the row
  if (2 * c2 >= cols) return;
  const int64_t r0 = blockIdx.y * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  double a0 = 0.0, a1 = 0.0;
#pragma unroll 4
  for (int64_t r = r0; r < r1; ++r) {
    const float2 h = pair_to_float2<T2>(hi[r * ld2 + c2]), l = pair_to_float2<T2>(lo[r * ld2 + c2]);
    const double v0 = static_cast<double>(h.x) + static_cast<double>(l.x), v1 = static_cast<double>(h.y) + static_cast<double>(l.y);
    a0 = fma(v0, v0, a0);
    a1 = fma(v1, v1, a1);
  }
  atomicAdd(out + 2 * c2, a0);
  if (2 * c2 + 1 < cols) atomicAdd(out + 2 * c2 + 1, a1);
}
void launch_colsumsq_pair(const void* hi, const void* lo, bool f16, int64_t ld, int64_t rows, int cols, double* out, cudaStream_t st) {
  if (rows == 0 || cols == 0) return;
  const int64_t rpb = 512;
  dim3 grid(static_cast<unsigned>((cols / 2 + 1 + 127) / 128), static_cast<unsigned>((rows + rpb - 1) / rpb));
  if (f16)
    colsumsq_pair_kernel<__half2><<<grid, 128, 0, st>>>(static_cast<const __half2*>(hi), static_cast<const __half2*>(lo), ld / 2, rows,
                                                         cols, out, rpb);
  else
    colsumsq_pair_kernel<float2><<<grid, 128, 0, st>>>(static_cast<const float2*>(hi), static_cast<const float2*>(lo), ld / 2, rows, cols,
                                                        out, rpb);
}

// ------------------------------------------------------------------ reduced system assembly (fp64)
// cross (optional, split-operand mode): full b x b matrix S_hi^T S_lo; the Gram of S = S_hi + S_lo is then
// S_hi^T S_hi + cross + cross^T (the lo x lo term, ~2^-22 of the diagonal, is dropped)
__global__ void build_system_kernel(const float* __restrict__ G, int ldg, const double* __restrict__ delta, double n_total,
                                    double lam, double* __restrict__ H, int b, const float* __restrict__ cross,
                                    const double* __restrict__ exact_diag) {
  const int64_t total = static_cast<int64_t>(b) * b;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i / b), r = static_cast<int>(i - static_cast<int64_t>(c) * b);
    const int lo = min(r, c), hi = max(r, c);
    double g = static_cast<double>(G[static_cast<int64_t>(lo) * ldg + hi]);  // upper triangle is the computed one
    if (cross) g += static_cast<double>(cross[static_cast<int64_t>(r) * ldg + c]) + static_cast<double>(cross[static_cast<int64_t>(c) * ldg + r]);
    if (exact_diag && r == c) g = exact_diag[r];  // launch_colsumsq_pair: the tensor core's diagonal is biased low
    H[i] = g - n_total * delta[r] * delta[c] + (r == c ? lam : 0.0);
  }
}
void launch_build_system(const float* G, int ldg, const double* delta, double n_total, double lam, double* H, int b,
                         cudaStream_t st, const float* cross, const double* exact_diag) {
  if (b == 0) return;
  build_system_kernel<<<grid_for(static_cast<int64_t>(b) * b, 256), 256, 0, st>>>(G, ldg, delta, n_total, lam, H, b, cross, exact_diag);
}

__global__ void build_rhs_kernel(const float* __restrict__ C, int ldc, const double* __restrict__ delta,
                                 const double* __restrict__ rsum, double n_total, double lam,
                                 const double* __restrict__ Wold, double* __restrict__ rhs, int b, int k,
                                 const float* __restrict__ c_scale) {
  const int64_t total = static_cast<int64_t>(b) * k;
  const double cs = c_scale ? static_cast<double>(__ldg(c_scale)) : 1.0;  // C was accumulated from a power-of-two scaled residual
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i / b), f = static_cast<int>(i - static_cast<int64_t>(c) * b);
    double v = static_cast<double>(C[static_cast<int64_t>(f) * ldc + c]) * cs - delta[f] * rsum[c];  // n * delta * (rsum / n)
    if (Wold) v -= lam * Wold[i];
    rhs[i] = v;
  }
}
void launch_build_rhs(const float* C, int ldc, const double* delta, const double* rsum, double n_total, double lam,
                      const double* Wold, double* rhs, int b, int k, cudaStream_t st, const float* c_scale) {
  if (b == 0 || k == 0) return;
  build_rhs_kernel<<<grid_for(static_cast<int64_t>(b) * k, 256), 256, 0, st>>>(C, ldc, delta, rsum, n_total, lam, Wold, rhs, b, k,
                                                                               c_scale);
}

// one block per class column c: packs dW[:, c] into the K-major GEMM operand row c and reduces delta . dW[:, c]
__global__ void pack_update_kernel(const double* __restrict__ dW, double* __restrict__ Wmodel,
                                   const double* __restrict__ delta, float* __restrict__ bop_hi,
                                   float* __restrict__ bop_lo, int ldb, float* __restrict__ cbias, int b, int k) {
  const int c = blockIdx.x;
  __shared__ double red[256];
  double acc = 0;
  for (int f = threadIdx.x; f < ldb; f += blockDim.x) {
    float h = 0.f, l = 0.f;
    if (c < k && f < b) {
      const double w = dW[static_cast<int64_t>(c) * b + f];
      if (Wmodel) Wmodel[static_cast<int64_t>(c) * b + f] += w;
      if (delta) acc += delta[f] * w;
      const float wf = static_cast<float>(w);
      h = round_tf32_rna(wf);
      l = round_tf32_rna(static_cast<float>(w - static_cast<double>(h)));
    }
    bop_hi[static_cast<int64_t>(c) * ldb + f] = h;
    if (bop_lo) bop_lo[static_cast<int64_t>(c) * ldb + f] = l;
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0 && cbias) cbias[c] = static_cast<float>(red[0]);
}
void launch_pack_update(const double* dW, double* Wmodel, const double* delta, float* bop_hi, float* bop_lo, int ldb,
                        float* cbias, int b, int k, int kpad, cudaStream_t st) {
  if (kpad == 0) return;
  pack_update_kernel<<<kpad, 256, 0, st>>>(dW, Wmodel, delta, bop_hi, bop_lo, ldb, cbias, b, k);
}

// cbias[c] = intercept[c] - sum_f (mean[f] - shift32[f]) W[f][c]: the slab was shifted by shift32 = fp32(mean), the rest of the
// mean goes into the constant
__global__ void pack_apply_kernel(const double* __restrict__ W, const double* __restrict__ mean, const float* __restrict__ shift32,
                                  const double* __restrict__ intercept, float* __restrict__ bop_hi, float* __restrict__ bop_lo,
                                  int ldb, float* __restrict__ cbias, int b, int k) {
  const int c = blockIdx.x;
  __shared__ double red[256];
  double acc = 0;
  for (int f = threadIdx.x; f < ldb; f += blockDim.x) {
    float h = 0.f, l = 0.f;
    if (c < k && f < b) {
      const double w = W[static_cast<int64_t>(c) * b + f];
      if (mean) acc -= (mean[f] - static_cast<double>(shift32[f])) * w;
      h = round_tf32_rna(static_cast<float>(w));
      l = round_tf32_rna(static_cast<float>(w - static_cast<double>(h)));
    }
    bop_hi[static_cast<int64_t>(c) * ldb + f] = h;
    if (bop_lo) bop_lo[static_cast<int64_t>(c) * ldb + f] = l;
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) cbias[c] = static_cast<float>(red[0] + ((intercept && c < k) ? intercept[c] : 0.0));
}
void launch_pack_apply(const double* W, const double* mean_or_null, const float* shift32, const double* intercept_or_null,
                       float* bop_hi, float* bop_lo, int ldb, float* cbias, int b, int k, int kpad, cudaStream_t st) {
  if (kpad == 0) return;
  pack_apply_kernel<<<kpad, 256, 0, st>>>(W, mean_or_null, shift32, intercept_or_null, bop_hi, bop_lo, ldb, cbias, b, k);
}

// CosineRandomFeatures W is (n_out x n_in) column-major fp64 (Breeze); the GEMM wants row-major [n_out][ld] tf32
__global__ void w_to_operand_kernel(const double* __restrict__ W, int64_t n_out, int64_t n_in, float* __restrict__ dst, int64_t ld,
                                    bool round) {
  const int64_t total = n_out * ld;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t o = i / ld, c = i - o * ld;
    const float v = c < n_in ? static_cast<float>(W[c * n_out + o]) : 0.f;
    dst[i] = round ? round_tf32_rna(v) : v;
  }
}
void launch_w_to_operand(const double* W_colmajor, int64_t n_out, int64_t n_in, float* dst, int64_t ld, cudaStream_t st, bool round) {
  if (n_out == 0) return;
  w_to_operand_kernel<<<grid_for(n_out * ld, 256), 256, 0, st>>>(W_colmajor, n_out, n_in, dst, ld, round);
}

// One CTA per image (8 warps); the image sits in shared memory, one warp builds one patch row at a time: lane l owns patch
// columns l, l + 32, ... (<= 8 per lane: patch dimension <= 256), warp-shuffle reductions for the row mean / variance.
__global__ void __launch_bounds__(256)
im2col_normalize_kernel(const float* __restrict__ images, int64_t ld_img, int x_dim, int y_dim, int ch, int conv, int normalize,
                        float var_constant, const float* __restrict__ wmeans, __half* __restrict__ out, int64_t ld_out, int concat3) {
  extern __shared__ float simg[];
  const int64_t img = blockIdx.x;
  const int npix = x_dim * y_dim * ch;
  for (int i = threadIdx.x; i < npix; i += blockDim.x) simg[i] = images[img * ld_img + i];
  __syncthreads();
  const int rw = x_dim - conv + 1, rh = y_dim - conv + 1, pd = conv * conv * ch;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int pr = warp; pr < rw * rh; pr += 8) {
    const int x = pr % rw, y = pr / rw;
    float v[8];
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int px = lane + 32 * j;
      v[j] = 0.f;
      if (px < pd) {
        const int c = px % ch, pox = (px / ch) % conv, poy = px / (ch * conv);
        v[j] = simg[c + (x + pox) * ch + (y + poy) * ch * x_dim];
        sum += v[j];
      }
    }
    if (normalize) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      const float mean = sum / static_cast<float>(pd);
      float ss = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (lane + 32 * j < pd) {
          v[j] -= mean;
          ss += v[j] * v[j];
        }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      const float inv = rsqrtf(ss / static_cast<float>(pd - 1) + var_constant);   // sample variance (n - 1), Stats.scala:117
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] *= inv;
    }
    __half* row = out + (img * static_cast<int64_t>(rw * rh) + pr) * ld_out;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int px = lane + 32 * j;
      if (px < pd) {
        const float val = v[j] - (wmeans ? wmeans[px] : 0.f);
        const __half h = __float2half_rn(val);
        row[px] = h;
        if (concat3) {
          row[pd + px] = __float2half_rn(val - __half2float(h));
          row[2 * pd + px] = h;
        }
      }
    }
    const int used = concat3 ? 3 * pd : pd;   // zero the padding columns of the row
    for (int px = used + lane; px < ld_out; px += 32) row[px] = __float2half_rn(0.f);
  }
}
void launch_im2col_normalize(const float* images, int64_t ld_img, int64_t n_images, int x_dim, int y_dim, int ch, int conv, int normalize,
                             float var_constant, const float* whitener_means, void* out16, int64_t ld_out, int concat3, cudaStream_t st) {
  if (n_images == 0) return;
  const size_t smem = sizeof(float) * static_cast<size_t>(x_dim) * y_dim * ch;
  im2col_normalize_kernel<<<static_cast<unsigned>(n_images), 256, smem, st>>>(images, ld_img, x_dim, y_dim, ch, conv, normalize,
                                                                            var_constant, whitener_means, static_cast<__half*>(out16),
                                                                            ld_out, concat3);
}

// PaddedFFT (K/nodes/stats/PaddedFFT.scala:13-21): Re(FFT(pad(x))) [f] = sum_n x[n] cos(2 pi f n / P); with RandomSignNode
// (K/nodes/stats/RandomSignNode.scala:11-16) in front, x[n] carries the sign s[n]: a fixed (P/2) x n_in matrix
__global__ void fft_real_matrix_kernel(const double* __restrict__ signs, int64_t n_in, int64_t P, float* __restrict__ dst,
                                       float* __restrict__ dst_full, int64_t ld) {
  const int64_t total = (P / 2) * ld;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t f = i / ld, n = i - f * ld;
    float v = 0.f;
    if (n < n_in) {
      const int64_t q = (f * n) % P;                       // exact phase reduction in integers
      v = static_cast<float>((signs ? signs[n] : 1.0) * cospi(2.0 * static_cast<double>(q) / static_cast<double>(P)));
    }
    dst[i] = round_tf32_rna(v);
    dst_full[i] = v;
  }
}
void launch_fft_real_matrix(const double* signs, int64_t n_in, int64_t P, float* dst, float* dst_full, int64_t ld, cudaStream_t st) {
  fft_real_matrix_kernel<<<grid_for((P / 2) * ld, 256), 256, 0, st>>>(signs, n_in, P, dst, dst_full, ld);
}

__global__ void matrix_map_kernel(const float* __restrict__ src, float* __restrict__ dst, int64_t ld, int64_t rows, int cols, int op,
                                  const float* __restrict__ colvec, float a, float b) {
  const int64_t total = rows * ld;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % ld);
    float v = 0.f;
    if (c < cols) v = op == 0 ? src[i] * colvec[c] : fmaxf(a, src[i] - b);
    dst[i] = v;
  }
}
void launch_matrix_map(const float* src, float* dst, int64_t ld, int64_t rows, int cols, int op, const float* colvec, float a, float b,
                       cudaStream_t st) {
  if (rows == 0) return;
  matrix_map_kernel<<<grid_for(rows * ld, 256), 256, 0, st>>>(src, dst, ld, rows, cols, op, colvec, a, b);
}

// ------------------------------------------------------------------ MaxClassifier (K/nodes/util/MaxClassifier.scala:9-11)
__global__ void argmax_rows_kernel(const float* __restrict__ Y, int64_t ld, int64_t rows, int k, int32_t* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  for (int64_t r = warp; r < rows; r += nwarps) {
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int c = lane; c < k; c += 32) {
      const float v = Y[r * ld + c];
      if (v > best) { best = v; bi = c; }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, off);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (lane == 0) out[r] = bi < k ? bi : 0;  // all-NaN / all -inf row: an in-range index, like Breeze's argmax
  }
}
void launch_argmax_rows(const float* Y, int64_t ld, int64_t rows, int k, int32_t* out, cudaStream_t st) {
  if (rows == 0) return;
  argmax_rows_kernel<<<grid_for(rows * 32, 256), 256, 0, st>>>(Y, ld, rows, k, out);
}

__global__ void sq_err_kernel(const float* __restrict__ Y, int64_t ldy, const float* __restrict__ L, int64_t ldl,
                              int64_t rows, int k, double* __restrict__ out) {
  double acc = 0;
  const int64_t total = rows * k;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / k;
    const int c = static_cast<int>(i - r * k);
    const double d = static_cast<double>(Y[r * ldy + c]) - static_cast<double>(L[r * ldl + c]);
    acc += d * d;
  }
  __shared__ double red[256];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) atomicAdd(out, red[0]);
}
void launch_sq_err(const float* Y, int64_t ldy, const float* L, int64_t ldl, int64_t rows, int k, double* out,
                   cudaStream_t st) {
  if (rows == 0) return;
  sq_err_kernel<<<grid_for(rows * k, 256), 256, 0, st>>>(Y, ldy, L, ldl, rows, k, out);
}

// =====================================================================================
// fp16 operand path (precision mode KS_PRECISION_F16): fp16 has the 10-bit mantissa of tf32 but a 5-bit exponent, so the
// operands whose magnitude the data decides (residual, weight increments) are multiplied by a power of two chosen on the
// device from their largest magnitude; the power of two is divided out again in fp32 / fp64 after the MMA.
// =====================================================================================
// maxbits: bit pattern of the largest |x| seen (non-negative floats order like unsigned integers); must be zeroed
__global__ void max_abs_f32_kernel(const float* __restrict__ p, int64_t ld, int64_t rows, int cols, unsigned* __restrict__ maxbits) {
  float m = 0.f;
  const int64_t total = rows * cols;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / cols;
    const int c = static_cast<int>(i - r * cols);
    m = fmaxf(m, fabsf(p[r * ld + c]));
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(maxbits, __float_as_uint(m));
}
__global__ void max_abs_f64_kernel(const double* __restrict__ p, int64_t n, unsigned* __restrict__ maxbits) {
  float m = 0.f;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    m = fmaxf(m, fabsf(static_cast<float>(p[i])));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(maxbits, __float_as_uint(m));
}
// scale[0] = 2^e with max * 2^e in [target / 2, target], scale[1] = 2^-e   (max == 0, inf or nan: 1, 1)
__global__ void pow2_scale_kernel(const unsigned* __restrict__ maxbits, float target, float* __restrict__ scale) {
  const float m = __uint_as_float(*maxbits);
  float s = 1.f, inv = 1.f;
  if (m > 0.f && m < 3.0e38f) {
    int e = static_cast<int>(floorf(log2f(target / m)));
    e = max(-100, min(100, e));
    s = exp2f(static_cast<float>(e));
    inv = exp2f(static_cast<float>(-e));
    if (m * s > target) { s *= 0.5f; inv *= 2.f; }  // log2f rounding at an exact power of two
  }
  scale[0] = s;
  scale[1] = inv;
}
void launch_max_abs_f32(const float* p, int64_t ld, int64_t rows, int cols, unsigned* maxbits, cudaStream_t st) {
  if (rows == 0 || cols == 0) return;
  max_abs_f32_kernel<<<grid_for(rows * cols, 256), 256, 0, st>>>(p, ld, rows, cols, maxbits);
}
void launch_max_abs_f64(const double* p, int64_t n, unsigned* maxbits, cudaStream_t st) {
  if (n == 0) return;
  max_abs_f64_kernel<<<grid_for(n, 256, 132 * 2), 256, 0, st>>>(p, n, maxbits);
}
void launch_pow2_scale(const unsigned* maxbits, float target, float* scale, cudaStream_t st) {
  pow2_scale_kernel<<<1, 1, 0, st>>>(maxbits, target, scale);
}

__global__ void f32_to_f16_rows_kernel(const float* __restrict__ src, int64_t src_ld, __half* __restrict__ dst, int64_t dst_ld,
                                       int64_t rows, int64_t cols, const float* __restrict__ scale) {
  const int64_t total = rows * dst_ld;
  const float sc = scale ? __ldg(scale) : 1.f;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / dst_ld, c = i - r * dst_ld;
    dst[i] = __float2half_rn(c < cols ? src[r * src_ld + c] * sc : 0.f);
  }
}
void launch_f32_to_f16_rows(const float* src, int64_t src_ld, void* dst, int64_t dst_ld, int64_t rows, int64_t cols, cudaStream_t st,
                            const float* scale) {
  if (rows == 0) return;
  f32_to_f16_rows_kernel<<<grid_for(rows * dst_ld, 256), 256, 0, st>>>(src, src_ld, static_cast<__half*>(dst), dst_ld, rows, cols,
                                                                       scale);
}

// fp16 twin of round_colsum_kernel: R16[:, :k] = fp16(R * scale[0]), columns >= k zero; sums as before (of R itself)
// R16lo (optional, split-operand mode): the fp16 rounding error of the scaled value, fp16(R * scale - R16)
__global__ void round_colsum16_kernel(const float* __restrict__ R, __half* __restrict__ R16, int64_t ld, int64_t rows, int k,
                                      double* __restrict__ sums, int64_t rows_per_block, const float* __restrict__ scale,
                                      __half* __restrict__ R16lo, unsigned* __restrict__ overflow) {
  __shared__ double red[8][128];
  const float sc = __ldg(scale);
  const int c4 = (blockIdx.x * 32 + threadIdx.x) * 4;
  const int64_t r_begin = blockIdx.y * rows_per_block;
  const int64_t r_end = min(rows, r_begin + rows_per_block);
  double a[4] = {0, 0, 0, 0};
  if (c4 < ld) {
    for (int64_t r = r_begin + threadIdx.y; r < r_end; r += 8) {
      const float4 v = *reinterpret_cast<const float4*>(R + r * ld + c4);
      const float in[4] = {v.x, v.y, v.z, v.w};
      float o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = c4 + j;
        if (c < k) {
          a[j] += in[j];
          o[j] = in[j] * sc;
          // the residual's scale was fixed from max|R_0| with 16x headroom; a residual that grew past fp16's range (its max
          // norm is not monotone under block coordinate descent) must not turn into inf silently
          if (overflow && !(fabsf(o[j]) <= 65504.f)) *overflow = 1u;
        } else {
          o[j] = 0.f;
        }
      }
      const __half2 h0 = f16_hi2(o[0], o[1]), h1 = f16_hi2(o[2], o[3]);
      uint2 pk;
      pk.x = *reinterpret_cast<const unsigned*>(&h0);
      pk.y = *reinterpret_cast<const unsigned*>(&h1);
      *reinterpret_cast<uint2*>(R16 + r * ld + c4) = pk;
      if (R16lo) {
        const __half2 l0 = f16_lo2(o[0], o[1], h0), l1 = f16_lo2(o[2], o[3], h1);
        uint2 pl;
        pl.x = *reinterpret_cast<const unsigned*>(&l0);
        pl.y = *reinterpret_cast<const unsigned*>(&l1);
        *reinterpret_cast<uint2*>(R16lo + r * ld + c4) = pl;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) red[threadIdx.y][threadIdx.x * 4 + j] = a[j];
  __syncthreads();
  const int t = threadIdx.y * 32 + threadIdx.x;
  if (t < 128) {
    double s = 0;
#pragma unroll
    for (int y = 0; y < 8; ++y) s += red[y][t];
    const int c = blockIdx.x * 128 + t;
    if (c < k) atomicAdd(sums + c, s);
  }
}
void launch_round_colsum16(const float* R, void* R16, int64_t ld, int64_t rows, int k, double* sums, const float* scale,
                           cudaStream_t st, void* R16lo, unsigned* overflow) {
  if (rows == 0) return;
  const int64_t rpb = 1024;
  dim3 grid(static_cast<unsigned>((ld + 127) / 128), static_cast<unsigned>((rows + rpb - 1) / rpb));
  round_colsum16_kernel<<<grid, dim3(32, 8), 0, st>>>(R, static_cast<__half*>(R16), ld, rows, k, sums, rpb, scale,
                                                      static_cast<__half*>(R16lo), overflow);
}

// fp16 twin of pack_update_kernel: bop16[c][f] = fp16(dW[f][c] * scale[0]); Wmodel and cbias exactly as the tf32 version
__global__ void pack_update16_kernel(const double* __restrict__ dW, double* __restrict__ Wmodel,
                                     const double* __restrict__ delta, __half* __restrict__ bop, int ldb,
                                     float* __restrict__ cbias, int b, int k, const float* __restrict__ scale,
                                     __half* __restrict__ bop_lo) {
  const int c = blockIdx.x;
  const double sc = static_cast<double>(__ldg(scale));
  __shared__ double red[256];
  double acc = 0;
  for (int f = threadIdx.x; f < ldb; f += blockDim.x) {
    double ws = 0.0;
    if (c < k && f < b) {
      const double w = dW[static_cast<int64_t>(c) * b + f];
      if (Wmodel) Wmodel[static_cast<int64_t>(c) * b + f] += w;
      if (delta) acc += delta[f] * w;
      ws = w * sc;
    }
    const __half hh = __float2half_rn(static_cast<float>(ws));
    bop[static_cast<int64_t>(c) * ldb + f] = hh;
    if (bop_lo) bop_lo[static_cast<int64_t>(c) * ldb + f] = __float2half_rn(static_cast<float>(ws - static_cast<double>(__half2float(hh))));
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0 && cbias) cbias[c] = static_cast<float>(red[0]);
}
void launch_pack_update16(const double* dW, double* Wmodel, const double* delta, void* bop16, int ldb, float* cbias, int b, int k,
                          int kpad, const float* scale, cudaStream_t st, void* bop16_lo) {
  if (kpad == 0) return;
  pack_update16_kernel<<<kpad, 256, 0, st>>>(dW, Wmodel, delta, static_cast<__half*>(bop16), ldb, cbias, b, k, scale,
                                             static_cast<__half*>(bop16_lo));
}

// ---- split-operand mode (fp16 x 2): v = hi + lo with hi = fp16(v), lo = fp16(v - hi)  (21 significant bits in two fp16)
// projection operands, concatenated along K so that ONE GEMM of depth 3 * cols accumulates hi*hi + lo*hi + hi*lo:
//   pattern 0 (left operand X):  dst row = [ hi | lo | hi ],   pattern 1 (right operand W): dst row = [ hi | hi | lo ]
__global__ void split_concat3_kernel(const float* __restrict__ src, int64_t ld_src, int64_t rows, int cols,
                                     const float* __restrict__ scale, __half* __restrict__ dst, int64_t ld_dst, int pattern) {
  const float sc = scale ? __ldg(scale) : 1.f;
  const int64_t total = rows * ld_dst;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / ld_dst;
    const int c = static_cast<int>(i - r * ld_dst);
    __half out = __float2half_rn(0.f);
    if (c < 3 * cols) {
      const int part = c / cols, cc = c - part * cols;
      const float v = src[r * ld_src + cc] * sc;
      const __half h = __float2half_rn(v);
      const bool want_lo = pattern == 0 ? part == 1 : part == 2;
      out = want_lo ? __float2half_rn(v - __half2float(h)) : h;
    }
    dst[i] = out;
  }
}
void launch_split_concat3(const float* src, int64_t ld_src, int64_t rows, int cols, const float* scale, void* dst, int64_t ld_dst,
                          int pattern, cudaStream_t st) {
  if (rows == 0) return;
  split_concat3_kernel<<<grid_for(rows * ld_dst, 256), 256, 0, st>>>(src, ld_src, rows, cols, scale, static_cast<__half*>(dst), ld_dst,
                                                                    pattern);
}

// ---- evaluation: confusion matrix counts[actual * k + predicted] += 1 (K/evaluation/MulticlassClassifierEvaluator.scala:149-160)
__global__ void confusion_kernel(const int32_t* __restrict__ pred, const int32_t* __restrict__ act, int64_t n, int k,
                                 unsigned long long* __restrict__ counts) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int p = pred[i], a = act[i];
    if (static_cast<unsigned>(p) < static_cast<unsigned>(k) && static_cast<unsigned>(a) < static_cast<unsigned>(k))
      atomicAdd(counts + static_cast<int64_t>(a) * k + p, 1ULL);
  }
}
void launch_confusion(const int32_t* pred, const int32_t* act, int64_t n, int k, unsigned long long* counts, cudaStream_t st) {
  if (n == 0) return;
  confusion_kernel<<<grid_for(n, 256), 256, 0, st>>>(pred, act, n, k, counts);
}

}  // namespace ks
