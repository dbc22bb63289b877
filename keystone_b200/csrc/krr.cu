// Gaussian-kernel ridge regression on the device: GaussianKernelGenerator / KernelMatrix / KernelRidgeRegression /
// KernelBlockLinearMapper (K/nodes/learning/{KernelGenerator,KernelMatrix,KernelRidgeRegression,KernelBlockLinearMapper}.scala).
//
// The fit solves (K + lambda I) W = Y by block Gauss-Seidel over contiguous blocks of TRAINING ROWS (trainWithL2,
// KernelRidgeRegression.scala:116-200), in increment form:
//   C      = K_B^T W                    split-operand Gram of the generated slab K_B [n_loc x b] against W's fp16 pair
//   rhs    = Y_B - C - lambda W_B       (Y_B folded into the all-reduce of C: every rank subtracts the rows it owns)
//   dW     = (K_BB + lambda I) \ rhs    K_BB in fp64 from the replicated training rows, Cholesky, potrs
//   W_B   += dW
// which is the reference's W_B = (K_BB + lambda I) \ (Y_B - C + K_BB W_B,old) with (K_BB + lambda I) W_B,old subtracted from
// both sides.  The kernel block K_B is regenerated every step by the projection GEMM with the EPI_RBF epilogue.  DESIGN.md 13.
#include "engine.h"

#include <cuda_fp16.h>
#include <math.h>

#include <algorithm>
#include <chrono>
#include <sstream>

namespace ks {

static unsigned krr_grid(int64_t n, int threads = 256, int64_t cap = 132 * 16) {
  int64_t g = (n + threads - 1) / threads;
  return static_cast<unsigned>(std::max<int64_t>(1, std::min(g, cap)));
}

static void tmap16(CUtensorMap* m, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_cols, int box_rows, int sw) {
  const int r = make_tmap_any(m, base, rows, cols, ld, box_cols, box_rows, 2, sw);
  if (r != 0)
    throw KsError{KS_ERR_CUDA, "cuTensorMapEncodeTiled (fp16) failed (" + std::to_string(r) + ") rows=" + std::to_string(rows) +
                                   " cols=" + std::to_string(cols) + " ld=" + std::to_string(ld)};
}

// ------------------------------------------------------------------------------------ small kernels
// exact fp64 column sums in a fixed order (the same bits on every rank): partial sums per 256-row chunk, then over the chunks
__global__ void colsum_chunks_kernel(const float* __restrict__ X, int64_t ld, int64_t rows, int cols, int64_t rpc,
                                     double* __restrict__ part) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  const int64_t r0 = blockIdx.y * rpc, r1 = min(rows, r0 + rpc);
  double s = 0;
  for (int64_t r = r0; r < r1; ++r) s += X[r * ld + c];
  part[blockIdx.y * static_cast<int64_t>(cols) + c] = s;
}
__global__ void mean_from_chunks_kernel(const double* __restrict__ part, int chunks, int cols, double inv_n, double* __restrict__ mean) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  double s = 0;
  for (int q = 0; q < chunks; ++q) s += part[static_cast<int64_t>(q) * cols + c];
  mean[c] = s * inv_n;
}
// dst[r][c] = fp32(src[r][c] - mean[c]) (fp64 difference), padding columns zero; dst may equal src
__global__ void shift_rows_kernel(const float* src, int64_t lds, int64_t rows, int cols, const double* __restrict__ mean, float* dst,
                                  int64_t ldd) {
  const int64_t total = rows * ldd;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / ldd;
    const int c = static_cast<int>(i - r * ldd);
    dst[i] = c < cols ? static_cast<float>(static_cast<double>(src[r * lds + c]) - mean[c]) : 0.f;
  }
}
// out[r] = sum_c ((hi + lo) 2^-e)^2 with hi = fp16(2^e x), lo = fp16(2^e x - hi) exactly as launch_split_concat3 forms them:
// the squared norm of the values the MMA operands represent.  One warp per row.
__global__ void pair_norms_kernel(const float* __restrict__ X, int64_t ld, int64_t rows, int cols, const float* __restrict__ scale,
                                  float* __restrict__ out) {
  const int64_t r = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float s = scale[0];
  const double inv = static_cast<double>(scale[1]);
  double acc = 0;
  for (int c = lane; c < cols; c += 32) {
    const float v = X[r * ld + c] * s;
    const __half h = __float2half_rn(v);
    const __half l = __float2half_rn(v - __half2float(h));
    const double q = (static_cast<double>(__half2float(h)) + static_cast<double>(__half2float(l))) * inv;
    acc += q * q;
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) out[r] = static_cast<float>(acc);
}
__global__ void mul_scales_kernel(const float* a, const float* b, float* out) { out[0] = a[1] * b[1]; }
__global__ void neg_inv_scale_kernel(float* s) { s[2] = -s[1]; }
__global__ void set_unit_scale_kernel(float* s) { s[0] = 1.f; s[1] = 1.f; }

// H (fp64, column-major b x b, lower triangle) = exp(-gamma |x_i - x_j|^2) + lam I over the rows of one block of the shifted
// training X (KernelGenerator.scala:186-194 builds it from the raw block in fp64).  64 x 64 tiles on 256 threads (4 x 4 each);
// tiles above the diagonal are skipped (the Cholesky reads the lower triangle only).
__global__ void __launch_bounds__(256) kbb_kernel(const float* __restrict__ X, int64_t ld, int d, int b, double gamma, double lam,
                                                  double* __restrict__ H) {
  const int ti = blockIdx.y, tj = blockIdx.x;
  if (tj > ti) return;
  __shared__ double As[32][65], Bs[32][65];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  double acc[4][4];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) acc[u][v] = 0.0;
  for (int k0 = 0; k0 < d; k0 += 32) {
    for (int e = threadIdx.x; e < 64 * 32; e += 256) {
      const int r = e >> 5, kk = e & 31, kc = k0 + kk;
      const int gi = ti * 64 + r, gj = tj * 64 + r;
      As[kk][r] = (gi < b && kc < d) ? static_cast<double>(X[static_cast<int64_t>(gi) * ld + kc]) : 0.0;
      Bs[kk][r] = (gj < b && kc < d) ? static_cast<double>(X[static_cast<int64_t>(gj) * ld + kc]) : 0.0;
    }
    __syncthreads();
#pragma unroll 4
    for (int kk = 0; kk < 32; ++kk) {
      double a[4], bb[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) a[u] = As[kk][ty + 16 * u];
#pragma unroll
      for (int v = 0; v < 4; ++v) bb[v] = Bs[kk][tx + 16 * v];
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          const double df = a[u] - bb[v];
          acc[u][v] = fma(df, df, acc[u][v]);
        }
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int i = ti * 64 + ty + 16 * u, j = tj * 64 + tx + 16 * v;
      if (i < b && j < b) H[static_cast<int64_t>(j) * b + i] = exp(-gamma * acc[u][v]) + (i == j ? lam : 0.0);
    }
}

// C[f][c] -= 2^e Y(c0 + f)[c] for the rows of block [c0, c0 + b) this rank owns; summed over the ranks, C = 2^e (K_B^T W - Y_B)
__global__ void fold_labels_kernel(float* __restrict__ C, int ldc, const float* __restrict__ Y, int64_t ldy, int k, int64_t f0,
                                   int64_t nf, int64_t y0, const float* __restrict__ sc) {
  const float s = sc[0];
  const int64_t total = nf * k;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t q = i / k;
    const int c = static_cast<int>(i - q * k);
    C[(f0 + q) * ldc + c] -= s * Y[(y0 + q) * ldy + c];
  }
}
// rhs (fp64 column-major b x k) = -2^-e C - lam W_B = Y_B - K_B^T W - lam W_B
__global__ void krr_rhs_kernel(const float* __restrict__ C, int ldc, const float* __restrict__ sc, double lam, const double* __restrict__ Wb,
                               double* __restrict__ rhs, int b, int k) {
  const double inv = static_cast<double>(sc[1]);
  const int64_t total = static_cast<int64_t>(b) * k;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i / b), f = static_cast<int>(i - static_cast<int64_t>(c) * b);
    rhs[i] = -static_cast<double>(C[static_cast<int64_t>(f) * ldc + c]) * inv - lam * Wb[i];
  }
}
__global__ void add_f64_kernel(double* __restrict__ dst, const double* __restrict__ src, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    dst[i] += src[i];
}
// W's operand scale 2^e from the running max |W| (largest magnitude mapped into [2048, 4096], as launch_pow2_scale);
// *changed = 1 when e moved, and then every packed row of W has to be packed again
__global__ void w_scale_kernel(const unsigned* __restrict__ maxbits, float* __restrict__ sc, unsigned* __restrict__ changed) {
  const float m = __uint_as_float(*maxbits);
  float s = 1.f, inv = 1.f;
  if (m > 0.f && m < 3.0e38f) {
    int e = static_cast<int>(floorf(log2f(4096.f / m)));
    e = max(-100, min(100, e));
    s = exp2f(static_cast<float>(e));
    inv = exp2f(static_cast<float>(-e));
    if (m * s > 4096.f) { s *= 0.5f; inv *= 2.f; }
  }
  *changed = s != sc[0] ? 1u : 0u;
  sc[0] = s;
  sc[1] = inv;
}
// W operand of this rank's rows, Wop hi / lo [n_loc][kpad] = fp16 pair of 2^e W(row_off + r, :); W in block layout (block j at
// W + c0_j k, column-major b_j x k).  Rows: all of them when the scale changed, else those of block [c0, c0 + b)
__global__ void pack_wop_kernel(const double* __restrict__ W, int64_t n, int bs, int k, int kpad, int64_t row_off, int64_t n_loc,
                                int64_t c0, int b, const float* __restrict__ sc, const unsigned* __restrict__ changed,
                                __half* __restrict__ hi, __half* __restrict__ lo) {
  int64_t r0 = 0, r1 = n_loc;
  if (!*changed) {
    r0 = max(static_cast<int64_t>(0), c0 - row_off);
    r1 = min(n_loc, c0 + b - row_off);
  }
  if (r1 <= r0) return;
  const float s = sc[0];
  const int64_t total = (r1 - r0) * kpad;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = r0 + i / kpad;
    const int c = static_cast<int>(i % kpad);
    float v = 0.f;
    if (c < k) {
      const int64_t g = row_off + r, bc0 = g / bs * bs, bj = min(static_cast<int64_t>(bs), n - bc0);
      v = static_cast<float>(W[bc0 * k + c * bj + (g - bc0)] * static_cast<double>(s));
    }
    const __half h = __float2half_rn(v);
    hi[r * kpad + c] = h;
    lo[r * kpad + c] = __float2half_rn(v - __half2float(h));
  }
}
__global__ void pair_to_f32_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo, int64_t lds, int64_t rows, int cols,
                                   float* __restrict__ out, int64_t ldo) {
  const int64_t total = rows * ldo;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / ldo;
    const int c = static_cast<int>(i - r * ldo);
    out[i] = c < cols ? __half2float(hi[r * lds + c]) + __half2float(lo[r * lds + c]) : 0.f;
  }
}

// ------------------------------------------------------------------------------------ row-side operands
// The row side of a generated kernel block: x - m as the K-concatenated fp16 pair [hi | lo | hi] of 2^e (x - m), its squared
// norms, and scale = {2^e, 2^-e, 2^-e 2^-e_train (the accumulator scale), max |x - m| bits}.
struct RowOps {
  DevBuf shifted, x3, norms, scale;
  int64_t rows = 0;
};

// x: fp32 rows (ldx).  shift: x is raw input (test rows): subtract m and choose its own scale; otherwise x is already shifted
// training data and takes the kernel's scale.
static void prep_rows(Ctx& c, const GaussKernel& K, const float* x, int64_t ldx, int64_t rows, bool shift, RowOps& o, cudaStream_t st) {
  o.rows = rows;
  const int d = static_cast<int>(K.d);
  o.scale.alloc(sizeof(float) * 4);
  float* sc = o.scale.as<float>();
  unsigned* mb = o.scale.as<unsigned>() + 3;
  const float* src = x;
  int64_t lds = ldx;
  if (shift) {
    o.shifted.alloc(sizeof(float) * static_cast<size_t>(std::max<int64_t>(rows, 1) * K.ld));
    if (rows > 0) shift_rows_kernel<<<krr_grid(rows * K.ld), 256, 0, st>>>(x, ldx, rows, d, K.mean.as<double>(), o.shifted.as<float>(), K.ld);
    src = o.shifted.as<float>();
    lds = K.ld;
    KS_CUDA(cudaMemsetAsync(mb, 0, sizeof(unsigned), st));
    launch_max_abs_f32(src, lds, rows, d, mb, st);
    launch_pow2_scale(mb, 4096.f, sc, st);
    c.launches += 3;
  } else {
    KS_CUDA(cudaMemcpyAsync(sc, K.scale.p, sizeof(float) * 2, cudaMemcpyDeviceToDevice, st));
  }
  mul_scales_kernel<<<1, 1, 0, st>>>(sc, K.scale.as<float>(), sc + 2);
  o.x3.alloc(2 * static_cast<size_t>(std::max<int64_t>(rows, 1) * K.ld3));
  launch_split_concat3(src, lds, rows, d, sc, o.x3.p, K.ld3, 0, st);
  o.norms.alloc(sizeof(float) * static_cast<size_t>(std::max<int64_t>(rows, 1)));
  if (rows > 0) pair_norms_kernel<<<static_cast<unsigned>((rows * 32 + 255) / 256), 256, 0, st>>>(src, lds, rows, d, sc, o.norms.as<float>());
  c.launches += 3;
}

// slab hi / lo [rows x cols] (fp16 pair, ld lds) = K(rows [r0, r0 + rows) of A, training rows [c0, c0 + cols)): the projection
// GEMM over the concatenated operands (depth 3 d: hi hi + lo hi + hi lo) with the EPI_RBF epilogue
static void gen_rbf(Ctx& c, const GaussKernel& K, const RowOps& A, int64_t r0, int64_t rows, int64_t c0, int cols, void* hi, void* lo,
                    int64_t lds, cudaStream_t st) {
  if (rows <= 0 || cols <= 0) return;
  KmLaunch k;
  const int64_t kdepth = 3 * K.d;
  tmap16(&k.tmA, static_cast<const uint16_t*>(A.x3.p) + r0 * K.ld3, rows, kdepth, K.ld3, 64, 128, TMAP_SW128);
  tmap16(&k.tmB, static_cast<const uint16_t*>(K.xb3.p) + c0 * K.ld3, cols, kdepth, K.ld3, 64, 128, TMAP_SW128);
  tmap16(&k.tmOut, hi, rows, cols, lds, 32, 32, TMAP_NONE);
  tmap16(&k.tmOut2, lo, rows, cols, lds, 32, 32, TMAP_NONE);
  k.f16 = 1;
  k.out16 = 2;
  k.p.acc_scale_ptr = A.scale.as<float>() + 2;
  k.p.vec0 = K.norms.as<float>() + c0;
  k.p.vec1 = nullptr;
  k.p.colsum = nullptr;
  k.p.row_vec = A.norms.as<float>() + r0;
  k.p.gamma = static_cast<float>(K.gamma);
  k.p.M = static_cast<int>(rows);
  k.p.N = cols;
  k.p.K = static_cast<int>(kdepth);
  k.p.flags = 0;
  k.epi = EPI_RBF;
  // persistent kernel: beside the solve chain leave it a few SMs (as produce_slab does)
  k.num_sms = (st == c.st2) ? std::max(1, c.num_sms - c.reserve_sms) : c.num_sms;
  if (c.dyn_tiles) k.p.tile_counter = c.next_tile_counter(st);
  KS_CUDA(launch_kmajor(k, st));
  c.launches += 1;
}

// ------------------------------------------------------------------------------------ GaussianKernelGenerator.fit
int64_t gaussian_kernel_create(Ctx& c, Matrix& X, double gamma) {
  if (!(gamma > 0) || !std::isfinite(gamma)) throw KsError{KS_ERR_INVALID, "gamma must be finite and > 0"};
  auto K = std::make_shared<GaussKernel>();
  K->gamma = gamma;
  K->d = X.cols;
  K->ld = X.ld;
  K->ld3 = round_up(3 * K->d, 64);
  cudaStream_t st = c.st;
  // every rank's row count and width
  std::vector<double> meta(2 * c.world, 0.0);
  meta[c.rank] = static_cast<double>(X.rows);
  meta[c.world + c.rank] = static_cast<double>(X.cols);
  if (c.world > 1) {
    DevBuf dm;
    dm.alloc(sizeof(double) * meta.size());
    KS_CUDA(cudaMemcpyAsync(dm.p, meta.data(), dm.bytes, cudaMemcpyHostToDevice, st));
    c.allreduce_f64(dm.as<double>(), meta.size());
    KS_CUDA(cudaMemcpyAsync(meta.data(), dm.p, sizeof(double) * meta.size(), cudaMemcpyDeviceToHost, st));
    KS_CUDA(cudaStreamSynchronize(st));
  }
  std::vector<int64_t> counts(c.world), offs(c.world + 1, 0);
  for (int r = 0; r < c.world; ++r) {
    counts[r] = static_cast<int64_t>(meta[r]);
    if (static_cast<int64_t>(meta[c.world + r]) != X.cols)
      throw KsError{KS_ERR_INVALID, "the training rows of every rank must have the same column count"};
    offs[r + 1] = offs[r] + counts[r];
  }
  K->n = offs[c.world];
  K->row_off = offs[c.rank];
  K->n_loc = X.rows;
  if (K->n < 1 || K->d < 1) throw KsError{KS_ERR_INVALID, "empty training set"};
  const int64_t n = K->n, ld = K->ld;
  const int d = static_cast<int>(K->d);
  // the whole training X on every rank, in the global row order (rank by rank: zipWithIndex)
  K->xs.alloc(sizeof(float) * static_cast<size_t>(n * ld));
  if (X.rows > 0)
    KS_CUDA(cudaMemcpyAsync(K->xs.as<float>() + K->row_off * ld, X.d, sizeof(float) * X.rows * ld, cudaMemcpyDeviceToDevice, st));
  if (c.world > 1) {
    KS_NCCL(nccl_api().GroupStart());
    for (int r = 0; r < c.world; ++r) {
      if (counts[r] == 0) continue;
      float* p = K->xs.as<float>() + offs[r] * ld;
      KS_NCCL(nccl_api().Broadcast(p, p, static_cast<size_t>(counts[r] * ld), ncclFloat32, r, c.comm, st));
    }
    KS_NCCL(nccl_api().GroupEnd());
  }
  // exact fp64 column mean m, then x - m in place
  const int64_t rpc = 256, chunks = (n + rpc - 1) / rpc;
  DevBuf part;
  part.alloc(sizeof(double) * static_cast<size_t>(chunks * d));
  K->mean.alloc(sizeof(double) * d);
  colsum_chunks_kernel<<<dim3((d + 127) / 128, static_cast<unsigned>(chunks)), 128, 0, st>>>(K->xs.as<float>(), ld, n, d, rpc, part.as<double>());
  mean_from_chunks_kernel<<<(d + 127) / 128, 128, 0, st>>>(part.as<double>(), static_cast<int>(chunks), d, 1.0 / static_cast<double>(n),
                                                           K->mean.as<double>());
  shift_rows_kernel<<<krr_grid(n * ld), 256, 0, st>>>(K->xs.as<float>(), ld, n, d, K->mean.as<double>(), K->xs.as<float>(), ld);
  // operand scale, column-side operand [hi | hi | lo], norms
  K->scale.alloc(sizeof(float) * 4);
  unsigned* mb = K->scale.as<unsigned>() + 3;
  KS_CUDA(cudaMemsetAsync(mb, 0, sizeof(unsigned), st));
  launch_max_abs_f32(K->xs.as<float>(), ld, n, d, mb, st);
  launch_pow2_scale(mb, 4096.f, K->scale.as<float>(), st);
  K->xb3.alloc(2 * static_cast<size_t>(n * K->ld3));
  launch_split_concat3(K->xs.as<float>(), ld, n, d, K->scale.as<float>(), K->xb3.p, K->ld3, 1, st);
  K->norms.alloc(sizeof(float) * static_cast<size_t>(n));
  pair_norms_kernel<<<static_cast<unsigned>((n * 32 + 255) / 256), 256, 0, st>>>(K->xs.as<float>(), ld, n, d, K->scale.as<float>(),
                                                                                K->norms.as<float>());
  c.launches += 7;
  c.check_async("GaussianKernelGenerator.fit");
  const int64_t h = c.next_id++;
  c.kernels[h] = std::move(K);
  return h;
}

// ------------------------------------------------------------------------------------ KernelMatrix(colIdxs)
std::unique_ptr<Matrix> gaussian_kernel_block(Ctx& c, const GaussKernel& K, Matrix& x, int64_t col0, int64_t cols) {
  if (x.cols != K.d) throw KsError{KS_ERR_INVALID, "input rows have a different column count than the training rows"};
  if (col0 < 0 || cols < 1 || col0 + cols > K.n) throw KsError{KS_ERR_INVALID, "column range outside the training rows"};
  if (cols > (1 << 30)) throw KsError{KS_ERR_INVALID, "column range too large"};
  cudaStream_t st = c.st;
  RowOps A;
  prep_rows(c, K, x.d, x.ld, x.rows, true, A, st);
  const int64_t lds = round_up(cols, 32);
  DevBuf hi, lo;
  hi.alloc(2 * static_cast<size_t>(std::max<int64_t>(x.rows, 1) * lds));
  lo.alloc(hi.bytes);
  gen_rbf(c, K, A, 0, x.rows, col0, static_cast<int>(cols), hi.p, lo.p, lds, st);
  auto out = new_matrix(x.rows, cols);
  if (x.rows > 0) {
    pair_to_f32_kernel<<<krr_grid(x.rows * out->ld), 256, 0, st>>>(hi.as<__half>(), lo.as<__half>(), lds, x.rows, static_cast<int>(cols),
                                                                  out->d, out->ld);
    c.launches += 1;
  }
  c.check_async("KernelMatrix");
  return out;
}

// ------------------------------------------------------------------------------------ KernelRidgeRegression.fit
int64_t fit_krr(Ctx& c, const std::shared_ptr<GaussKernel>& Kp, Matrix& Y, double lam, int bs, int epochs, const int32_t* order) {
  GaussKernel& K = *Kp;
  if (bs < 1) throw KsError{KS_ERR_INVALID, "blockSize must be >= 1"};
  if (epochs < 1) throw KsError{KS_ERR_INVALID, "numEpochs must be >= 1"};
  if (!(lam >= 0) || !std::isfinite(lam)) throw KsError{KS_ERR_INVALID, "lambda must be finite and >= 0"};
  if (Y.rows != K.n_loc) throw KsError{KS_ERR_INVALID, "labels have a different row count than this rank's training rows"};
  if (Y.cols < 1) throw KsError{KS_ERR_INVALID, "labels have no columns"};
  const int64_t n = K.n, n_loc = K.n_loc, row_off = K.row_off;
  const int nb = static_cast<int>((n + bs - 1) / bs);
  const int k = static_cast<int>(Y.cols);
  std::vector<int> steps;  // block of every step
  for (int e = 0; e < epochs; ++e) {
    std::vector<char> seen(nb, 0);
    for (int q = 0; q < nb; ++q) {
      const int j = order ? order[static_cast<int64_t>(e) * nb + q] : q;
      if (j < 0 || j >= nb || seen[j]) throw KsError{KS_ERR_INVALID, "block_order row " + std::to_string(e) + " is not a permutation of the blocks"};
      seen[j] = 1;
      steps.push_back(j);
    }
  }
  const int T = static_cast<int>(steps.size());
  const int bmax = static_cast<int>(std::min<int64_t>(bs, n));
  const int64_t lds = round_up(bmax, 32), kpad = round_up(k, 32);
  const int ldc = static_cast<int>(kpad);
  auto block = [&](int j, int64_t* c0) {
    *c0 = static_cast<int64_t>(j) * bs;
    return static_cast<int>(std::min<int64_t>(n, *c0 + bs) - *c0);
  };
  cudaStream_t S1 = c.st, ST = c.st2, SF = c.st3, S5 = c.st5;
  cudaStream_t SS = S1;  // the residual chain: all-reduce, rhs, solve, W update, operand re-pack
  const auto host_t0 = std::chrono::steady_clock::now();
  c.spans.clear();
  const int64_t launches0 = c.launches;
  auto new_event = [&]() {
    cudaEvent_t e = c.get_event();
    c.fit_events.push_back(e);
    return e;
  };
  cudaEvent_t ev0 = new_event(), ev1 = new_event(), ev_init = new_event();
  KS_CUDA(cudaStreamSynchronize(ST));
  KS_CUDA(cudaStreamSynchronize(SF));
  KS_CUDA(cudaStreamSynchronize(S5));
  KS_CUDA(cudaEventRecord(ev0, S1));

  auto model = std::make_unique<Model>();
  model->kernel = Kp;
  model->block_size = bs;
  model->k = k;
  for (int j = 0; j < nb; ++j) {
    int64_t c0;
    const int b = block(j, &c0);
    model->brows.push_back(b);
    auto W = std::make_unique<DevBuf>();
    W->alloc(sizeof(double) * static_cast<size_t>(b) * k);
    model->W.push_back(std::move(W));
  }
  model->intercept.alloc(sizeof(double) * k);
  if (c.host_mirror) model_alloc_host(*model);

  // ---- workspace
  const bool cache_factors = epochs > 1;
  DevBuf Wall, wop_hi, wop_lo, cm, rhs, state;
  DevBuf slab_hi[2], slab_lo[2], Hbuf[2];
  std::vector<std::unique_ptr<DevBuf>> factors(nb);
  Wall.alloc(sizeof(double) * static_cast<size_t>(n) * k);
  wop_hi.alloc(2 * static_cast<size_t>(std::max<int64_t>(n_loc, 1) * kpad));
  wop_lo.alloc(wop_hi.bytes);
  cm.alloc(sizeof(float) * static_cast<size_t>(bmax) * ldc);
  rhs.alloc(sizeof(double) * static_cast<size_t>(bmax) * k);
  for (int i = 0; i < 2; ++i) {
    slab_hi[i].alloc(2 * static_cast<size_t>(std::max<int64_t>(n_loc, 1) * lds));
    slab_lo[i].alloc(slab_hi[i].bytes);
    if (!cache_factors) Hbuf[i].alloc(sizeof(double) * static_cast<size_t>(bmax) * bmax);
  }
  state.alloc(sizeof(float) * 4);  // [0] 2^e, [1] 2^-e of W's operand, [2] running max |W| bits, [3] scale-changed flag
  float* wsc = state.as<float>();
  unsigned* wmax = state.as<unsigned>() + 2;
  unsigned* wchanged = state.as<unsigned>() + 3;
  c.span_begin(PH_OTHER);
  KS_CUDA(cudaMemsetAsync(Wall.p, 0, Wall.bytes, S1));
  KS_CUDA(cudaMemsetAsync(wop_hi.p, 0, wop_hi.bytes, S1));
  KS_CUDA(cudaMemsetAsync(wop_lo.p, 0, wop_lo.bytes, S1));
  KS_CUDA(cudaMemsetAsync(state.p, 0, state.bytes, S1));
  set_unit_scale_kernel<<<1, 1, 0, S1>>>(wsc);
  RowOps A;  // row side of the generation: this rank's training rows
  prep_rows(c, K, K.xs.as<float>() + row_off * K.ld, K.ld, n_loc, false, A, S1);
  c.launches += 1;
  c.span_end();
  KS_CUDA(cudaEventRecord(ev_init, S1));
  KS_CUDA(cudaStreamWaitEvent(ST, ev_init, 0));
  KS_CUDA(cudaStreamWaitEvent(SF, ev_init, 0));

  std::vector<cudaEvent_t> ev_c(T), ev_fact(T), ev_packed(T);
  for (int t = 0; t < T; ++t) {
    ev_c[t] = new_event();
    ev_fact[t] = new_event();
    ev_packed[t] = new_event();
  }
  std::vector<int> first_step(nb, -1);
  int info_slot = 0;
  double flops = 0, gen_flops = 0;
  const int64_t x2_chunk = c.split_chunk_rows;

  // ---- factor(t): K_BB + lambda I in fp64 and its Cholesky, on SF (independent of W)
  auto do_factor = [&](int t) {
    const int j = steps[t];
    int64_t c0;
    const int b = block(j, &c0);
    if (cache_factors && first_step[j] >= 0) return;  // ev_fact of the first visit stands for this one
    first_step[j] = t;
    double* H;
    if (cache_factors) {
      factors[j] = std::make_unique<DevBuf>();
      factors[j]->alloc(sizeof(double) * static_cast<size_t>(b) * b);
      H = factors[j]->as<double>();
    } else {
      H = Hbuf[t % 2].as<double>();
      if (t >= 2) KS_CUDA(cudaStreamWaitEvent(SF, ev_packed[t - 2], 0));  // the solve of step t - 2 read this buffer
    }
    c.span_begin(PH_SOLVE, SF);
    const unsigned tiles = static_cast<unsigned>((b + 63) / 64);
    kbb_kernel<<<dim3(tiles, tiles), 256, 0, SF>>>(K.xs.as<float>() + c0 * K.ld, K.ld, static_cast<int>(K.d), b, K.gamma, lam, H);
    c.launches += 1;
    c.potrf(H, b, info_slot++, SF);
    c.span_end(SF);
    KS_CUDA(cudaEventRecord(ev_fact[t], SF));
    flops += 2.0 * b * static_cast<double>(b) * K.d + static_cast<double>(b) * b * b / 3.0;
  };
  auto fact_event = [&](int t) { return ev_fact[cache_factors ? first_step[steps[t]] : t]; };
  auto factor_of = [&](int t) { return cache_factors ? factors[steps[t]]->as<double>() : Hbuf[t % 2].as<double>(); };
  // ---- gen(t): the kernel block K(local rows, block rows) as an fp16 pair, on ST
  auto do_gen = [&](int t) {
    const int j = steps[t];
    int64_t c0;
    const int b = block(j, &c0);
    c.span_begin(PH_FEATURIZE, ST);
    gen_rbf(c, K, A, 0, n_loc, c0, b, slab_hi[t % 2].p, slab_lo[t % 2].p, lds, ST);
    c.span_end(ST);
    const double f = 6.0 * static_cast<double>(n_loc) * K.d * b;  // three products of depth d
    gen_flops += f;
    flops += f;
  };
  // ---- cgram(t): C = K_B^T W (split Gram, C tiles only) and the label fold, on ST after the operand of step t - 1 is packed
  auto do_cgram = [&](int t) {
    const int j = steps[t];
    int64_t c0;
    const int b = block(j, &c0);
    if (t > 0) KS_CUDA(cudaStreamWaitEvent(ST, ev_packed[t - 1], 0));
    c.span_begin(PH_GRAM, ST);
    KS_CUDA(cudaMemsetAsync(cm.p, 0, cm.bytes, ST));
    launch_gram_block(c, slab_hi[t % 2].p, lds, n_loc, b, wop_hi.p, kpad, k, nullptr, 0, cm.as<float>(), ldc, false, true, ST, true,
                      x2_chunk, slab_lo[t % 2].p, wop_lo.p);
    const int64_t f0 = std::max(c0, row_off), f1 = std::min(c0 + b, row_off + n_loc);
    if (f1 > f0) {
      fold_labels_kernel<<<krr_grid((f1 - f0) * k), 256, 0, ST>>>(cm.as<float>(), ldc, Y.d, Y.ld, k, f0 - c0, f1 - f0, f0 - row_off, wsc);
      c.launches += 1;
    }
    c.span_end(ST);
    KS_CUDA(cudaEventRecord(ev_c[t], ST));
    flops += 6.0 * static_cast<double>(n_loc) * b * k;
  };
  // ---- solve(t): all-reduce of C - Y_B, rhs, triangular solves, W_B += dW, W's scale, operand re-pack, on SS
  auto do_solve = [&](int t) {
    const int j = steps[t];
    int64_t c0;
    const int b = block(j, &c0);
    double* Wb = Wall.as<double>() + c0 * k;
    KS_CUDA(cudaStreamWaitEvent(SS, ev_c[t], 0));
    c.span_begin(PH_ALLREDUCE, SS);
    c.allreduce_f32(cm.as<float>(), static_cast<size_t>(b) * ldc);
    c.span_end(SS);
    KS_CUDA(cudaStreamWaitEvent(SS, fact_event(t), 0));
    c.span_begin(PH_SOLVE, SS);
    krr_rhs_kernel<<<krr_grid(static_cast<int64_t>(b) * k), 256, 0, SS>>>(cm.as<float>(), ldc, wsc, lam, Wb, rhs.as<double>(), b, k);
    c.launches += 1;
    c.potrs(factor_of(t), b, rhs.as<double>(), k, info_slot++, SS);
    c.span_end(SS);
    c.span_begin(PH_UPDATE, SS);
    add_f64_kernel<<<krr_grid(static_cast<int64_t>(b) * k), 256, 0, SS>>>(Wb, rhs.as<double>(), static_cast<int64_t>(b) * k);
    launch_max_abs_f64(Wb, static_cast<int64_t>(b) * k, wmax, SS);
    w_scale_kernel<<<1, 1, 0, SS>>>(wmax, wsc, wchanged);
    pack_wop_kernel<<<krr_grid(n_loc * kpad), 256, 0, SS>>>(Wall.as<double>(), n, bs, k, static_cast<int>(kpad), row_off, n_loc, c0, b,
                                                            wsc, wchanged, wop_hi.as<__half>(), wop_lo.as<__half>());
    c.launches += 4;
    c.span_end(SS);
    KS_CUDA(cudaEventRecord(ev_packed[t], SS));
    flops += 2.0 * static_cast<double>(b) * b * k;
    if (t >= T - nb) {  // last epoch: W_j is final; copy it into the model and its pinned host mirror while the fit goes on
      KS_CUDA(cudaStreamWaitEvent(S5, ev_packed[t], 0));
      KS_CUDA(cudaMemcpyAsync(model->W[j]->p, Wb, sizeof(double) * static_cast<size_t>(b) * k, cudaMemcpyDeviceToDevice, S5));
      model_block_to_host(*model, j, S5);
    }
  };

  // Enqueue order (a wait on an event not yet recorded counts as complete, so every record precedes its waits):
  //   ST: gen(0) | C(0) gen(1) | C(1) gen(2) | ...   -- gen(t + 1) runs while the chain of step t solves on SS
  //   SF: factor(0) factor(1) ... one step ahead of the solve that needs it
  do_factor(0);
  do_gen(0);
  for (int t = 0; t < T; ++t) {
    if (t + 1 < T) do_factor(t + 1);
    do_cgram(t);
    if (t + 1 < T) do_gen(t + 1);
    do_solve(t);
  }
  KS_CUDA(cudaStreamWaitEvent(S1, ev_packed[T - 1], 0));
  cudaEvent_t ev_copy = new_event();
  KS_CUDA(cudaEventRecord(ev_copy, S5));
  KS_CUDA(cudaStreamWaitEvent(S1, ev_copy, 0));
  KS_CUDA(cudaEventRecord(ev1, S1));
  c.check_async("KernelRidgeRegression.fit");
  c.check_infos(info_slot);
  float total_ms = 0;
  cudaEventElapsedTime(&total_ms, ev0, ev1);
  double ms[PH_COUNT];
  c.collect_spans(ms);
  for (cudaEvent_t e : c.fit_events) c.event_pool.push_back(e);
  c.fit_events.clear();
  std::ostringstream js;
  js << "{\"solver\":\"krr\",\"n_local\":" << n_loc << ",\"n_total\":" << n << ",\"d\":" << K.d << ",\"k\":" << k
     << ",\"block_size\":" << bs << ",\"num_blocks\":" << nb << ",\"num_epochs\":" << epochs << ",\"world\":" << c.world
     << ",\"total_ms\":" << total_ms << ",\"generate_ms\":" << ms[PH_FEATURIZE] << ",\"gram_ms\":" << ms[PH_GRAM]
     << ",\"allreduce_ms\":" << ms[PH_ALLREDUCE] << ",\"solve_ms\":" << ms[PH_SOLVE] << ",\"update_ms\":" << ms[PH_UPDATE]
     << ",\"other_ms\":" << ms[PH_OTHER] << ",\"local_flops\":" << flops << ",\"generate_mma_flops\":" << gen_flops
     << ",\"launches\":" << (c.launches - launches0) << ",\"mma\":\"f16x2\",\"solve\":\"potrs\",\"cached_factors\":"
     << (cache_factors ? 1 : 0) << ",\"host_mirror\":" << (model->host_valid ? 1 : 0) << ",\"host_ms\":"
     << std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count() << "}";
  c.stats_json = js.str();
  return c.add(std::move(model));
}

// ------------------------------------------------------------------------------------ KernelBlockLinearMapper.apply
// sum_j K(x, X_j) W_j: per block the generated slab, then one split update out += 0 - S (2^e W_j) (-2^-e)
std::unique_ptr<Matrix> kernel_model_apply(Ctx& c, Model& md, Matrix& x) {
  const GaussKernel& K = *md.kernel;
  if (x.cols != K.d) throw KsError{KS_ERR_INVALID, "input rows have a different column count than the kernel model's training rows"};
  cudaStream_t st = c.st;
  const int k = static_cast<int>(md.k);
  const int64_t n_t = x.rows;
  auto out = new_matrix(n_t, k);
  KS_CUDA(cudaMemsetAsync(out->d, 0, out->buf.bytes, st));
  RowOps A;
  prep_rows(c, K, x.d, x.ld, n_t, true, A, st);
  int bmax = 1;
  for (auto r : md.brows) bmax = std::max<int>(bmax, static_cast<int>(r));
  const int64_t lds = round_up(bmax, 32), kpad = round_up(k, 32);
  DevBuf hi, lo, bop, bop_lo, wsc;
  hi.alloc(2 * static_cast<size_t>(std::max<int64_t>(n_t, 1) * lds));
  lo.alloc(hi.bytes);
  bop.alloc(2 * static_cast<size_t>(kpad * lds));
  bop_lo.alloc(bop.bytes);
  wsc.alloc(sizeof(float) * 4);  // [0] 2^e, [1] 2^-e, [2] -2^-e, [3] max |W_j| bits
  unsigned* mb = wsc.as<unsigned>() + 3;
  int64_t c0 = 0;
  for (size_t j = 0; j < md.brows.size(); ++j) {
    const int b = static_cast<int>(md.brows[j]);
    gen_rbf(c, K, A, 0, n_t, c0, b, hi.p, lo.p, lds, st);
    KS_CUDA(cudaMemsetAsync(mb, 0, sizeof(unsigned), st));
    launch_max_abs_f64(md.W[j]->as<double>(), static_cast<int64_t>(b) * k, mb, st);
    launch_pow2_scale(mb, 4096.f, wsc.as<float>(), st);
    neg_inv_scale_kernel<<<1, 1, 0, st>>>(wsc.as<float>());
    launch_pack_update16(md.W[j]->as<double>(), nullptr, nullptr, bop.p, static_cast<int>(lds), nullptr, b, k, static_cast<int>(kpad),
                         wsc.as<float>(), st, bop_lo.p);
    c.launches += 4;
    launch_update(c, hi.p, lds, n_t, b, bop.p, lds, k, out->d, out->ld, nullptr, EPI_UPDATE, /*reduce=*/true, st, true,
                  wsc.as<float>() + 2, lo.p, bop_lo.p);
    c0 += b;
  }
  c.check_async("KernelBlockLinearMapper.apply");
  return out;
}

// ------------------------------------------------------------------------------------ new KernelBlockLinearMapper(xs, ...)
int64_t kernel_model_from_host(Ctx& c, const std::shared_ptr<GaussKernel>& Kp, const double* const* xs, const int64_t* block_rows,
                               int32_t n_blocks, int64_t k, int32_t block_size) {
  if (!xs || !block_rows || n_blocks <= 0 || k <= 0 || block_size <= 0) throw KsError{KS_ERR_INVALID, "bad model arguments"};
  int64_t sum = 0;
  for (int j = 0; j < n_blocks; ++j) {
    if (block_rows[j] <= 0 || block_rows[j] > block_size) throw KsError{KS_ERR_INVALID, "block_rows out of range"};
    if (!xs[j]) throw KsError{KS_ERR_INVALID, "null model block"};
    sum += block_rows[j];
  }
  if (sum != Kp->n) throw KsError{KS_ERR_INVALID, "block rows do not sum to the kernel's training row count"};
  auto m = std::make_unique<Model>();
  m->kernel = Kp;
  m->block_size = block_size;
  m->k = k;
  for (int j = 0; j < n_blocks; ++j) {
    auto W = std::make_unique<DevBuf>();
    W->alloc(sizeof(double) * static_cast<size_t>(block_rows[j] * k));
    KS_CUDA(cudaMemcpyAsync(W->p, xs[j], sizeof(double) * block_rows[j] * k, cudaMemcpyHostToDevice, c.st));
    m->W.push_back(std::move(W));
    m->brows.push_back(block_rows[j]);
  }
  m->intercept.alloc(sizeof(double) * static_cast<size_t>(k));
  KS_CUDA(cudaStreamSynchronize(c.st));
  return c.add(std::move(m));
}

}  // namespace ks
