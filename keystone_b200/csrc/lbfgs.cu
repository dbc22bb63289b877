// Dense L-BFGS least squares on the device: DenseLBFGSwithL2 with LeastSquaresDenseGradient
// (K/nodes/learning/LBFGS.scala:14-192, K/nodes/learning/Gradient.scala:29-53).  DESIGN.md section 14.
//
//   f(W) = |A_c W - Y_c|_F^2 / (2N) + lambda/2 |W|_F^2,   g = A_c^T (A_c W - Y_c) / N + lambda W,   W_0 = 0
//
// Every iteration runs two products over the feature source, block by block (the slab of a block is produced again for each:
// generated features are never stored):
//   Q = A_c P     K-major update GEMM (P packed per feature block like the block solver's dW)
//   C = A_c^T R   Gram kernel, C strip only, after R += alpha Q
// The residual is kept with the block solver's sign, R = Y_c - A_c W (so its products are the block solver's), and Q holds
// -A_c P as the update epilogue produces it; both signs are folded into the fp64 kernels below.
// The step is the exact minimiser along P, alpha = -<g, P> / (|A_c P|^2 / N + lambda |P|^2).  The two-loop recursion, alpha,
// W, the history and the stop test run in fp64 on the device after the one all-reduce of C.  Every fp64 reduction of the
// iteration (dot products, norms, |Q|^2, |R|^2 and R's column sums) has a fixed grid and a fixed summation order, and every
// rank reads the same all-reduced inputs, so every rank computes the same bits and the models are bit-identical.  Not ordered:
// the split-K reduce-add of the tensor-core products and the column sums of the mean passes, as in the block solver, so one
// rank's fit repeats only up to rounding from run to run.
#include "engine.h"
#include "operand_split.cuh"

#include <cuda_fp16.h>
#include <math.h>

#include <algorithm>
#include <chrono>
#include <deque>
#include <sstream>

namespace ks {

static constexpr int kRedBlocks = 264;  // grid of every fp64 reduction below: partial sums per block, then summed in block order
static constexpr int kRedThreads = 256;

// block-wide sum (op 0) or max (op 1) of a per-thread value; the result is valid in thread 0
__device__ double lb_block_reduce(double v, int op) {
  __shared__ double red[kRedThreads];
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] = op == 0 ? red[threadIdx.x] + red[threadIdx.x + s] : fmax(red[threadIdx.x], red[threadIdx.x + s]);
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

// term = mul * (coef ? *coef : 1) * v[i]  (v null: 0)
struct LbTerm {
  const double* v = nullptr;
  const double* coef = nullptr;
  double mul = 1.0;
};
__device__ __forceinline__ double lb_term(const LbTerm& t, double c, int64_t i) { return t.v ? t.mul * c * t.v[i] : 0.0; }

// x[i] = (gscale ? *gscale : 1) * (t0 + t1); out[i] = x[i] (out may alias t0.v); part[d * kRedBlocks + block] += w_d[i] x[i]
// for d < ndots (w_d null: x itself)
__global__ void __launch_bounds__(kRedThreads) lb_lin_dot_kernel(double* out, LbTerm t0, LbTerm t1, const double* gscale, int ndots,
                                                                 const double* w0, const double* w1, int64_t n, double* part) {
  const double c0 = t0.coef ? *t0.coef : 1.0, c1 = t1.coef ? *t1.coef : 1.0, gs = gscale ? *gscale : 1.0;
  double a0 = 0.0, a1 = 0.0;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const double x = gs * (lb_term(t0, c0, i) + lb_term(t1, c1, i));
    if (out) out[i] = x;
    if (ndots > 0) a0 = fma(w0 ? w0[i] : x, x, a0);
    if (ndots > 1) a1 = fma(w1 ? w1[i] : x, x, a1);
  }
  if (ndots > 0) {
    const double s = lb_block_reduce(a0, 0);
    if (threadIdx.x == 0) part[blockIdx.x] = s;
  }
  if (ndots > 1) {
    const double s = lb_block_reduce(a1, 0);
    if (threadIdx.x == 0) part[kRedBlocks + blockIdx.x] = s;
  }
}

// dst = (base ? *base : 0) + mul * (scale ? *scale : 1) * reduce(part[0 .. nparts)), op 0 sum / 1 max, in a fixed order
__global__ void __launch_bounds__(kRedThreads) lb_finish_kernel(const double* part, int nparts, int op, double* dst, const double* base,
                                                                const double* scale, double mul) {
  double a = 0.0;
  for (int i = threadIdx.x; i < nparts; i += blockDim.x) a = op == 0 ? a + part[i] : fmax(a, part[i]);
  const double s = lb_block_reduce(a, op);
  if (threadIdx.x == 0) *dst = (base ? *base : 0.0) + mul * (scale ? *scale : 1.0) * s;
}

// Scalar slots of the fit (fp64, device).  The host reads [0, kScHost) once per iteration for the stop decision.
enum {
  SC_LOSS = 0, SC_GMAX, SC_SY, SC_RESET, SC_CURV, SC_YY, kScHost,
  SC_GG = kScHost, SC_GP, SC_PP, SC_QQ, SC_WW, SC_ALPHA, SC_GAMMA,
  SC_HIST  // then per history slot: a, coef, rho
};

// After the direction: if <g, P> >= 0 (not a descent direction after rounding) P = -g; the history is dropped by the host
__global__ void lb_fallback_kernel(double* P, const double* g, int64_t n, const double* sc) {
  if (!(sc[SC_GP] >= 0.0)) return;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    P[i] = -g[i];
}
__global__ void lb_fallback_scalars_kernel(double* sc) {
  sc[SC_RESET] = 0.0;
  if (sc[SC_GP] >= 0.0) {
    sc[SC_RESET] = 1.0;
    sc[SC_GP] = -sc[SC_GG];
    sc[SC_PP] = sc[SC_GG];
  }
}
// the exact minimiser along P: alpha = -<g, P> / (|A_c P|^2 / N + lambda |P|^2); a curvature that is not > 0 stops the fit
__global__ void lb_alpha_kernel(double* sc, double inv_n, double lam) {
  const double den = sc[SC_QQ] * inv_n + lam * sc[SC_PP];
  if (den > 0.0 && isfinite(den)) {
    sc[SC_ALPHA] = -sc[SC_GP] / den;
    sc[SC_CURV] = 0.0;
  } else {
    sc[SC_ALPHA] = 0.0;
    sc[SC_CURV] = 1.0;
  }
}
// loss of the new iterate, rho and gamma of the new pair (slot h)
__global__ void lb_end_kernel(double* sc, const double* rr, double inv_n, double lam, int h) {
  sc[SC_LOSS] = 0.5 * (*rr) * inv_n + 0.5 * lam * sc[SC_WW];
  if (h < 0) return;
  const double sy = sc[SC_SY], yy = sc[SC_YY];
  sc[SC_HIST + 3 * h + 2] = sy > 0.0 ? 1.0 / sy : 0.0;
  sc[SC_GAMMA] = yy > 0.0 ? sy / yy : 1.0;
}

// g_new = -(C cs - delta rsum) / N + lambda W over the blocked flat layout (block j: features [j bs, j bs + b_j), column-major
// b_j x k at offset j bs k); C is row-major D x ldc (feature, class).  y = g_new - g_old and s . y, y . y when y is given.
// part: [0] |g|^2, [1] s . y, [2] y . y, [3] max |g|
__global__ void __launch_bounds__(kRedThreads) lb_gradient_kernel(const float* __restrict__ C, int64_t ldc, const double* __restrict__ delta,
                                                                  const double* __restrict__ rsum, const float* __restrict__ c_scale,
                                                                  const double* __restrict__ W, double* g, double* y,
                                                                  const double* __restrict__ s, double inv_n, double lam, int64_t D,
                                                                  int k, int bs, int64_t n, double* part) {
  const double cs = c_scale ? static_cast<double>(*c_scale) : 1.0;
  const int64_t blk = static_cast<int64_t>(bs) * k;
  double gg = 0.0, sy = 0.0, yy = 0.0, gm = 0.0;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t j = i / blk, r = i - j * blk;
    const int64_t bj = min(static_cast<int64_t>(bs), D - j * bs);
    const int64_t c = r / bj, f = j * bs + (r - c * bj);
    double v = static_cast<double>(C[f * ldc + c]) * cs;
    if (delta) v -= delta[f] * rsum[c];
    const double gn = -v * inv_n + lam * W[i];
    if (y) {
      const double yi = gn - g[i];
      y[i] = yi;
      sy = fma(s[i], yi, sy);
      yy = fma(yi, yi, yy);
    }
    g[i] = gn;
    gg = fma(gn, gn, gg);
    gm = fmax(gm, fabs(gn));
  }
  double t = lb_block_reduce(gg, 0);
  if (threadIdx.x == 0) part[blockIdx.x] = t;
  t = lb_block_reduce(sy, 0);
  if (threadIdx.x == 0) part[kRedBlocks + blockIdx.x] = t;
  t = lb_block_reduce(yy, 0);
  if (threadIdx.x == 0) part[2 * kRedBlocks + blockIdx.x] = t;
  t = lb_block_reduce(gm, 1);
  if (threadIdx.x == 0) part[3 * kRedBlocks + blockIdx.x] = t;
}

// Fused residual step: R[:, :k] += alpha Q (Q null: R unchanged), then the operand of the next C = A^T R product from the new R
// (tf32: tf32_pair(R); F16: f16_hi2 / f16_lo2 of R 2^e; the lo plane only in the parity mode), the column sums of R per CTA row into
// cpart[blockIdx.y * ld + c] and |R|^2 per CTA into part[blockIdx.y * gridDim.x + blockIdx.x]; both are finished in a fixed order.
// Block (32, 8), 4 columns per thread, rows strided by 8: the access pattern of round_colsum_kernel.
template <bool F16>
__global__ void __launch_bounds__(256) lb_residual_kernel(float* __restrict__ R, const float* __restrict__ Q, const double* __restrict__ alpha,
                                                          int64_t ld, int64_t rows, int k, void* __restrict__ op, void* __restrict__ op_lo,
                                                          const float* __restrict__ scale, double* __restrict__ cpart,
                                                          double* __restrict__ part, unsigned* __restrict__ overflow, int64_t rpb) {
  __shared__ double red[8][128];
  const double a = Q ? *alpha : 0.0;
  const float sc = F16 ? *scale : 1.f;
  const int c4 = (blockIdx.x * 32 + threadIdx.x) * 4;
  const int64_t r_begin = blockIdx.y * rpb, r_end = min(rows, r_begin + rpb);
  double cs[4] = {0, 0, 0, 0}, sq = 0.0;
  if (c4 < ld) {
    for (int64_t r = r_begin + threadIdx.y; r < r_end; r += 8) {
      float4 v4 = *reinterpret_cast<const float4*>(R + r * ld + c4);
      float v[4] = {v4.x, v4.y, v4.z, v4.w};
      if (Q) {
        const float4 q4 = *reinterpret_cast<const float4*>(Q + r * ld + c4);
        const float q[4] = {q4.x, q4.y, q4.z, q4.w};
#pragma unroll
        for (int jj = 0; jj < 4; ++jj)
          if (c4 + jj < k) v[jj] = static_cast<float>(static_cast<double>(v[jj]) + a * static_cast<double>(q[jj]));
        *reinterpret_cast<float4*>(R + r * ld + c4) = make_float4(v[0], v[1], v[2], v[3]);
      }
      float hi[4] = {0.f, 0.f, 0.f, 0.f}, lo[4] = {0.f, 0.f, 0.f, 0.f}, o[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        if (c4 + jj >= k) continue;
        cs[jj] += v[jj];
        sq = fma(static_cast<double>(v[jj]), static_cast<double>(v[jj]), sq);
        if (F16) {
          o[jj] = v[jj] * sc;
          if (!(fabsf(o[jj]) <= 65504.f)) *overflow = 1u;  // the fit's residual scale was fixed from max|R_0|
        } else {
          tf32_pair(v[jj], hi[jj], lo[jj]);
        }
      }
      if (F16) {
        const __half2 h0 = f16_hi2(o[0], o[1]), h1 = f16_hi2(o[2], o[3]);
        uint2 pk;
        pk.x = *reinterpret_cast<const unsigned*>(&h0);
        pk.y = *reinterpret_cast<const unsigned*>(&h1);
        *reinterpret_cast<uint2*>(static_cast<__half*>(op) + r * ld + c4) = pk;
        if (op_lo) {
          const __half2 l0 = f16_lo2(o[0], o[1], h0), l1 = f16_lo2(o[2], o[3], h1);
          pk.x = *reinterpret_cast<const unsigned*>(&l0);
          pk.y = *reinterpret_cast<const unsigned*>(&l1);
          *reinterpret_cast<uint2*>(static_cast<__half*>(op_lo) + r * ld + c4) = pk;
        }
      } else {
        *reinterpret_cast<float4*>(static_cast<float*>(op) + r * ld + c4) = make_float4(hi[0], hi[1], hi[2], hi[3]);
        if (op_lo) *reinterpret_cast<float4*>(static_cast<float*>(op_lo) + r * ld + c4) = make_float4(lo[0], lo[1], lo[2], lo[3]);
      }
    }
  }
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) red[threadIdx.y][threadIdx.x * 4 + jj] = cs[jj];
  __syncthreads();
  const int t = threadIdx.y * 32 + threadIdx.x;
  if (t < 128) {
    double s = 0;
#pragma unroll
    for (int yy = 0; yy < 8; ++yy) s += red[yy][t];
    const int c = blockIdx.x * 128 + t;
    if (c < ld) cpart[blockIdx.y * ld + c] = s;
  }
  __syncthreads();
  // |R|^2 of this CTA: threads in a fixed order
  double* flat = &red[0][0];
  flat[t] = sq;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (t < s) flat[t] += flat[t + s];
    __syncthreads();
  }
  if (t == 0) part[blockIdx.y * gridDim.x + blockIdx.x] = flat[0];
}
// rsum[c] = sum over the CTA rows q of cpart[q * ld + c], in row order
__global__ void lb_colsum_finish_kernel(const double* __restrict__ cpart, int nrows, int64_t ld, int k, double* __restrict__ rsum) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= k) return;
  double s = 0.0;
  for (int q = 0; q < nrows; ++q) s += cpart[q * ld + c];
  rsum[c] = s;
}

// |Q[:, :k]|^2 per CTA into part[block] (fixed grid of kRedBlocks CTAs; padding columns of Q are zero)
__global__ void __launch_bounds__(kRedThreads) lb_sumsq_f32_kernel(const float* __restrict__ Q, int64_t total, double* part) {
  double a = 0.0;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const double q = Q[i];
    a = fma(q, q, a);
  }
  const double s = lb_block_reduce(a, 0);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

// materialised features: mean = fsum / N (fp64), shift = fp32(mean), delta = mean - shift
__global__ void lb_mean_shift_kernel(const double* __restrict__ fsum, double inv_n, double* mean, float* shift, double* delta, int64_t D) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= D) return;
  const double m = fsum[i] * inv_n;
  const float s = static_cast<float>(m);
  mean[i] = m;
  shift[i] = s;
  delta[i] = m - static_cast<double>(s);
}

// ------------------------------------------------------------------------------------ the fit
int64_t fit_lbfgs(Ctx& c, FeatSrc& src, Matrix& Y, bool fit_intercept, int m, double tol, int num_iter, double lam, int precision) {
  if (m < 1) throw KsError{KS_ERR_INVALID, "numCorrections must be >= 1"};
  if (num_iter < 1) throw KsError{KS_ERR_INVALID, "numIterations must be >= 1"};
  if (!(lam >= 0.0) || !std::isfinite(lam)) throw KsError{KS_ERR_INVALID, "regParam must be finite and >= 0"};
  if (!(tol >= 0.0) || !std::isfinite(tol)) throw KsError{KS_ERR_INVALID, "convergenceTol must be finite and >= 0"};
  if (Y.rows != src.n_rows) throw KsError{KS_ERR_INVALID, "features and labels have different row counts"};
  const int64_t n_loc = Y.rows, D = src.D;
  const int k = static_cast<int>(Y.cols);
  if (D <= 0 || k <= 0) throw KsError{KS_ERR_INVALID, "empty problem"};
  const int bs = static_cast<int>(std::min<int64_t>(D, 4096));  // feature block of the two products (columns per slab)
  const int nb = static_cast<int>((D + bs - 1) / bs);
  const int64_t lds = round_up(bs, 32), kpad = round_up(k, 32);
  const int64_t n = D * k;  // length of W, g, P and every history vector (blocked layout)
  cudaStream_t st = c.st;
  const auto host_t0 = std::chrono::steady_clock::now();
  c.spans.clear();
  const int64_t launches0 = c.launches;
  double flops = 0;
  cudaEvent_t ev0 = c.get_event(), ev1 = c.get_event();
  c.fit_events.push_back(ev0);
  c.fit_events.push_back(ev1);
  KS_CUDA(cudaEventRecord(ev0, st));

  // operand modes: the block solver's (engine.cu fit_blockls)
  const bool x2 = precision == KS_PRECISION_F16X2 && (src.F || src.proj_x2);
  const bool f16 = !src.F && src.kind == 0 && (precision == KS_PRECISION_F16 || x2);
  const size_t es = f16 ? 2 : 4;
  const int64_t x2_chunk = c.split_chunk_rows;

  // ---- label mean + global row count
  c.span_begin(PH_OTHER);
  DevBuf ysum;
  ysum.alloc(sizeof(double) * (k + 1));
  KS_CUDA(cudaMemsetAsync(ysum.p, 0, ysum.bytes, st));
  if (fit_intercept) {
    launch_colsum(Y.d, nullptr, Y.ld, n_loc, k, ysum.as<double>(), st);
    c.launches += 1;
  }
  launch_set_f64(ysum.as<double>() + k, static_cast<double>(n_loc), st);
  c.launches += 1;
  c.allreduce_f64(ysum.as<double>(), k + 1);
  double n_total = 0;
  KS_CUDA(cudaMemcpyAsync(&n_total, ysum.as<double>() + k, sizeof(double), cudaMemcpyDeviceToHost, st));
  KS_CUDA(cudaStreamSynchronize(st));
  if (n_total < 1) throw KsError{KS_ERR_INVALID, "no training rows"};
  const double inv_n = 1.0 / n_total;

  // ---- workspace (every buffer from the pool; an exception returns all of it, the model is only created at the end)
  DevBuf ymean, W, g, P, hist, sc, part, rpart, cpart, Cbuf, red64, shift, delta, mean, fsum, R, Q, r_op, r_lo, scales, samp;
  DevBuf slab, slab_lo, sf32, bop, bop_lo, cbias;
  ymean.alloc(sizeof(double) * k);
  launch_scale_f64(ysum.as<double>(), inv_n, nullptr, ymean.as<double>(), k, st);
  c.launches += 1;
  W.alloc(sizeof(double) * n);
  g.alloc(sizeof(double) * n);
  P.alloc(sizeof(double) * n);
  hist.alloc(sizeof(double) * 2 * static_cast<size_t>(m) * n);  // S slots [0, m), Y slots [m, 2m)
  auto S_slot = [&](int h) { return hist.as<double>() + static_cast<size_t>(h) * n; };
  auto Y_slot = [&](int h) { return hist.as<double>() + static_cast<size_t>(m + h) * n; };
  sc.alloc(sizeof(double) * (SC_HIST + 3 * m));
  part.alloc(sizeof(double) * 4 * kRedBlocks);
  const int64_t rpb = 1024;
  const int res_gx = static_cast<int>((kpad + 127) / 128), res_gy = static_cast<int>((std::max<int64_t>(n_loc, 1) + rpb - 1) / rpb);
  rpart.alloc(sizeof(double) * static_cast<size_t>(res_gx) * res_gy);
  cpart.alloc(sizeof(double) * static_cast<size_t>(res_gy) * kpad);
  Cbuf.alloc(sizeof(float) * static_cast<size_t>(D * kpad + round_up(D, 32)));  // C (D x kpad), then the slab column sums (D)
  float* Cm = Cbuf.as<float>();
  float* ssum = Cm + D * kpad;
  red64.alloc(sizeof(double) * (k + 1));  // column sums of R, then |R|^2
  shift.alloc(sizeof(float) * round_up(D, 32));
  mean.alloc(sizeof(double) * D);
  delta.alloc(sizeof(double) * D);
  R.alloc(sizeof(float) * static_cast<size_t>(std::max<int64_t>(n_loc, 1) * kpad));
  Q.alloc(R.bytes);
  r_op.alloc(f16 ? R.bytes / 2 : R.bytes);
  if (x2) r_lo.alloc(r_op.bytes);
  slab.alloc(es * static_cast<size_t>(std::max<int64_t>(n_loc, 1) * lds));
  if (x2) slab_lo.alloc(slab.bytes);
  if (x2 && !src.F && !f16) sf32.alloc(sizeof(float) * static_cast<size_t>(std::max<int64_t>(n_loc, 1) * lds));
  bop.alloc(es * static_cast<size_t>(nb) * kpad * lds);  // P^T packed per feature block
  if (x2) bop_lo.alloc(bop.bytes);
  cbias.alloc(sizeof(float) * static_cast<size_t>(nb) * kpad);
  scales.alloc(sizeof(float) * 8);  // [0] max|R0| bits, [1] max|P| bits, [2,3] residual {2^e, 2^-e}, [4,5] P {2^e, 2^-e}, [6] overflow
  unsigned* maxbits = scales.as<unsigned>();
  const float* rscale = scales.as<float>() + 2;
  float* pscale = scales.as<float>() + 4;
  KS_CUDA(cudaMemsetAsync(W.p, 0, W.bytes, st));
  KS_CUDA(cudaMemsetAsync(sc.p, 0, sc.bytes, st));
  KS_CUDA(cudaMemsetAsync(shift.p, 0, shift.bytes, st));
  KS_CUDA(cudaMemsetAsync(mean.p, 0, mean.bytes, st));
  KS_CUDA(cudaMemsetAsync(delta.p, 0, delta.bytes, st));
  KS_CUDA(cudaMemsetAsync(scales.p, 0, scales.bytes, st));
  launch_init_residual(Y.d, Y.ld, ymean.as<double>(), R.as<float>(), kpad, n_loc, k, st);  // R_0 = Y - ybar (W_0 = 0)
  c.launches += 1;
  if (f16) {  // one power-of-two scale of R for the whole fit, from max|R_0| with 16x headroom (the block solver's rule)
    launch_max_abs_f32(R.as<float>(), kpad, n_loc, k, maxbits, st);
    c.allreduce_max_u32(maxbits, 1);
    launch_pow2_scale(maxbits, 4096.f, scales.as<float>() + 2, st);
    c.launches += 2;
  }
  c.span_end();

  auto block_cols = [&](int j, int64_t* c0) {
    *c0 = static_cast<int64_t>(j) * bs;
    return static_cast<int>(std::min<int64_t>(D, *c0 + bs) - *c0);
  };
  // slab of feature block j over rows [0, rows): S = features - shift (tf32 / fp16 / pairs), column sums of S into cs (fp32)
  auto make_slab = [&](int j, int64_t rows, float* cs, bool sample) {
    int64_t c0;
    const int b = block_cols(j, &c0);
    const float* sh = sample ? src.zeros.as<float>() : shift.as<float>() + c0;
    c.span_begin(PH_FEATURIZE);
    if (x2 && src.F) {
      launch_center_round(src.F->d, src.F->ld, static_cast<int>(c0), sh, slab.as<float>(), cs, lds, rows, b, st, slab_lo.as<float>());
      c.launches += 1;
    } else if (x2 && f16) {
      produce_slab(c, src, c0, b, sh, slab.p, lds, 0, rows, /*round_out=*/false, cs, st, false, true, slab_lo.p);
      flops += 4.0 * static_cast<double>(rows) * src.d_in * b;
    } else if (x2) {
      produce_slab(c, src, c0, b, sh, sf32.p, lds, 0, rows, /*round_out=*/false, nullptr, st, false, true);
      launch_center_round(sf32.as<float>(), lds, 0, src.zeros.as<float>(), slab.as<float>(), cs, lds, rows, b, st, slab_lo.as<float>());
      c.launches += 1;
      flops += 4.0 * static_cast<double>(rows) * src.d_in * b;
    } else {
      produce_slab(c, src, c0, b, sh, slab.p, lds, 0, rows, /*round_out=*/!sample, cs, st, f16);
    }
    if (!src.F) flops += 2.0 * static_cast<double>(rows) * src.d_in * b;
    c.span_end();
  };

  // ---- feature means: exact for materialised features (one fp64 pass over F), a row-sample estimate for generated ones whose
  // error is measured by the column sums of the first full pass (delta) and corrected in every product, as in the block solver
  const bool gen_mean = fit_intercept && !src.F;
  if (fit_intercept && src.F) {
    c.span_begin(PH_FEATURIZE);
    fsum.alloc(sizeof(double) * static_cast<size_t>(src.F->ld));
    KS_CUDA(cudaMemsetAsync(fsum.p, 0, fsum.bytes, st));
    launch_colsum(src.F->d, nullptr, src.F->ld, n_loc, static_cast<int>(D), fsum.as<double>(), st);
    c.allreduce_f64(fsum.as<double>(), static_cast<size_t>(D));
    lb_mean_shift_kernel<<<static_cast<unsigned>((D + 255) / 256), 256, 0, st>>>(fsum.as<double>(), inv_n, mean.as<double>(),
                                                                                 shift.as<float>(), delta.as<double>(), D);
    c.launches += 2;
    c.span_end();
  } else if (gen_mean) {
    const int64_t ns = std::min<int64_t>(n_loc, c.sample_rows);
    samp.alloc(sizeof(double) * (D + 1));
    KS_CUDA(cudaMemsetAsync(ssum, 0, sizeof(float) * D, st));
    for (int j = 0; j < nb; ++j) {
      int64_t c0;
      block_cols(j, &c0);
      make_slab(j, ns, ssum + c0, /*sample=*/true);
    }
    launch_f32_to_f64_rows(ssum, D, samp.as<double>(), D, 1, D, st);
    launch_set_f64(samp.as<double>() + D, static_cast<double>(ns), st);
    c.allreduce_f64(samp.as<double>(), static_cast<size_t>(D + 1));
    launch_divide_by_count(samp.as<double>(), samp.as<double>() + D, shift.as<float>(), nullptr, static_cast<int>(D), st);
    c.launches += 3;
  }
  const double* dl = fit_intercept ? delta.as<double>() : nullptr;

  // ---- the pieces of an iteration
  auto finish = [&](const double* p, int nparts, int op, int slot, const double* base = nullptr, const double* scale = nullptr,
                    double mul = 1.0) {
    lb_finish_kernel<<<1, kRedThreads, 0, st>>>(p, nparts, op, sc.as<double>() + slot, base, scale, mul);
    c.launches += 1;
  };
  auto lin = [&](double* out, LbTerm t0, LbTerm t1, const double* gscale, int ndots, const double* w0, const double* w1) {
    lb_lin_dot_kernel<<<kRedBlocks, kRedThreads, 0, st>>>(out, t0, t1, gscale, ndots, w0, w1, n, part.as<double>());
    c.launches += 1;
  };
  auto scp = [&](int slot) { return sc.as<double>() + slot; };
  auto a_of = [&](int h) { return SC_HIST + 3 * h; };
  auto cf_of = [&](int h) { return SC_HIST + 3 * h + 1; };
  auto rho_of = [&](int h) { return SC_HIST + 3 * h + 2; };
  // R += alpha Q (Q null: R as it is), the operand of the next A^T R, its column sums and |R|^2 (into red64[k], rank-local)
  auto residual = [&](bool with_q) {
    c.span_begin(PH_OTHER);
    KS_CUDA(cudaMemsetAsync(red64.p, 0, red64.bytes, st));
    const dim3 grid(res_gx, res_gy), blk(32, 8);
    const double* al = scp(SC_ALPHA);
    if (n_loc > 0) {
      if (f16)
        lb_residual_kernel<true><<<grid, blk, 0, st>>>(R.as<float>(), with_q ? Q.as<float>() : nullptr, al, kpad, n_loc, k, r_op.p,
                                                       x2 ? r_lo.p : nullptr, rscale, cpart.as<double>(), rpart.as<double>(),
                                                       maxbits + 6, rpb);
      else
        lb_residual_kernel<false><<<grid, blk, 0, st>>>(R.as<float>(), with_q ? Q.as<float>() : nullptr, al, kpad, n_loc, k, r_op.p,
                                                        x2 ? r_lo.p : nullptr, nullptr, cpart.as<double>(), rpart.as<double>(), nullptr,
                                                        rpb);
      lb_colsum_finish_kernel<<<(k + 127) / 128, 128, 0, st>>>(cpart.as<double>(), res_gy, kpad, k, red64.as<double>());
      lb_finish_kernel<<<1, kRedThreads, 0, st>>>(rpart.as<double>(), res_gx * res_gy, 0, red64.as<double>() + k, nullptr, nullptr, 1.0);
      c.launches += 3;
    }
    c.span_end();
  };
  // C = A_c^T R (all blocks), the slab column sums on request, then the one all-reduce of the iteration
  auto gradient_pass = [&](bool colsums) {
    KS_CUDA(cudaMemsetAsync(Cbuf.p, 0, Cbuf.bytes, st));
    for (int j = 0; j < nb; ++j) {
      int64_t c0;
      const int b = block_cols(j, &c0);
      make_slab(j, n_loc, colsums ? ssum + c0 : nullptr, false);
      c.span_begin(PH_GRAM);
      float* Cj = Cm + c0 * kpad;
      if (x2 && f16) {
        launch_gram_block(c, slab.p, lds, n_loc, b, r_op.p, kpad, k, nullptr, 0, Cj, static_cast<int>(kpad), false, true, st, true,
                          x2_chunk, slab_lo.p, r_lo.p);
        flops += 4.0 * n_loc * static_cast<double>(b) * k;
      } else {
        launch_gram_block(c, slab.p, lds, n_loc, b, r_op.p, kpad, k, nullptr, 0, Cj, static_cast<int>(kpad), false, true, st, f16,
                          x2 ? x2_chunk : 0);
      }
      if (x2 && !f16) {  // + S_lo^T R_hi + S_hi^T R_lo
        launch_gram_block(c, slab_lo.p, lds, n_loc, b, r_op.p, kpad, k, nullptr, 0, Cj, static_cast<int>(kpad), false, true, st, false,
                          x2_chunk);
        launch_gram_block(c, slab.p, lds, n_loc, b, r_lo.p, kpad, k, nullptr, 0, Cj, static_cast<int>(kpad), false, true, st, false,
                          x2_chunk);
        flops += 4.0 * n_loc * static_cast<double>(b) * k;
      }
      flops += 2.0 * n_loc * static_cast<double>(b) * k;
      c.span_end();
    }
    c.span_begin(PH_ALLREDUCE);
    c.allreduce_f32(Cm, static_cast<size_t>(D * kpad + (colsums ? D : 0)));
    c.allreduce_f64(red64.as<double>(), static_cast<size_t>(k + 1));
    c.span_end();
  };
  // g = A_c^T (A_c W - Y_c) / N + lambda W; with slot h >= 0 also y_h = g_new - g_old, s_h . y_h, y_h . y_h
  auto new_gradient = [&](int h) {
    c.span_begin(PH_SOLVE);
    lb_gradient_kernel<<<kRedBlocks, kRedThreads, 0, st>>>(Cm, kpad, dl, red64.as<double>(), f16 ? rscale + 1 : nullptr, W.as<double>(),
                                                           g.as<double>(), h >= 0 ? Y_slot(h) : nullptr, h >= 0 ? S_slot(h) : nullptr,
                                                           inv_n, lam, D, k, bs, n, part.as<double>());
    c.launches += 1;
    finish(part.as<double>(), kRedBlocks, 0, SC_GG);
    if (h >= 0) {
      finish(part.as<double>() + kRedBlocks, kRedBlocks, 0, SC_SY);
      finish(part.as<double>() + 2 * kRedBlocks, kRedBlocks, 0, SC_YY);
    }
    finish(part.as<double>() + 3 * kRedBlocks, kRedBlocks, 1, SC_GMAX);
    lb_end_kernel<<<1, 1, 0, st>>>(sc.as<double>(), red64.as<double>() + k, inv_n, lam, h);
    c.launches += 1;
    c.span_end();
  };
  double host_sc[kScHost];
  auto read_scalars = [&]() {
    KS_CUDA(cudaMemcpyAsync(host_sc, sc.p, sizeof(host_sc), cudaMemcpyDeviceToHost, st));
    KS_CUDA(cudaStreamSynchronize(st));
  };

  // ---- f(W_0), g(W_0)
  residual(false);
  gradient_pass(gen_mean);
  if (gen_mean) {  // exact means: mean = shift + (column sums of S) / N
    launch_delta_mean(ssum, shift.as<float>(), n_total, delta.as<double>(), mean.as<double>(), static_cast<int>(D), st);
    c.launches += 1;
  }
  new_gradient(-1);
  read_scalars();
  std::vector<double> losses{host_sc[SC_LOSS]};
  std::deque<int> order;  // history slots, oldest first
  int iterations = 0;
  std::string stop = "max_iterations";
  if (host_sc[SC_GMAX] == 0.0) stop = "zero_gradient";
  const int64_t pad_cols = kpad;

  for (int t = 0; t < num_iter && stop != "zero_gradient"; ++t) {
    // ---- direction: two-loop recursion over the history (P is the work vector), then the descent check
    c.span_begin(PH_SOLVE);
    const int L = static_cast<int>(order.size());
    if (L == 0) {
      lin(P.as<double>(), LbTerm{g.as<double>(), nullptr, -1.0}, LbTerm{}, nullptr, 2, g.as<double>(), nullptr);
    } else {
      for (int q = L - 1; q >= 0; --q) {  // newest first: a_i = rho_i s_i . q;  q -= a_i y_i
        const int h = order[q];
        if (q == L - 1) lin(P.as<double>(), LbTerm{g.as<double>()}, LbTerm{}, nullptr, 1, S_slot(h), nullptr);
        else lin(P.as<double>(), LbTerm{P.as<double>()}, LbTerm{Y_slot(order[q + 1]), scp(a_of(order[q + 1])), -1.0}, nullptr, 1, S_slot(h), nullptr);
        finish(part.as<double>(), kRedBlocks, 0, a_of(h), nullptr, scp(rho_of(h)), 1.0);
      }
      // r = gamma (q - a_0 y_0); then oldest first: b_i = rho_i y_i . r;  r += (a_i - b_i) s_i
      for (int q = 0; q < L; ++q) {
        const int h = order[q];
        if (q == 0) lin(P.as<double>(), LbTerm{P.as<double>()}, LbTerm{Y_slot(h), scp(a_of(h)), -1.0}, scp(SC_GAMMA), 1, Y_slot(h), nullptr);
        else lin(P.as<double>(), LbTerm{P.as<double>()}, LbTerm{S_slot(order[q - 1]), scp(cf_of(order[q - 1])), 1.0}, nullptr, 1, Y_slot(h), nullptr);
        finish(part.as<double>(), kRedBlocks, 0, cf_of(h), scp(a_of(h)), scp(rho_of(h)), -1.0);
      }
      const int hn = order[L - 1];  // P = -(r + (a_n - b_n) s_n)
      lin(P.as<double>(), LbTerm{P.as<double>(), nullptr, -1.0}, LbTerm{S_slot(hn), scp(cf_of(hn)), -1.0}, nullptr, 2, g.as<double>(), nullptr);
    }
    finish(part.as<double>(), kRedBlocks, 0, SC_GP);
    finish(part.as<double>() + kRedBlocks, kRedBlocks, 0, SC_PP);
    lb_fallback_kernel<<<kRedBlocks, kRedThreads, 0, st>>>(P.as<double>(), g.as<double>(), n, sc.as<double>());
    lb_fallback_scalars_kernel<<<1, 1, 0, st>>>(sc.as<double>());
    c.launches += 2;
    // ---- P^T packed per feature block (fp16: one power-of-two scale for all of P), cbias_j = delta_j . P_j
    if (f16) {
      KS_CUDA(cudaMemsetAsync(maxbits + 1, 0, sizeof(unsigned), st));
      launch_max_abs_f64(P.as<double>(), n, maxbits + 1, st);
      launch_pow2_scale(maxbits + 1, 8192.f, pscale, st);
      c.launches += 2;
    }
    for (int j = 0; j < nb; ++j) {
      int64_t c0;
      const int b = block_cols(j, &c0);
      const double* Pj = P.as<double>() + c0 * k;
      const size_t boff = static_cast<size_t>(j) * kpad * lds;
      if (f16)
        launch_pack_update16(Pj, nullptr, dl ? dl + c0 : nullptr, static_cast<uint16_t*>(bop.p) + boff, static_cast<int>(lds),
                             cbias.as<float>() + j * kpad, b, k, static_cast<int>(kpad), pscale, st,
                             x2 ? static_cast<uint16_t*>(bop_lo.p) + boff : nullptr);
      else
        launch_pack_update(Pj, nullptr, dl ? dl + c0 : nullptr, bop.as<float>() + boff, x2 ? bop_lo.as<float>() + boff : nullptr,
                           static_cast<int>(lds), cbias.as<float>() + j * kpad, b, k, static_cast<int>(kpad), st);
      c.launches += 1;
    }
    c.span_end();
    // ---- Q = -A_c P (the update epilogue's sign), |Q|^2, alpha
    KS_CUDA(cudaMemsetAsync(Q.p, 0, Q.bytes, st));
    for (int j = 0; j < nb; ++j) {
      int64_t c0;
      const int b = block_cols(j, &c0);
      make_slab(j, n_loc, nullptr, false);
      c.span_begin(PH_UPDATE);
      const size_t boff = static_cast<size_t>(j) * kpad * lds;
      const void* bj = static_cast<const uint8_t*>(bop.p) + es * boff;
      const void* bj_lo = x2 ? static_cast<const uint8_t*>(bop_lo.p) + es * boff : nullptr;
      const float* cb = cbias.as<float>() + j * kpad;
      if (x2 && f16) {
        launch_update(c, slab.p, lds, n_loc, b, bj, lds, k, Q.as<float>(), kpad, cb, EPI_UPDATE, true, st, true, pscale + 1, slab_lo.p, bj_lo);
        flops += 4.0 * n_loc * static_cast<double>(b) * k;
      } else {
        launch_update(c, slab.p, lds, n_loc, b, bj, lds, k, Q.as<float>(), kpad, cb, EPI_UPDATE, true, st, f16, f16 ? pscale + 1 : nullptr);
      }
      if (x2 && !f16) {
        launch_update(c, slab_lo.p, lds, n_loc, b, bj, lds, k, Q.as<float>(), kpad, nullptr, EPI_UPDATE, true, st, false, nullptr);
        launch_update(c, slab.p, lds, n_loc, b, bj_lo, lds, k, Q.as<float>(), kpad, nullptr, EPI_UPDATE, true, st, false, nullptr);
        flops += 4.0 * n_loc * static_cast<double>(b) * k;
      }
      flops += 2.0 * n_loc * static_cast<double>(b) * k;
      c.span_end();
    }
    c.span_begin(PH_OTHER);
    lb_sumsq_f32_kernel<<<kRedBlocks, kRedThreads, 0, st>>>(Q.as<float>(), n_loc * pad_cols, part.as<double>());
    finish(part.as<double>(), kRedBlocks, 0, SC_QQ);
    c.launches += 1;
    c.span_end();
    c.span_begin(PH_ALLREDUCE);
    c.allreduce_f64(scp(SC_QQ), 1);
    c.span_end();
    c.span_begin(PH_SOLVE);
    lb_alpha_kernel<<<1, 1, 0, st>>>(sc.as<double>(), inv_n, lam);
    c.launches += 1;
    // ---- the new history slot: the oldest one when the history is full
    const int h = order.empty() ? 0 : (static_cast<int>(order.size()) == m ? order.front() : (order.back() + 1) % m);
    lin(W.as<double>(), LbTerm{W.as<double>()}, LbTerm{P.as<double>(), scp(SC_ALPHA), 1.0}, nullptr, 1, nullptr, nullptr);  // W += alpha P
    finish(part.as<double>(), kRedBlocks, 0, SC_WW);
    lin(S_slot(h), LbTerm{P.as<double>(), scp(SC_ALPHA), 1.0}, LbTerm{}, nullptr, 0, nullptr, nullptr);  // s = alpha P
    c.span_end();
    residual(true);  // R = Y_c - A_c W_new
    gradient_pass(false);
    new_gradient(h);
    read_scalars();
    if (host_sc[SC_CURV] != 0.0) {  // no step was taken
      stop = "non_positive_curvature";
      break;
    }
    iterations = t + 1;
    const double f = host_sc[SC_LOSS], gmax = host_sc[SC_GMAX];
    losses.push_back(f);
    if (host_sc[SC_RESET] != 0.0) order.clear();
    if (!(host_sc[SC_SY] > 0.0)) {
      stop = "non_positive_curvature";
      break;
    }
    if (static_cast<int>(order.size()) == m) order.pop_front();
    order.push_back(h);
    if (gmax == 0.0) {
      stop = "zero_gradient";
      break;
    }
    if (t + 1 == num_iter) {
      stop = "max_iterations";
      break;
    }
    if (tol > 0.0) {
      const size_t L2 = losses.size();
      double mx = -INFINITY;
      for (size_t q = (L2 > 11 ? L2 - 11 : 0); q + 1 < L2; ++q) mx = std::max(mx, losses[q]);
      if (mx - f <= tol * std::fabs(f)) {
        stop = "function_values_converged";
        break;
      }
      if (gmax <= std::max(tol * std::fabs(f), 1e-8)) {
        stop = "gradient_converged";
        break;
      }
    }
  }

  // ---- the model: LinearMapper(W, Some(ybar), Some(mean)) / LinearMapper(W, None, None), W in blocks of bs features
  auto model = std::make_unique<Model>();
  model->block_size = bs;
  model->k = k;
  model->has_mean = fit_intercept;
  model->has_intercept = fit_intercept;
  model->intercept.alloc(sizeof(double) * k);
  KS_CUDA(cudaMemcpyAsync(model->intercept.p, ymean.p, sizeof(double) * k, cudaMemcpyDeviceToDevice, st));
  for (int j = 0; j < nb; ++j) {
    int64_t c0;
    const int b = block_cols(j, &c0);
    model->brows.push_back(b);
    auto Wj = std::make_unique<DevBuf>();
    Wj->alloc(sizeof(double) * static_cast<size_t>(b) * k);
    KS_CUDA(cudaMemcpyAsync(Wj->p, W.as<double>() + c0 * k, Wj->bytes, cudaMemcpyDeviceToDevice, st));
    model->W.push_back(std::move(Wj));
    if (fit_intercept) {
      auto mj = std::make_unique<DevBuf>();
      mj->alloc(sizeof(double) * b);
      KS_CUDA(cudaMemcpyAsync(mj->p, mean.as<double>() + c0, mj->bytes, cudaMemcpyDeviceToDevice, st));
      model->mean.push_back(std::move(mj));
    }
  }
  if (c.host_mirror) {
    model_alloc_host(*model);
    for (int j = 0; j < nb; ++j) model_block_to_host(*model, j, st);
    model_intercept_to_host(*model, st);
  }
  KS_CUDA(cudaEventRecord(ev1, st));
  c.check_async("DenseLBFGSwithL2.fit");
  if (f16) {  // every rank scales alike, but only some may overflow -> all-reduce the flag first
    c.allreduce_max_u32(maxbits + 6, 1);
    unsigned ovf = 0;
    KS_CUDA(cudaMemcpyAsync(&ovf, maxbits + 6, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    KS_CUDA(cudaStreamSynchronize(st));
    if (ovf)
      throw KsError{KS_ERR_INVALID, "the residual left fp16's range during the fit (it grew more than 16x over the centred labels): "
                                    "use KS_PRECISION_TF32 for this problem"};
  }
  float total_ms = 0;
  cudaEventElapsedTime(&total_ms, ev0, ev1);
  double ms[PH_COUNT];
  c.collect_spans(ms);
  for (cudaEvent_t e : c.fit_events) c.event_pool.push_back(e);
  c.fit_events.clear();
  std::ostringstream js;
  js.precision(17);
  js << "{\"solver\":\"lbfgs\",\"n_local\":" << n_loc << ",\"n_total\":" << static_cast<int64_t>(n_total) << ",\"d\":" << D
     << ",\"k\":" << k << ",\"block_size\":" << bs << ",\"num_blocks\":" << nb << ",\"num_corrections\":" << m
     << ",\"world\":" << c.world << ",\"iterations\":" << iterations << ",\"stop_reason\":\"" << stop << "\",\"loss_history\":[";
  for (size_t q = 0; q < losses.size(); ++q) js << (q ? "," : "") << losses[q];
  js << "],\"total_ms\":" << total_ms << ",\"featurize_ms\":" << ms[PH_FEATURIZE] << ",\"gram_ms\":" << ms[PH_GRAM]
     << ",\"allreduce_ms\":" << ms[PH_ALLREDUCE] << ",\"solve_ms\":" << ms[PH_SOLVE] << ",\"update_ms\":" << ms[PH_UPDATE]
     << ",\"other_ms\":" << ms[PH_OTHER] << ",\"local_flops\":" << flops << ",\"launches\":" << (c.launches - launches0)
     << ",\"mma\":\"" << (x2 ? (f16 ? "f16x2" : "tf32x2") : f16 ? "f16" : "tf32x1") << "\",\"host_ms\":"
     << std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count() << "}";
  c.stats_json = js.str();
  return c.add(std::move(model));
}

}  // namespace ks
