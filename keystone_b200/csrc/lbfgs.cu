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
//
// The sparse fit (SparseLBFGSwithL2, DESIGN.md section 20) at the end of the file drives the same recursion (LbCore) with the fp64
// gather products of sparse.cu in place of the two GEMMs.
#include "engine.h"
#include "lbfgs_core.cuh"
#include "operand_split.cuh"

#include <cuda_fp16.h>
#include <math.h>

#include <algorithm>
#include <chrono>
#include <deque>
#include <sstream>

namespace ks {

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

// |Q|^2 per CTA into part[block] over a dense fp64 vector (the sparse fit's Q, N x k row-major)
__global__ void __launch_bounds__(kRedThreads) lb_sumsq_f64_kernel(const double* __restrict__ Q, int64_t total, double* part) {
  double a = 0.0;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    a = fma(Q[i], Q[i], a);
  const double s = lb_block_reduce(a, 0);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}


static void check_lbfgs_args(int m, double tol, int num_iter, double lam) {
  if (m < 1) throw KsError{KS_ERR_INVALID, "numCorrections must be >= 1"};
  if (num_iter < 1) throw KsError{KS_ERR_INVALID, "numIterations must be >= 1"};
  if (!(lam >= 0.0) || !std::isfinite(lam)) throw KsError{KS_ERR_INVALID, "regParam must be finite and >= 0"};
  if (!(tol >= 0.0) || !std::isfinite(tol)) throw KsError{KS_ERR_INVALID, "convergenceTol must be finite and >= 0"};
}

// ------------------------------------------------------------------------------------ the fit
int64_t fit_lbfgs(Ctx& c, FeatSrc& src, Matrix& Y, bool fit_intercept, int m, double tol, int num_iter, double lam, int precision) {
  check_lbfgs_args(m, tol, num_iter, lam);
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
  DevBuf ymean, rpart, cpart, Cbuf, red64, shift, delta, mean, fsum, R, Q, r_op, r_lo, scales, samp;
  DevBuf slab, slab_lo, sf32, bop, bop_lo, cbias;
  ymean.alloc(sizeof(double) * k);
  launch_scale_f64(ysum.as<double>(), inv_n, nullptr, ymean.as<double>(), k, st);
  c.launches += 1;
  LbCore core(c, n, m, inv_n, lam);
  DevBuf& W = core.W;
  DevBuf& P = core.P;
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
  auto scp = [&](int slot) { return core.scp(slot); };
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
    core.new_gradient<float>(Cm, kpad, dl, red64.as<double>(), f16 ? rscale + 1 : nullptr, D, k, bs, red64.as<double>() + k, h);
  };

  // ---- f(W_0), g(W_0)
  residual(false);
  gradient_pass(gen_mean);
  if (gen_mean) {  // exact means: mean = shift + (column sums of S) / N
    launch_delta_mean(ssum, shift.as<float>(), n_total, delta.as<double>(), mean.as<double>(), static_cast<int>(D), st);
    c.launches += 1;
  }
  new_gradient(-1);
  const bool nothing_to_do = core.start();
  const int64_t pad_cols = kpad;

  for (int t = 0; t < num_iter && !nothing_to_do; ++t) {
    // ---- direction: two-loop recursion over the history (P is the work vector), then the descent check
    c.span_begin(PH_SOLVE);
    core.direction();
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
    lb_sumsq_f32_kernel<<<kRedBlocks, kRedThreads, 0, st>>>(Q.as<float>(), n_loc * pad_cols, core.part.as<double>());
    core.finish(core.part.as<double>(), kRedBlocks, 0, SC_QQ);
    c.launches += 1;
    c.span_end();
    c.span_begin(PH_ALLREDUCE);
    c.allreduce_f64(scp(SC_QQ), 1);
    c.span_end();
    c.span_begin(PH_SOLVE);
    const int h = core.step();
    c.span_end();
    residual(true);  // R = Y_c - A_c W_new
    gradient_pass(false);
    new_gradient(h);
    if (core.accept(t, h, num_iter, tol)) break;
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
     << ",\"world\":" << c.world;
  core.history_json(js);
  js << ",\"total_ms\":" << total_ms << ",\"featurize_ms\":" << ms[PH_FEATURIZE] << ",\"gram_ms\":" << ms[PH_GRAM]
     << ",\"allreduce_ms\":" << ms[PH_ALLREDUCE] << ",\"solve_ms\":" << ms[PH_SOLVE] << ",\"update_ms\":" << ms[PH_UPDATE]
     << ",\"other_ms\":" << ms[PH_OTHER] << ",\"local_flops\":" << flops << ",\"launches\":" << (c.launches - launches0)
     << ",\"mma\":\"" << (x2 ? (f16 ? "f16x2" : "tf32x2") : f16 ? "f16" : "tf32x1") << "\",\"host_ms\":"
     << std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count() << "}";
  c.stats_json = js.str();
  return c.add(std::move(model));
}

// ------------------------------------------------------------------------------------ the sparse fit
// SparseLBFGSwithL2 with LeastSquaresSparseGradient (K/nodes/learning/LBFGS.scala:208-281), DESIGN.md section 20: no centring; with
// an intercept the unknowns are x = [W; b] over [A 1] (the ones column is implicit), and b is regularised in f and in g:
//   f = |[A 1] x - Y|_F^2 / (2N) + lambda/2 |x|_F^2,   g = [A 1]^T ([A 1] x - Y) / N + lambda x,   x_0 = 0.
// Everything after the fp32 labels is fp64.  R = Y - [A 1] x (the dense fit's sign), Q = [A 1] P, R -= alpha Q.

// R = Y (x_0 = 0), fp32 labels widened to fp64, row-major ld k
__global__ void sp_init_residual_kernel(const float* __restrict__ Y, int64_t ldy, int64_t rows, int k, double* __restrict__ R) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= rows * k) return;
  const int64_t r = i / k;
  R[i] = static_cast<double>(Y[r * ldy + (i - r * k)]);
}
// R -= alpha Q (Q null: R unchanged), then the column sums of R per CTA into cpart[blockIdx.x * k + c] and |R|^2 per CTA into
// part[blockIdx.x].  CTA = rows [blockIdx.x rpb, +rpb); thread (tx, ty) = threadIdx (% 32, / 32) takes columns c0 + tx, rows
// ty, ty + 8, ...; both sums are finished in a fixed order.
__global__ void __launch_bounds__(256) sp_residual_kernel(double* __restrict__ R, const double* __restrict__ Q, const double* __restrict__ alpha,
                                                          int64_t rows, int k, int64_t rpb, double* __restrict__ cpart,
                                                          double* __restrict__ part) {
  __shared__ double red[8][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const double a = Q ? *alpha : 0.0;
  const int64_t r_begin = blockIdx.x * rpb, r_end = min(rows, r_begin + rpb);
  double sq = 0.0;
  for (int c0 = 0; c0 < k; c0 += 32) {
    const int c = c0 + tx;
    double cs = 0.0;
    if (c < k) {
      for (int64_t r = r_begin + ty; r < r_end; r += 8) {
        double v = R[r * k + c];
        if (Q) {
          v -= a * Q[r * k + c];
          R[r * k + c] = v;
        }
        cs += v;
        sq = fma(v, v, sq);
      }
    }
    red[ty][tx] = cs;
    __syncthreads();
    if (ty == 0 && c < k) {
      double s = 0.0;
#pragma unroll
      for (int y = 0; y < 8; ++y) s += red[y][tx];
      cpart[blockIdx.x * static_cast<int64_t>(k) + c] = s;
    }
    __syncthreads();
  }
  const double t = lb_block_reduce(sq, 0);
  if (threadIdx.x == 0) part[blockIdx.x] = t;
}
int64_t fit_sparse_lbfgs(Ctx& c, const SparseMat& A, Matrix& Y, bool fit_intercept, int m, double tol, int num_iter, double lam) {
  check_lbfgs_args(m, tol, num_iter, lam);
  if (Y.rows != A.rows) throw KsError{KS_ERR_INVALID, "features and labels have different row counts"};
  const int64_t n_loc = A.rows, D = A.cols;
  const int k = static_cast<int>(Y.cols);
  if (k <= 0) throw KsError{KS_ERR_INVALID, "empty problem"};
  const int bs = static_cast<int>(std::min<int64_t>(D, 4096));  // feature block of the model (as the dense fit's)
  const int nb = static_cast<int>((D + bs - 1) / bs);
  const int64_t n = D * k + (fit_intercept ? k : 0);  // [W; b]: W blocked as in the dense fit, then b
  cudaStream_t st = c.st;
  const auto host_t0 = std::chrono::steady_clock::now();
  c.spans.clear();
  const int64_t launches0 = c.launches;
  cudaEvent_t ev0 = c.get_event(), ev1 = c.get_event();
  c.fit_events.push_back(ev0);
  c.fit_events.push_back(ev1);
  KS_CUDA(cudaEventRecord(ev0, st));

  // ---- global row and entry counts
  c.span_begin(PH_OTHER);
  DevBuf cnt;
  cnt.alloc(sizeof(double) * 2);
  launch_set_f64(cnt.as<double>(), static_cast<double>(n_loc), st);
  launch_set_f64(cnt.as<double>() + 1, static_cast<double>(A.nnz), st);
  c.launches += 2;
  c.allreduce_f64(cnt.as<double>(), 2);
  double tot[2] = {0, 0};
  KS_CUDA(cudaMemcpyAsync(tot, cnt.p, sizeof(tot), cudaMemcpyDeviceToHost, st));
  KS_CUDA(cudaStreamSynchronize(st));
  if (tot[0] < 1) throw KsError{KS_ERR_INVALID, "no training rows"};
  const double n_total = tot[0], inv_n = 1.0 / n_total;

  LbCore core(c, n, m, inv_n, lam);
  const int64_t rpb = 1024, nrb = (std::max<int64_t>(n_loc, 1) + rpb - 1) / rpb;
  DevBuf R, Q, Xr, Cbuf, red64, rpart, cpart;
  R.alloc(sizeof(double) * static_cast<size_t>(std::max<int64_t>(n_loc, 1)) * k);
  Q.alloc(R.bytes);
  Xr.alloc(sizeof(double) * static_cast<size_t>(n));
  Cbuf.alloc(sizeof(double) * static_cast<size_t>(D) * k);
  red64.alloc(sizeof(double) * (k + 1));  // column sums of R, then |R|^2
  rpart.alloc(sizeof(double) * static_cast<size_t>(nrb));
  cpart.alloc(sizeof(double) * static_cast<size_t>(nrb) * k);
  if (n_loc > 0) {
    sp_init_residual_kernel<<<static_cast<unsigned>((n_loc * k + 255) / 256), 256, 0, st>>>(Y.d, Y.ld, n_loc, k, R.as<double>());
    c.launches += 1;
  }
  c.span_end();

  // R -= alpha Q (Q null: R as it is), its column sums and |R|^2 into red64 (rank-local)
  auto residual = [&](bool with_q) {
    c.span_begin(PH_OTHER);
    sp_residual_kernel<<<static_cast<unsigned>(nrb), 256, 0, st>>>(R.as<double>(), with_q ? Q.as<double>() : nullptr, core.scp(SC_ALPHA), n_loc,
                                                                   k, rpb, cpart.as<double>(), rpart.as<double>());
    lb_colsum_finish_kernel<<<(k + 127) / 128, 128, 0, st>>>(cpart.as<double>(), static_cast<int>(nrb), k, k, red64.as<double>());
    lb_finish_kernel<<<1, kRedThreads, 0, st>>>(rpart.as<double>(), static_cast<int>(nrb), 0, red64.as<double>() + k, nullptr, nullptr, 1.0);
    c.launches += 3;
    c.span_end();
  };
  // C = A^T R, then the all-reduces of C and of (column sums of R, |R|^2)
  auto gradient_pass = [&]() {
    c.span_begin(PH_GRAM);
    KS_CUDA(cudaMemsetAsync(Cbuf.p, 0, Cbuf.bytes, st));
    sparse_product(c, A, true, R.as<double>(), k, nullptr, Cbuf.as<double>(), st);
    c.span_end();
    c.span_begin(PH_ALLREDUCE);
    c.allreduce_f64(Cbuf.as<double>(), static_cast<size_t>(D) * k);
    c.allreduce_f64(red64.as<double>(), static_cast<size_t>(k + 1));
    c.span_end();
  };
  auto new_gradient = [&](int h) {
    core.new_gradient<double>(Cbuf.as<double>(), k, nullptr, red64.as<double>(), nullptr, D, k, bs, red64.as<double>() + k, h);
  };

  // ---- f(x_0), g(x_0)
  residual(false);
  gradient_pass();
  new_gradient(-1);
  const bool nothing_to_do = core.start();
  for (int t = 0; t < num_iter && !nothing_to_do; ++t) {
    c.span_begin(PH_SOLVE);
    core.direction();
    for (int j = 0; j < nb; ++j) {  // P row-major for the gathers: its blocks are the model's layout
      const int64_t c0 = static_cast<int64_t>(j) * bs;
      launch_rows_from_block(c, core.P.as<double>() + c0 * k, std::min<int64_t>(D, c0 + bs) - c0, k, c0, Xr.as<double>(), st);
    }
    if (fit_intercept)
      KS_CUDA(cudaMemcpyAsync(Xr.as<double>() + D * k, core.P.as<double>() + D * k, sizeof(double) * k, cudaMemcpyDeviceToDevice, st));
    c.span_end();
    // ---- Q = [A 1] P, |Q|^2, alpha
    c.span_begin(PH_UPDATE);
    if (n_loc > 0) KS_CUDA(cudaMemsetAsync(Q.p, 0, Q.bytes, st));
    sparse_product(c, A, false, Xr.as<double>(), k, fit_intercept ? Xr.as<double>() + D * k : nullptr, Q.as<double>(), st);
    c.span_end();
    c.span_begin(PH_OTHER);
    lb_sumsq_f64_kernel<<<kRedBlocks, kRedThreads, 0, st>>>(Q.as<double>(), n_loc * k, core.part.as<double>());
    core.finish(core.part.as<double>(), kRedBlocks, 0, SC_QQ);
    c.launches += 1;
    c.span_end();
    c.span_begin(PH_ALLREDUCE);
    c.allreduce_f64(core.scp(SC_QQ), 1);
    c.span_end();
    c.span_begin(PH_SOLVE);
    const int h = core.step();
    c.span_end();
    residual(true);
    gradient_pass();
    new_gradient(h);
    if (core.accept(t, h, num_iter, tol)) break;
  }

  // ---- the model: SparseLinearMapper(W, Some(b)) / SparseLinearMapper(W, None), W in blocks of bs features, no feature means
  auto model = std::make_unique<Model>();
  model->block_size = bs;
  model->k = k;
  model->has_mean = false;
  model->has_intercept = fit_intercept;
  model->intercept.alloc(sizeof(double) * k);
  if (fit_intercept)
    KS_CUDA(cudaMemcpyAsync(model->intercept.p, core.W.as<double>() + D * k, sizeof(double) * k, cudaMemcpyDeviceToDevice, st));
  else
    KS_CUDA(cudaMemsetAsync(model->intercept.p, 0, sizeof(double) * k, st));
  for (int j = 0; j < nb; ++j) {
    const int64_t c0 = static_cast<int64_t>(j) * bs;
    const int64_t b = std::min<int64_t>(D, c0 + bs) - c0;
    model->brows.push_back(b);
    auto Wj = std::make_unique<DevBuf>();
    Wj->alloc(sizeof(double) * static_cast<size_t>(b) * k);
    KS_CUDA(cudaMemcpyAsync(Wj->p, core.W.as<double>() + c0 * k, Wj->bytes, cudaMemcpyDeviceToDevice, st));
    model->W.push_back(std::move(Wj));
  }
  if (c.host_mirror) {
    model_alloc_host(*model);
    for (int j = 0; j < nb; ++j) model_block_to_host(*model, j, st);
    model_intercept_to_host(*model, st);
  }
  KS_CUDA(cudaEventRecord(ev1, st));
  c.check_async("SparseLBFGSwithL2.fit");
  float total_ms = 0;
  cudaEventElapsedTime(&total_ms, ev0, ev1);
  double ms[PH_COUNT];
  c.collect_spans(ms);
  for (cudaEvent_t e : c.fit_events) c.event_pool.push_back(e);
  c.fit_events.clear();
  std::ostringstream js;
  js.precision(17);
  js << "{\"solver\":\"sparse_lbfgs\",\"n_local\":" << n_loc << ",\"n_total\":" << static_cast<int64_t>(n_total) << ",\"d\":" << D
     << ",\"k\":" << k << ",\"nnz_local\":" << A.nnz << ",\"nnz\":" << static_cast<int64_t>(tot[1]) << ",\"fit_intercept\":"
     << (fit_intercept ? "true" : "false") << ",\"block_size\":" << bs << ",\"num_blocks\":" << nb << ",\"num_corrections\":" << m
     << ",\"world\":" << c.world;
  core.history_json(js);
  js << ",\"total_ms\":" << total_ms << ",\"ap_ms\":" << ms[PH_UPDATE] << ",\"atr_ms\":" << ms[PH_GRAM]
     << ",\"allreduce_ms\":" << ms[PH_ALLREDUCE] << ",\"solve_ms\":" << ms[PH_SOLVE] << ",\"other_ms\":" << ms[PH_OTHER]
     << ",\"launches\":" << (c.launches - launches0) << ",\"host_ms\":"
     << std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count() << "}";
  c.stats_json = js.str();
  return c.add(std::move(model));
}

}  // namespace ks
