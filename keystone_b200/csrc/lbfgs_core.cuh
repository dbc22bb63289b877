// The L-BFGS recursion shared by the least-squares fits (lbfgs.cu) and the logistic-regression fit (logistic.cu): the fp64
// reduction kernels, the scalar slots, the gradient kernel and LbCore (two-loop direction, step bookkeeping, stop rules).
// Every kernel here is static: each fit's translation unit carries its own copy.
#pragma once
#include "engine.h"

#include <math.h>

#include <algorithm>
#include <deque>
#include <ostream>
#include <string>
#include <vector>

namespace ks {

static constexpr int kRedBlocks = 264;  // grid of every fp64 reduction below: partial sums per block, then summed in block order
static constexpr int kRedThreads = 256;

// block-wide sum (op 0) or max (op 1) of a per-thread value; the result is valid in thread 0
static __device__ double lb_block_reduce(double v, int op) {
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
static __global__ void __launch_bounds__(kRedThreads) lb_lin_dot_kernel(double* out, LbTerm t0, LbTerm t1, const double* gscale, int ndots,
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
static __global__ void __launch_bounds__(kRedThreads) lb_finish_kernel(const double* part, int nparts, int op, double* dst, const double* base,
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
  SC_WP,   // <W, P>: the logistic fit's line search (logistic.cu)
  SC_HIST  // then per history slot: a, coef, rho
};

// After the direction: if <g, P> >= 0 (not a descent direction after rounding) P = -g; the history is dropped by the host
static __global__ void lb_fallback_kernel(double* P, const double* g, int64_t n, const double* sc) {
  if (!(sc[SC_GP] >= 0.0)) return;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    P[i] = -g[i];
}
static __global__ void lb_fallback_scalars_kernel(double* sc) {
  sc[SC_RESET] = 0.0;
  if (sc[SC_GP] >= 0.0) {
    sc[SC_RESET] = 1.0;
    sc[SC_GP] = -sc[SC_GG];
    sc[SC_PP] = sc[SC_GG];
  }
}
// the exact minimiser along P: alpha = -<g, P> / (|A_c P|^2 / N + lambda |P|^2); a curvature that is not > 0 stops the fit
static __global__ void lb_alpha_kernel(double* sc, double inv_n, double lam) {
  const double den = sc[SC_QQ] * inv_n + lam * sc[SC_PP];
  if (den > 0.0 && isfinite(den)) {
    sc[SC_ALPHA] = -sc[SC_GP] / den;
    sc[SC_CURV] = 0.0;
  } else {
    sc[SC_ALPHA] = 0.0;
    sc[SC_CURV] = 1.0;
  }
}
// loss of the new iterate, loss_mul *rr / N + lambda / 2 |W|^2 (least squares: loss_mul = 1/2, rr = |R|^2), rho and gamma of the
// new pair (slot h)
static __global__ void lb_end_kernel(double* sc, const double* rr, double loss_mul, double inv_n, double lam, int h) {
  sc[SC_LOSS] = loss_mul * (*rr) * inv_n + 0.5 * lam * sc[SC_WW];
  if (h < 0) return;
  const double sy = sc[SC_SY], yy = sc[SC_YY];
  sc[SC_HIST + 3 * h + 2] = sy > 0.0 ? 1.0 / sy : 0.0;
  sc[SC_GAMMA] = yy > 0.0 ? sy / yy : 1.0;
}

// g_new = -(C cs - delta rsum) / N + lambda W over the blocked flat layout (block j: features [j bs, j bs + b_j), column-major
// b_j x k at offset j bs k); C is row-major D x ldc (feature, class), fp32 (dense fit) or fp64 (sparse fit).  Entries past D k
// (n = D k + k: the sparse fit's bias row) take rsum in place of C.  y = g_new - g_old and s . y, y . y when y is given.
// part: [0] |g|^2, [1] s . y, [2] y . y, [3] max |g|
template <class CT>
static __global__ void __launch_bounds__(kRedThreads) lb_gradient_kernel(const CT* __restrict__ C, int64_t ldc, const double* __restrict__ delta,
                                                                  const double* __restrict__ rsum, const float* __restrict__ c_scale,
                                                                  const double* __restrict__ W, double* g, double* y,
                                                                  const double* __restrict__ s, double inv_n, double lam, int64_t D,
                                                                  int k, int bs, int64_t n, double* part) {
  const double cs = c_scale ? static_cast<double>(*c_scale) : 1.0;
  const int64_t blk = static_cast<int64_t>(bs) * k, dk = D * k;
  double gg = 0.0, sy = 0.0, yy = 0.0, gm = 0.0;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    double v;
    if (i < dk) {
      const int64_t j = i / blk, r = i - j * blk;
      const int64_t bj = min(static_cast<int64_t>(bs), D - j * bs);
      const int64_t c = r / bj, f = j * bs + (r - c * bj);
      v = static_cast<double>(C[f * ldc + c]) * cs;
      if (delta) v -= delta[f] * rsum[c];
    } else {  // n > D k: the bias row of the implicit ones column (sparse fit), whose product with R is R's column sums
      v = rsum[i - dk];
    }
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

// ------------------------------------------------------------------------------------ the recursion shared by both fits
// The fp64 state of an L-BFGS least-squares fit over a flat vector of n unknowns and everything that does not touch the data:
// the two-loop direction, the exact step, the new gradient from the all-reduced C = A^T R, and the host's stop rules.  The
// dense fit (fit_lbfgs) and the sparse fit (fit_sparse_lbfgs) supply the products A P and A^T R around it.
struct LbCore {
  Ctx& c;
  cudaStream_t st;
  int64_t n;
  int m;
  double inv_n, lam;
  double loss_mul = 0.5;  // f = loss_mul * rr / N + lambda / 2 |W|^2 for the rr new_gradient is given
  DevBuf W, g, P, hist, sc, part;
  std::deque<int> order;  // history slots, oldest first
  std::vector<double> losses;
  int iterations = 0;
  std::string stop = "max_iterations";
  double host_sc[kScHost];

  LbCore(Ctx& c_, int64_t n_, int m_, double inv_n_, double lam_) : c(c_), st(c_.st), n(n_), m(m_), inv_n(inv_n_), lam(lam_) {
    W.alloc(sizeof(double) * n);
    g.alloc(sizeof(double) * n);
    P.alloc(sizeof(double) * n);
    hist.alloc(sizeof(double) * 2 * static_cast<size_t>(m) * n);  // S slots [0, m), Y slots [m, 2m)
    sc.alloc(sizeof(double) * (SC_HIST + 3 * m));
    part.alloc(sizeof(double) * 4 * kRedBlocks);
    KS_CUDA(cudaMemsetAsync(W.p, 0, W.bytes, st));
    KS_CUDA(cudaMemsetAsync(sc.p, 0, sc.bytes, st));
  }
  double* S_slot(int h) { return hist.as<double>() + static_cast<size_t>(h) * n; }
  double* Y_slot(int h) { return hist.as<double>() + static_cast<size_t>(m + h) * n; }
  double* scp(int slot) { return sc.as<double>() + slot; }
  static int a_of(int h) { return SC_HIST + 3 * h; }
  static int cf_of(int h) { return SC_HIST + 3 * h + 1; }
  static int rho_of(int h) { return SC_HIST + 3 * h + 2; }
  void finish(const double* p, int nparts, int op, int slot, const double* base = nullptr, const double* scale = nullptr, double mul = 1.0) {
    lb_finish_kernel<<<1, kRedThreads, 0, st>>>(p, nparts, op, sc.as<double>() + slot, base, scale, mul);
    c.launches += 1;
  }
  void lin(double* out, LbTerm t0, LbTerm t1, const double* gscale, int ndots, const double* w0, const double* w1) {
    lb_lin_dot_kernel<<<kRedBlocks, kRedThreads, 0, st>>>(out, t0, t1, gscale, ndots, w0, w1, n, part.as<double>());
    c.launches += 1;
  }

  // g = -(C - delta rsum) / N + lambda W (C = A^T R with R = Y - A W, all-reduced); with slot h >= 0 also y_h = g_new - g_old,
  // s_h . y_h, y_h . y_h; then the loss from rr = |R|^2
  template <class CT>
  void new_gradient(const CT* C, int64_t ldc, const double* delta, const double* rsum, const float* c_scale, int64_t D, int k, int bs,
                    const double* rr, int h) {
    c.span_begin(PH_SOLVE);
    lb_gradient_kernel<CT><<<kRedBlocks, kRedThreads, 0, st>>>(C, ldc, delta, rsum, c_scale, W.as<double>(), g.as<double>(),
                                                               h >= 0 ? Y_slot(h) : nullptr, h >= 0 ? S_slot(h) : nullptr, inv_n, lam, D,
                                                               k, bs, n, part.as<double>());
    c.launches += 1;
    finish(part.as<double>(), kRedBlocks, 0, SC_GG);
    if (h >= 0) {
      finish(part.as<double>() + kRedBlocks, kRedBlocks, 0, SC_SY);
      finish(part.as<double>() + 2 * kRedBlocks, kRedBlocks, 0, SC_YY);
    }
    finish(part.as<double>() + 3 * kRedBlocks, kRedBlocks, 1, SC_GMAX);
    lb_end_kernel<<<1, 1, 0, st>>>(sc.as<double>(), rr, loss_mul, inv_n, lam, h);
    c.launches += 1;
    c.span_end();
  }
  void read_scalars() {
    KS_CUDA(cudaMemcpyAsync(host_sc, sc.p, sizeof(host_sc), cudaMemcpyDeviceToHost, st));
    KS_CUDA(cudaStreamSynchronize(st));
  }
  // after f(W_0), g(W_0): true when there is nothing to do
  bool start() {
    read_scalars();
    losses.assign(1, host_sc[SC_LOSS]);
    if (host_sc[SC_GMAX] == 0.0) stop = "zero_gradient";
    return stop == "zero_gradient";
  }
  // two-loop recursion over the history into P, <g, P> and |P|^2, then the descent check (P = -g if <g, P> >= 0)
  void direction() {
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
  }
  // after the all-reduce of |A P|^2 into SC_QQ: alpha, W += alpha P, |W|^2 and s = alpha P into the new history slot (returned)
  int step() {
    lb_alpha_kernel<<<1, 1, 0, st>>>(sc.as<double>(), inv_n, lam);
    c.launches += 1;
    return take_step();
  }
  // with alpha in SC_ALPHA: W += alpha P, |W|^2 and s = alpha P into the new history slot (returned)
  int take_step() {
    // the new history slot: the oldest one when the history is full
    const int h = order.empty() ? 0 : (static_cast<int>(order.size()) == m ? order.front() : (order.back() + 1) % m);
    lin(W.as<double>(), LbTerm{W.as<double>()}, LbTerm{P.as<double>(), scp(SC_ALPHA), 1.0}, nullptr, 1, nullptr, nullptr);  // W += alpha P
    finish(part.as<double>(), kRedBlocks, 0, SC_WW);
    lin(S_slot(h), LbTerm{P.as<double>(), scp(SC_ALPHA), 1.0}, LbTerm{}, nullptr, 0, nullptr, nullptr);  // s = alpha P
    return h;
  }
  // after new_gradient(h) of step t: reads the scalars and applies the stop rules; true ends the fit
  bool accept(int t, int h, int num_iter, double tol) {
    read_scalars();
    if (host_sc[SC_CURV] != 0.0) {  // no step was taken
      stop = "non_positive_curvature";
      return true;
    }
    iterations = t + 1;
    const double f = host_sc[SC_LOSS], gmax = host_sc[SC_GMAX];
    losses.push_back(f);
    if (host_sc[SC_RESET] != 0.0) order.clear();
    if (!(host_sc[SC_SY] > 0.0)) {
      stop = "non_positive_curvature";
      return true;
    }
    if (static_cast<int>(order.size()) == m) order.pop_front();
    order.push_back(h);
    if (gmax == 0.0) {
      stop = "zero_gradient";
      return true;
    }
    if (t + 1 == num_iter) {
      stop = "max_iterations";
      return true;
    }
    if (tol > 0.0) {
      const size_t L2 = losses.size();
      double mx = -INFINITY;
      for (size_t q = (L2 > 11 ? L2 - 11 : 0); q + 1 < L2; ++q) mx = std::max(mx, losses[q]);
      if (mx - f <= tol * std::fabs(f)) {
        stop = "function_values_converged";
        return true;
      }
      if (gmax <= std::max(tol * std::fabs(f), 1e-8)) {
        stop = "gradient_converged";
        return true;
      }
    }
    return false;
  }
  void history_json(std::ostream& js) const {
    js << ",\"iterations\":" << iterations << ",\"stop_reason\":\"" << stop << "\",\"loss_history\":[";
    for (size_t q = 0; q < losses.size(); ++q) js << (q ? "," : "") << losses[q];
    js << "]";
  }
};

}  // namespace ks
