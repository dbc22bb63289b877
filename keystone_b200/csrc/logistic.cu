// Logistic regression and multinomial naive Bayes on the device: LogisticRegressionEstimator and NaiveBayesEstimator
// (K/nodes/learning/{LogisticRegressionModel,NaiveBayesModel}.scala, which wrap Spark MLlib).  DESIGN.md section 22.
//
// Logistic regression (MLlib's LogisticGradient + SquaredL2Updater, no intercept, pivot class 0), W: d x (k-1), W_0 = 0:
//   Z = A W,  f(W) = (1/N) sum_i [lse(0, Z_i) - Z_{i,y_i}] + lambda/2 |W|_F^2,  g = A^T (softmax(Z) - onehot(y)) / N + lambda W
// (columns 1 .. k-1; class 0 has margin 0).  The direction, history and stop rules are LbCore's (lbfgs_core.cuh); the step comes
// from a strong-Wolfe line search modelled on Breeze's StrongWolfeLineSearch, run by the host on all-reduced scalars.  Every
// iteration makes one forward product Q = A P and one transposed product C = A^T R; a line-search trial is one fused pass over
// Z + t Q (the data term and phi'(t)) plus the regulariser from |W|^2, <W, P> and |P|^2, so it never touches A.
//
// Naive Bayes (MLlib's multinomial NaiveBayes.train): S = A^T onehot(y) (d x k), class counts n_c from the host labels,
//   pi_c = log(n_c + lambda) - log(N + k lambda),  theta_cj = log(S_jc + lambda) - log(sum_j S_jc + d lambda),
// the model being W = theta^T (d x k) with intercept pi.
//
// Both fits are collective and read either a materialised fp32 matrix (products: the fp64 DMMA kernels of pca.cu) or a sparse
// matrix (the fp64 gathers of sparse.cu).  Every sum has a fixed order and every rank reads the same all-reduced scalars, so a refit
// is bit-identical and every rank ends with the same bits.  Checks that depend on one rank's data (labels, negative values, empty
// classes) are flagged, all-reduced and raised on every rank together.
#include "engine.h"
#include "lbfgs_core.cuh"

#include <math.h>

#include <algorithm>
#include <chrono>
#include <sstream>
#include <vector>

namespace ks {

// ------------------------------------------------------------------------------------ kernels
// per row: m = max(0, max_j z_j), s = e^-m + sum_j e^(z_j - m), lse = m + log s
__device__ __forceinline__ double lr_row_lse(const double* z, int kk, double* m_out, double* s_out) {
  double m = 0.0;
  for (int j = 0; j < kk; ++j) m = fmax(m, z[j]);
  double s = exp(-m);
  for (int j = 0; j < kk; ++j) s += exp(z[j] - m);
  *m_out = m;
  *s_out = s;
  return m + log(s);
}

// A line-search trial at step t: over the rows, the data loss sum_i [lse(0, z_i) - z_{i,y_i}] and sum_i (softmax(z_i) - onehot_i) . q_i
// with z = Z + t Q (recomputed in each pass over the row, never stored), into part[block] and part[kRedBlocks + block].  One thread
// per row, fixed grid; the formulas of lr_accept_kernel, so a trial at the accepted step sees the margins the accept stores.
__global__ void __launch_bounds__(kRedThreads) lr_trial_kernel(const double* __restrict__ Z, const double* __restrict__ Q, double t,
                                                               const int32_t* __restrict__ y, int64_t rows, int kk, double* part) {
  double loss = 0.0, dphi = 0.0;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < rows; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const double* zr = Z + i * kk;
    const double* qr = Q + i * kk;
    const int yi = y[i];
    double m = 0.0;
    for (int j = 0; j < kk; ++j) m = fmax(m, fma(t, qr[j], zr[j]));
    double s = exp(-m);
    for (int j = 0; j < kk; ++j) s += exp(fma(t, qr[j], zr[j]) - m);
    loss += m + log(s) - (yi > 0 ? fma(t, qr[yi - 1], zr[yi - 1]) : 0.0);
    double row_d = 0.0;
    for (int j = 0; j < kk; ++j) row_d = fma(exp(fma(t, qr[j], zr[j]) - m) / s - (yi == j + 1 ? 1.0 : 0.0), qr[j], row_d);
    dphi += row_d;
  }
  double r = lb_block_reduce(loss, 0);
  if (threadIdx.x == 0) part[blockIdx.x] = r;
  r = lb_block_reduce(dphi, 0);
  if (threadIdx.x == 0) part[kRedBlocks + blockIdx.x] = r;
}

// Accepting a step: Z += alpha Q (Q null: Z as it is), R = onehot(y) - softmax(Z) (columns 1 .. k-1) and the data loss per block into
// part[block].  Same row order and formulas as the trial kernel.
__global__ void __launch_bounds__(kRedThreads) lr_accept_kernel(double* __restrict__ Z, const double* __restrict__ Q, const double* __restrict__ alpha,
                                                                const int32_t* __restrict__ y, int64_t rows, int kk, double* __restrict__ R,
                                                                double* part) {
  const double a = Q ? *alpha : 0.0;
  double loss = 0.0;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < rows; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    double* zr = Z + i * kk;
    if (Q) {
      const double* qr = Q + i * kk;
      for (int j = 0; j < kk; ++j) zr[j] = fma(a, qr[j], zr[j]);
    }
    const int yi = y[i];
    double m, s;
    const double lse = lr_row_lse(zr, kk, &m, &s);
    loss += lse - (yi > 0 ? zr[yi - 1] : 0.0);
    double* rr = R + i * kk;
    for (int j = 0; j < kk; ++j) rr[j] = (yi == j + 1 ? 1.0 : 0.0) - exp(zr[j] - m) / s;
  }
  const double r = lb_block_reduce(loss, 0);
  if (threadIdx.x == 0) part[blockIdx.x] = r;
}

// Y (rows x k, fp64) = onehot(y); a label outside [0, k) gives a zero row (the fit is rejected before Y is used)
__global__ void nb_onehot_kernel(const int32_t* __restrict__ y, int64_t rows, int k, double* __restrict__ Y) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= rows * k) return;
  const int64_t r = i / k;
  Y[i] = y[r] == static_cast<int32_t>(i - r * k) ? 1.0 : 0.0;
}

// *flag = 1 when any value is negative or NaN (every writer stores the same value)
template <class T>
__global__ void nb_negative_flag_kernel(const T* __restrict__ v, int64_t rows, int64_t cols, int64_t ld, double* flag) {
  const int64_t n = rows * cols;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / cols;
    if (!(static_cast<double>(v[r * ld + (i - r * cols)]) >= 0.0)) *flag = 1.0;
  }
}

// One CTA per class c: the term total T_c = sum_j S_jc (threads in feature order, then a fixed tree), logT_c = log(T_c + d lambda),
// and pi_c = log(n_c + lambda) - log(N + k lambda) with N = sum_c n_c (exact: integer counts)
__global__ void __launch_bounds__(kRedThreads) nb_totals_kernel(const double* __restrict__ S, const double* __restrict__ counts, int64_t D,
                                                                int k, double lam, double* __restrict__ log_t, double* __restrict__ pi) {
  const int c = blockIdx.x;
  double a = 0.0;
  for (int64_t j = threadIdx.x; j < D; j += blockDim.x) a += S[j * k + c];
  const double t = lb_block_reduce(a, 0);
  if (threadIdx.x == 0) {
    double n = 0.0;
    for (int q = 0; q < k; ++q) n += counts[q];
    log_t[c] = log(t + static_cast<double>(D) * lam);
    pi[c] = log(counts[c] + lam) - log(n + static_cast<double>(k) * lam);
  }
}
// theta into model block j (column-major b x k, features [c0, c0 + b)): W_j[c b + r] = log(S_(c0+r)c + lambda) - logT_c
__global__ void nb_theta_kernel(const double* __restrict__ S, const double* __restrict__ log_t, int64_t c0, int64_t b, int k, double lam,
                                double* __restrict__ Wj) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= b * k) return;
  const int64_t c = i / b, r = i - c * b;
  Wj[i] = log(S[(c0 + r) * k + c] + lam) - log_t[c];
}

// ------------------------------------------------------------------------------------ shared set-up
namespace {

struct ClsData {
  Matrix* F = nullptr;
  const SparseMat* S = nullptr;
  int64_t n_loc = 0, D = 0;
};

ClsData cls_data(Ctx& c, int64_t features, int64_t sparse, int64_t n_labels, const int32_t* labels, int k) {
  if ((features == 0) == (sparse == 0)) throw KsError{KS_ERR_INVALID, "exactly one of features and sparse must be given"};
  ClsData d;
  if (features) {
    d.F = &c.matrix(features);
    d.n_loc = d.F->rows;
    d.D = d.F->cols;
  } else {
    d.S = &c.sparse(sparse);
    d.n_loc = d.S->rows;
    d.D = d.S->cols;
  }
  if (k < 2) throw KsError{KS_ERR_INVALID, "numClasses must be >= 2"};
  if (n_labels != d.n_loc) throw KsError{KS_ERR_INVALID, "n_labels differs from the rank's feature rows"};
  if (n_labels > 0 && !labels) throw KsError{KS_ERR_INVALID, "null labels"};
  if (d.D < 1) throw KsError{KS_ERR_INVALID, "no features"};
  return d;
}

GramOperand dense_operand(const Matrix& F) {
  GramOperand o;
  o.f32 = F.d;
  o.ld = F.ld;
  o.cols = static_cast<int>(F.cols);
  return o;
}
GramOperand f64_operand(const double* p, int64_t ld, int cols) {
  GramOperand o;
  o.f64 = p;
  o.ld = ld;
  o.cols = cols;
  return o;
}

// out (D x kk, row-major fp64) = A^T X for X (n_loc x kk, row-major)
void transposed_product(Ctx& c, const ClsData& d, const double* X, int kk, double* out) {
  if (d.S) {
    KS_CUDA(cudaMemsetAsync(out, 0, sizeof(double) * static_cast<size_t>(d.D) * kk, c.st));
    sparse_product(c, *d.S, true, X, kk, nullptr, out, c.st);
  } else {
    const GramOperand a = dense_operand(*d.F), b = f64_operand(X, kk, kk);
    gram_f64(c, a, &b, d.n_loc, out, kk);
  }
}

// the host's labels: class counts and the number outside [0, k)
void count_labels(const int32_t* labels, int64_t n, int k, std::vector<double>& counts, double* bad) {
  counts.assign(k, 0.0);
  *bad = 0.0;
  for (int64_t i = 0; i < n; ++i) {
    if (labels[i] < 0 || labels[i] >= k) *bad += 1.0;
    else counts[labels[i]] += 1.0;
  }
}

std::unique_ptr<Model> new_class_model(int64_t D, int k, int bs) {
  auto model = std::make_unique<Model>();
  model->block_size = bs;
  model->k = k;
  model->has_mean = false;
  model->intercept.alloc(sizeof(double) * k);
  for (int64_t c0 = 0; c0 < D; c0 += bs) {
    const int64_t b = std::min<int64_t>(D, c0 + bs) - c0;
    model->brows.push_back(b);
    auto Wj = std::make_unique<DevBuf>();
    Wj->alloc(sizeof(double) * static_cast<size_t>(b) * k);
    model->W.push_back(std::move(Wj));
  }
  return model;
}

void finish_model(Ctx& c, Model& m) {
  if (!c.host_mirror) return;
  model_alloc_host(m);
  for (size_t j = 0; j < m.W.size(); ++j) model_block_to_host(m, static_cast<int>(j), c.st);
  model_intercept_to_host(m, c.st);
}

}  // namespace

// ------------------------------------------------------------------------------------ logistic regression
namespace {

// Breeze's StrongWolfeLineSearch(maxZoomIter = 10, maxLineSearchIter = 10) as DESIGN.md section 22 restates it
struct LsPoint {
  double t, f, dd;
};
constexpr double kC1 = 1e-4, kC2 = 0.9;
constexpr int kMaxZoom = 10, kMaxBracket = 10;

double interp(const LsPoint& l, const LsPoint& r) {  // l.t < r.t; safeguarded cubic, clamped to [l + 0.1 w, l + 0.9 w]
  const double d1 = l.dd + r.dd - 3.0 * (l.f - r.f) / (l.t - r.t);
  const double rad = d1 * d1 - l.dd * r.dd;
  const double w = r.t - l.t;
  if (!(rad >= 0.0)) return l.t + 0.5 * w;
  const double d2 = std::sqrt(rad);
  const double t = r.t - w * (r.dd + d2 - d1) / (r.dd - l.dd + 2.0 * d2);
  if (!std::isfinite(t)) return l.t + 0.5 * w;
  return std::min(std::max(t, l.t + 0.1 * w), l.t + 0.9 * w);
}

}  // namespace

int64_t fit_logistic(Ctx& c, int64_t features, int64_t sparse, const int32_t* labels, int64_t n_labels, int k, double lam, int num_iter,
                     double tol) {
  const ClsData d = cls_data(c, features, sparse, n_labels, labels, k);
  if (num_iter < 1) throw KsError{KS_ERR_INVALID, "numIterations must be >= 1"};
  if (!(lam >= 0.0) || !std::isfinite(lam)) throw KsError{KS_ERR_INVALID, "regParam must be finite and >= 0"};
  if (!(tol >= 0.0) || !std::isfinite(tol)) throw KsError{KS_ERR_INVALID, "convergenceTol must be finite and >= 0"};
  const int64_t n_loc = d.n_loc, D = d.D;
  const int kk = k - 1;
  const int m = 10;  // MLlib's LBFGS default number of corrections
  const int bs = static_cast<int>(std::min<int64_t>(D, 4096));
  const int nb = static_cast<int>((D + bs - 1) / bs);
  const int64_t n = D * kk;
  cudaStream_t st = c.st;
  const auto host_t0 = std::chrono::steady_clock::now();
  c.spans.clear();
  const int64_t launches0 = c.launches;
  cudaEvent_t ev0 = c.get_event(), ev1 = c.get_event();
  c.fit_events.push_back(ev0);
  c.fit_events.push_back(ev1);
  KS_CUDA(cudaEventRecord(ev0, st));

  // ---- global row count and the label check, rejected on every rank together
  c.span_begin(PH_OTHER);
  std::vector<double> counts;
  double cnt_host[2] = {static_cast<double>(n_loc), 0.0};
  count_labels(labels, n_loc, k, counts, &cnt_host[1]);
  DevBuf cnt, lab;
  cnt.alloc(sizeof(double) * 2);
  KS_CUDA(cudaMemcpyAsync(cnt.p, cnt_host, sizeof(cnt_host), cudaMemcpyHostToDevice, st));
  c.allreduce_f64(cnt.as<double>(), 2);
  KS_CUDA(cudaMemcpyAsync(cnt_host, cnt.p, sizeof(cnt_host), cudaMemcpyDeviceToHost, st));
  KS_CUDA(cudaStreamSynchronize(st));
  c.span_end();
  if (cnt_host[1] != 0.0) throw KsError{KS_ERR_INVALID, "a label lies outside [0, numClasses)"};
  if (cnt_host[0] < 1) throw KsError{KS_ERR_INVALID, "no training rows"};
  const double n_total = cnt_host[0], inv_n = 1.0 / n_total;

  LbCore core(c, n, m, inv_n, lam);
  core.loss_mul = 1.0;
  const size_t zbytes = sizeof(double) * static_cast<size_t>(std::max<int64_t>(n_loc, 1)) * kk;
  DevBuf Z, Q, R, Xr, Cbuf, lspart, trial;
  lab.alloc(sizeof(int32_t) * static_cast<size_t>(std::max<int64_t>(n_loc, 1)));
  Z.alloc(zbytes);
  Q.alloc(zbytes);
  R.alloc(zbytes);
  Xr.alloc(sizeof(double) * static_cast<size_t>(n));
  Cbuf.alloc(sizeof(double) * static_cast<size_t>(n + 1));  // C = A^T R (D x kk row-major), then the data loss
  lspart.alloc(sizeof(double) * 2 * kRedBlocks);
  trial.alloc(sizeof(double) * 2);
  double* C = Cbuf.as<double>();
  double* lsum = C + n;
  if (n_loc > 0) KS_CUDA(cudaMemcpyAsync(lab.p, labels, sizeof(int32_t) * n_loc, cudaMemcpyHostToDevice, st));
  KS_CUDA(cudaMemsetAsync(Z.p, 0, Z.bytes, st));
  KS_CUDA(cudaMemsetAsync(Q.p, 0, Q.bytes, st));

  double t_ls = 0;  // host-clock ms of the line searches (device work and reads)
  // Z += alpha Q (with_q), R, the data loss; C = A^T R; one all-reduce of [C | loss]; g, y, s.y, y.y and f through LbCore
  auto accept_pass = [&](bool with_q, int h) {
    c.span_begin(PH_FEATURIZE);
    lr_accept_kernel<<<kRedBlocks, kRedThreads, 0, st>>>(Z.as<double>(), with_q ? Q.as<double>() : nullptr, core.scp(SC_ALPHA),
                                                         lab.as<int32_t>(), n_loc, kk, R.as<double>(), lspart.as<double>());
    lb_finish_kernel<<<1, kRedThreads, 0, st>>>(lspart.as<double>(), kRedBlocks, 0, lsum, nullptr, nullptr, 1.0);
    c.launches += 2;
    c.span_end();
    c.span_begin(PH_GRAM);
    transposed_product(c, d, R.as<double>(), kk, C);
    c.span_end();
    c.span_begin(PH_ALLREDUCE);
    c.allreduce_f64(C, static_cast<size_t>(n + 1));
    c.span_end();
    core.new_gradient<double>(C, kk, nullptr, nullptr, nullptr, D, kk, bs, lsum, h);
  };
  // one line-search trial at step t: (data loss, phi'_data) summed over all ranks, divided by N
  double host_trial[2];
  auto trial_eval = [&](double t, double* f_out, double* dd_out, double WW, double WP, double PP) {
    c.span_begin(PH_OTHER);
    lr_trial_kernel<<<kRedBlocks, kRedThreads, 0, st>>>(Z.as<double>(), Q.as<double>(), t, lab.as<int32_t>(), n_loc, kk, lspart.as<double>());
    lb_finish_kernel<<<1, kRedThreads, 0, st>>>(lspart.as<double>(), kRedBlocks, 0, trial.as<double>(), nullptr, nullptr, 1.0);
    lb_finish_kernel<<<1, kRedThreads, 0, st>>>(lspart.as<double>() + kRedBlocks, kRedBlocks, 0, trial.as<double>() + 1, nullptr, nullptr, 1.0);
    c.launches += 3;
    c.span_end();
    c.span_begin(PH_ALLREDUCE);
    c.allreduce_f64(trial.as<double>(), 2);
    c.span_end();
    KS_CUDA(cudaMemcpyAsync(host_trial, trial.p, sizeof(host_trial), cudaMemcpyDeviceToHost, st));
    KS_CUDA(cudaStreamSynchronize(st));
    *f_out = host_trial[0] * inv_n + 0.5 * lam * (WW + 2.0 * t * WP + t * t * PP);
    *dd_out = host_trial[1] * inv_n + lam * (WP + t * PP);
  };

  // ---- f(W_0), g(W_0)
  accept_pass(false, -1);
  const bool nothing_to_do = core.start();
  std::vector<int> ls_evals;
  bool failed_once = false;
  int t = 0;
  while (t < num_iter && !nothing_to_do) {
    // ---- direction, <W, P>, P row-major for the products
    c.span_begin(PH_SOLVE);
    core.direction();
    core.lin(nullptr, LbTerm{core.P.as<double>()}, LbTerm{}, nullptr, 1, core.W.as<double>(), nullptr);
    core.finish(core.part.as<double>(), kRedBlocks, 0, SC_WP);
    for (int j = 0; j < nb; ++j) {
      const int64_t c0 = static_cast<int64_t>(j) * bs;
      launch_rows_from_block(c, core.P.as<double>() + c0 * kk, std::min<int64_t>(D, c0 + bs) - c0, kk, c0, Xr.as<double>(), st);
    }
    c.span_end();
    // ---- Q = A P
    c.span_begin(PH_UPDATE);
    if (n_loc > 0) {
      if (d.S) {
        KS_CUDA(cudaMemsetAsync(Q.p, 0, Q.bytes, st));
        sparse_product(c, *d.S, false, Xr.as<double>(), kk, nullptr, Q.as<double>(), st);
      } else {
        skinny_f64(c, dense_operand(*d.F), n_loc, Xr.as<double>(), kk, kk, Q.as<double>(), kk);
      }
    }
    c.span_end();
    double s8[SC_WP - SC_GG + 1], reset = 0;
    KS_CUDA(cudaMemcpyAsync(s8, core.scp(SC_GG), sizeof(s8), cudaMemcpyDeviceToHost, st));
    KS_CUDA(cudaMemcpyAsync(&reset, core.scp(SC_RESET), sizeof(double), cudaMemcpyDeviceToHost, st));
    KS_CUDA(cudaStreamSynchronize(st));
    const double GG = s8[0], GP = s8[SC_GP - SC_GG], PP = s8[SC_PP - SC_GG], WW = s8[SC_WW - SC_GG], WP = s8[SC_WP - SC_GG];
    if (reset != 0.0) core.order.clear();

    // ---- the line search (host), every rank on the same all-reduced scalars
    const auto ls_t0 = std::chrono::steady_clock::now();
    const LsPoint p0{0.0, core.losses.back(), GP};
    int evals = 0;
    double alpha = 0.0;
    bool ok = false;
    auto phi = [&](double s) {
      LsPoint p{s, 0.0, 0.0};
      trial_eval(s, &p.f, &p.dd, WW, WP, PP);
      ++evals;
      return p;
    };
    auto suff_fails = [&](const LsPoint& p, const LsPoint& low) {
      return !std::isfinite(p.f) || p.f > p0.f + kC1 * p.t * p0.dd || p.f >= low.f;
    };
    auto zoom = [&](LsPoint low, LsPoint hi) {
      for (int i = 0; i < kMaxZoom; ++i) {
        const double s = low.t > hi.t ? interp(hi, low) : interp(low, hi);
        const LsPoint q = phi(s);
        if (suff_fails(q, low)) {
          hi = q;
        } else {
          if (std::fabs(q.dd) <= kC2 * std::fabs(p0.dd)) {
            alpha = q.t;
            return true;
          }
          if (q.dd * (hi.t - low.t) >= 0.0) hi = low;
          low = q;
        }
      }
      return false;
    };
    if (p0.dd < 0.0) {
      double s = t == 0 ? 1.0 / std::sqrt(PP) : 1.0;
      LsPoint low = p0;
      for (int i = 0; i < kMaxBracket; ++i) {
        const LsPoint q = phi(s);
        if (!std::isfinite(q.f) || q.f > p0.f + kC1 * s * p0.dd || (q.f >= low.f && i > 0)) {
          ok = zoom(low, q);
          break;
        }
        if (std::fabs(q.dd) <= kC2 * std::fabs(p0.dd)) {
          alpha = q.t;
          ok = true;
          break;
        }
        if (q.dd >= 0.0) {
          ok = zoom(q, low);
          break;
        }
        low = q;
        s *= 1.5;
      }
    }
    ls_evals.push_back(evals);
    t_ls += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - ls_t0).count();
    if (ok && alpha * std::sqrt(GG) < 1e-10) ok = false;  // Breeze's step-size underflow
    if (!ok) {
      if (failed_once) {
        core.stop = "line_search_failed";
        break;
      }
      failed_once = true;  // drop the history and retry this iteration from -g
      core.order.clear();
      continue;
    }

    // ---- W += alpha P, s = alpha P, Z += alpha Q, R, C, g
    c.span_begin(PH_SOLVE);
    launch_set_f64(core.scp(SC_ALPHA), alpha, st);
    c.launches += 1;
    const int h = core.take_step();
    c.span_end();
    accept_pass(true, h);
    if (core.accept(t, h, num_iter, tol)) break;
    ++t;
  }

  // ---- the model: d x k, column 0 zeros (the pivot class), columns 1 .. k-1 = W, no intercept, no means
  auto model = new_class_model(D, k, bs);
  model->has_intercept = false;
  KS_CUDA(cudaMemsetAsync(model->intercept.p, 0, model->intercept.bytes, st));
  for (int j = 0; j < nb; ++j) {
    const int64_t c0 = static_cast<int64_t>(j) * bs, b = model->brows[j];
    double* Wj = model->W[j]->as<double>();
    KS_CUDA(cudaMemsetAsync(Wj, 0, sizeof(double) * b, st));
    KS_CUDA(cudaMemcpyAsync(Wj + b, core.W.as<double>() + c0 * kk, sizeof(double) * b * kk, cudaMemcpyDeviceToDevice, st));
  }
  finish_model(c, *model);
  KS_CUDA(cudaEventRecord(ev1, st));
  c.check_async("LogisticRegressionEstimator.fit");
  float total_ms = 0;
  cudaEventElapsedTime(&total_ms, ev0, ev1);
  double ms[PH_COUNT];
  c.collect_spans(ms);
  for (cudaEvent_t e : c.fit_events) c.event_pool.push_back(e);
  c.fit_events.clear();
  std::ostringstream js;
  js.precision(17);
  js << "{\"solver\":\"logistic_regression\",\"input\":\"" << (d.S ? "sparse" : "dense") << "\",\"n_local\":" << n_loc
     << ",\"n_total\":" << static_cast<int64_t>(n_total) << ",\"d\":" << D << ",\"k\":" << k << ",\"num_corrections\":" << m
     << ",\"world\":" << c.world;
  core.history_json(js);
  js << ",\"line_search_evals\":[";
  for (size_t q = 0; q < ls_evals.size(); ++q) js << (q ? "," : "") << ls_evals[q];
  js << "],\"total_ms\":" << total_ms << ",\"ap_ms\":" << ms[PH_UPDATE] << ",\"atr_ms\":" << ms[PH_GRAM]
     << ",\"products_ms\":" << (ms[PH_UPDATE] + ms[PH_GRAM]) << ",\"line_search_ms\":" << ms[PH_OTHER]
     << ",\"softmax_ms\":" << ms[PH_FEATURIZE] << ",\"recursion_ms\":" << ms[PH_SOLVE] << ",\"allreduce_ms\":" << ms[PH_ALLREDUCE] << ",\"line_search_host_ms\":" << t_ls
     << ",\"launches\":" << (c.launches - launches0) << ",\"host_ms\":"
     << std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count() << "}";
  c.stats_json = js.str();
  return c.add(std::move(model));
}

// ------------------------------------------------------------------------------------ naive Bayes
int64_t fit_naive_bayes(Ctx& c, int64_t features, int64_t sparse, const int32_t* labels, int64_t n_labels, int k, double lam) {
  const ClsData d = cls_data(c, features, sparse, n_labels, labels, k);
  if (!(lam >= 0.0) || !std::isfinite(lam)) throw KsError{KS_ERR_INVALID, "lambda must be finite and >= 0"};
  const int64_t n_loc = d.n_loc, D = d.D;
  const int bs = static_cast<int>(std::min<int64_t>(D, 4096));
  cudaStream_t st = c.st;
  const auto host_t0 = std::chrono::steady_clock::now();
  c.spans.clear();
  const int64_t launches0 = c.launches;
  cudaEvent_t ev0 = c.get_event(), ev1 = c.get_event();
  c.fit_events.push_back(ev0);
  c.fit_events.push_back(ev1);
  KS_CUDA(cudaEventRecord(ev0, st));

  // [S (D x k) | n_c (k) | labels outside [0, k) | negative-value flag], all-reduced once
  std::vector<double> tail;
  double bad = 0.0;
  count_labels(labels, n_loc, k, tail, &bad);
  tail.push_back(bad);
  tail.push_back(0.0);
  const size_t ns = static_cast<size_t>(D) * k;
  DevBuf buf, lab, Y, log_t;
  buf.alloc(sizeof(double) * (ns + k + 2));
  double* S = buf.as<double>();
  double* cnts = S + ns;
  double* neg = cnts + k + 1;
  KS_CUDA(cudaMemcpyAsync(cnts, tail.data(), sizeof(double) * tail.size(), cudaMemcpyHostToDevice, st));
  c.span_begin(PH_OTHER);
  lab.alloc(sizeof(int32_t) * static_cast<size_t>(std::max<int64_t>(n_loc, 1)));
  Y.alloc(sizeof(double) * static_cast<size_t>(std::max<int64_t>(n_loc, 1)) * k);
  if (n_loc > 0) {
    KS_CUDA(cudaMemcpyAsync(lab.p, labels, sizeof(int32_t) * n_loc, cudaMemcpyHostToDevice, st));
    nb_onehot_kernel<<<static_cast<unsigned>((n_loc * k + 255) / 256), 256, 0, st>>>(lab.as<int32_t>(), n_loc, k, Y.as<double>());
    c.launches += 1;
    if (d.S) {
      if (d.S->nnz > 0) {
        nb_negative_flag_kernel<double><<<264, 256, 0, st>>>(d.S->values.as<double>(), d.S->nnz, 1, 1, neg);
        c.launches += 1;
      }
    } else {
      nb_negative_flag_kernel<float><<<264, 256, 0, st>>>(d.F->d, n_loc, D, d.F->ld, neg);
      c.launches += 1;
    }
  }
  c.span_end();
  c.span_begin(PH_GRAM);
  transposed_product(c, d, Y.as<double>(), k, S);
  c.span_end();
  c.span_begin(PH_ALLREDUCE);
  c.allreduce_f64(buf.as<double>(), ns + k + 2);
  c.span_end();
  KS_CUDA(cudaMemcpyAsync(tail.data(), cnts, sizeof(double) * tail.size(), cudaMemcpyDeviceToHost, st));
  KS_CUDA(cudaStreamSynchronize(st));
  if (tail[k] != 0.0) throw KsError{KS_ERR_INVALID, "a label lies outside [0, numClasses)"};
  if (tail[k + 1] != 0.0) throw KsError{KS_ERR_INVALID, "naive Bayes needs non-negative feature values (a value is negative or NaN)"};
  for (int q = 0; q < k; ++q)
    if (tail[q] == 0.0) throw KsError{KS_ERR_INVALID, "class " + std::to_string(q) + " has no training rows"};

  auto model = new_class_model(D, k, bs);
  model->has_intercept = true;
  c.span_begin(PH_SOLVE);
  log_t.alloc(sizeof(double) * k);
  nb_totals_kernel<<<k, kRedThreads, 0, st>>>(S, cnts, D, k, lam, log_t.as<double>(), model->intercept.as<double>());
  c.launches += 1;
  for (size_t j = 0; j < model->W.size(); ++j) {
    const int64_t b = model->brows[j];
    nb_theta_kernel<<<static_cast<unsigned>((b * k + 255) / 256), 256, 0, st>>>(S, log_t.as<double>(), static_cast<int64_t>(j) * bs, b, k, lam,
                                                                              model->W[j]->as<double>());
    c.launches += 1;
  }
  c.span_end();
  finish_model(c, *model);
  KS_CUDA(cudaEventRecord(ev1, st));
  c.check_async("NaiveBayesEstimator.fit");
  float total_ms = 0;
  cudaEventElapsedTime(&total_ms, ev0, ev1);
  double ms[PH_COUNT];
  c.collect_spans(ms);
  for (cudaEvent_t e : c.fit_events) c.event_pool.push_back(e);
  c.fit_events.clear();
  double n_total = 0.0;
  for (int q = 0; q < k; ++q) n_total += tail[q];
  std::ostringstream js;
  js.precision(17);
  js << "{\"solver\":\"naive_bayes\",\"input\":\"" << (d.S ? "sparse" : "dense") << "\",\"n_local\":" << n_loc
     << ",\"n_total\":" << static_cast<int64_t>(n_total) << ",\"d\":" << D << ",\"k\":" << k << ",\"world\":" << c.world
     << ",\"total_ms\":" << total_ms << ",\"products_ms\":" << ms[PH_GRAM] << ",\"allreduce_ms\":" << ms[PH_ALLREDUCE]
     << ",\"finish_ms\":" << ms[PH_SOLVE] << ",\"other_ms\":" << ms[PH_OTHER] << ",\"launches\":" << (c.launches - launches0)
     << ",\"host_ms\":" << std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count() << "}";
  c.stats_json = js.str();
  return c.add(std::move(model));
}

}  // namespace ks
