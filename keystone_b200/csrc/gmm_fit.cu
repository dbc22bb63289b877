// Gaussian-mixture EM and k-means++ on the device: GaussianMixtureModelEstimator, KMeansPlusPlusEstimator / KMeansModel and the row
// gather behind ColumnSampler (K/nodes/learning/{GaussianMixtureModelEstimator,KMeansPlusPlus}.scala, K/nodes/stats/Sampling.scala).
// DESIGN.md section 17.
//
//   E-step      gmm_posterior_kernel (fisher.cu) with the Xerox log-sum-exp epilogue; k-means assignment is the same kernel with the
//               one-hot epilogue on unit variances.
//   Statistics  [X | X o X | 1]^T Q by fv_stats_kernel (fisher.cu) over P pseudo-items of rows per posterior chunk, the P partial
//               blocks summed in a fixed order, the chunks accumulated in chunk order.
//   M-step      one CTA per component: w, mu, var (floored), 0.5 / var and ck into a second parameter buffer; the host swaps the two
//               buffers when the step is accepted.  It reads back K qSums and the cost per iteration.
//   k-means++   one pass per centre: d_n = min(d_n, 1/2 |x_n - c|^2) and per-block sums; the host picks the block, the device the row.
// No float atomics: a repeated fit returns identical bits.
#include "engine.h"

#include <math.h>

#include <algorithm>
#include <chrono>
#include <sstream>
#include <vector>

namespace ks {

static constexpr int kEpiLse = 1, kEpiAssign = 2;
static constexpr int kSumRows = 256;  // rows per block of the fixed-order sums (k-means++ weights, costs)

// ----------------------------------------------------------------------------------------------------------------- kernels
// Block b sums x[256 b, 256 b + 256) (zeros past n) by the tree red[t] += red[t + h], h = 128, 64, ..., 1 -> part[b].
__device__ __forceinline__ double block_tree_sum(double v, double* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int h = kSumRows / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] = red[threadIdx.x] + red[threadIdx.x + h];
    __syncthreads();
  }
  return red[0];
}

__global__ void __launch_bounds__(kSumRows) block_sum_kernel(const double* __restrict__ x, int64_t n, double* __restrict__ part) {
  __shared__ double red[kSumRows];
  const int64_t i = static_cast<int64_t>(blockIdx.x) * kSumRows + threadIdx.x;
  const double s = block_tree_sum(i < n ? x[i] : 0.0, red);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

// k-means++: d[n] = min(d[n], 1/2 sum_d (x_nd - c_d)^2) (first: d[n] = the distance) with c = row seeds[j] of X, the sum over d in
// order without fused multiply-adds; part[b] = the block's tree sum of the new d.
__global__ void __launch_bounds__(kSumRows) kmpp_update_kernel(const float* __restrict__ X, int64_t ldx, int64_t n, int D,
                                                               const int64_t* __restrict__ seeds, int j, int first, double* __restrict__ d,
                                                               double* __restrict__ part) {
  __shared__ double red[kSumRows];
  extern __shared__ double cen[];
  const float* crow = X + seeds[j] * ldx;
  for (int e = threadIdx.x; e < D; e += kSumRows) cen[e] = static_cast<double>(crow[e]);
  __syncthreads();
  const int64_t i = static_cast<int64_t>(blockIdx.x) * kSumRows + threadIdx.x;
  double v = 0.0;
  if (i < n) {
    const float* x = X + i * ldx;
    double acc = 0.0;
    for (int e = 0; e < D; ++e) {
      const double t = __dsub_rn(static_cast<double>(x[e]), cen[e]);
      acc = __dadd_rn(acc, __dmul_rn(t, t));
    }
    v = 0.5 * acc;
    if (!first) v = fmin(v, d[i]);
    d[i] = v;
  }
  const double s = block_tree_sum(v, red);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

// seeds[j] = the first row n of block b with base + s_n > target, s_n the block's inclusive prefix sum of d in row order; if rounding
// leaves none, the block's last row with d > 0
__global__ void kmpp_pick_kernel(const double* __restrict__ d, int64_t n, int64_t b, double base, double target, int64_t* __restrict__ seeds,
                                 int j) {
  const int64_t r0 = b * kSumRows, r1 = min(n, r0 + kSumRows);
  double s = 0.0;
  int64_t last_pos = r0;
  for (int64_t r = r0; r < r1; ++r) {
    s = s + d[r];
    if (d[r] > 0.0) last_pos = r;
    if (base + s > target) {
      seeds[j] = r;
      return;
    }
  }
  seeds[j] = last_pos;
}

// the unit-variance parameters of a hard assignment: mu[d][k] = row seeds[k] of X (seeds null: leave mu), hiv = 1/2, ck = 0
__global__ void unit_gmm_kernel(const float* __restrict__ X, int64_t ldx, const int64_t* __restrict__ seeds, int D, int K,
                                double* __restrict__ mu, double* __restrict__ hiv, double* __restrict__ ck) {
  const int64_t total = static_cast<int64_t>(D) * K;
  for (int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; t < total; t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int dd = static_cast<int>(t / K), k = static_cast<int>(t % K);
    if (seeds) mu[t] = static_cast<double>(X[seeds[k] * ldx + dd]);
    hiv[t] = 0.5;
    if (dd == 0) ck[k] = 0.0;
  }
}

// acc[e] (=, or += when accumulate) sum_p part[p][e] for p = 0, 1, ..., P - 1 in order
__global__ void stats_sum_kernel(const double* __restrict__ part, int P, int64_t per, double* __restrict__ acc, int accumulate) {
  for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < per; e += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    double s = part[e];
    for (int p = 1; p < P; ++p) s += part[static_cast<int64_t>(p) * per + e];
    acc[e] = accumulate ? acc[e] + s : s;
  }
}

// k-means update (KMeansPlusPlus.scala:167-169): mu[d][k] = S[d][k] / S[2D][k]
__global__ void kmeans_means_kernel(const double* __restrict__ S, int D, int K, double* __restrict__ mu) {
  const int64_t total = static_cast<int64_t>(D) * K;
  for (int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; t < total; t += static_cast<int64_t>(gridDim.x) * blockDim.x)
    mu[t] = S[t] / S[2LL * D * K + t % K];
}

// M-step of component blockIdx.x (GaussianMixtureModelEstimator.scala:180-185, :73-75 for the hard assignment of the k-means start):
// w = qSum / N, mu = (1 / qSum) S1, var = max((1 / qSum) S2 - mu^2, lb), then hiv = 0.5 / var and
// ck = -D/2 log 2 pi - 1/2 sum_d log var + log w with the sum over d by a fixed tree.  Products are rounded separately, as Breeze does.
__global__ void __launch_bounds__(256) gmm_mstep_kernel(const double* __restrict__ S, int D, int K, double n, const double* __restrict__ lb,
                                                        double* __restrict__ mu, double* __restrict__ var, double* __restrict__ hiv,
                                                        double* __restrict__ ck, double* __restrict__ w) {
  __shared__ double red[256];
  const int k = blockIdx.x;
  const double qs = S[2LL * D * K + k], inv = 1.0 / qs;
  double slog = 0.0;
  for (int d = threadIdx.x; d < D; d += 256) {
    const int64_t e = static_cast<int64_t>(d) * K + k;
    const double m = __dmul_rn(inv, S[e]);
    const double v = fmax(__dsub_rn(__dmul_rn(inv, S[static_cast<int64_t>(D + d) * K + k]), __dmul_rn(m, m)), lb[d]);
    mu[e] = m;
    var[e] = v;
    hiv[e] = 0.5 / v;
    slog += log(v);
  }
  red[threadIdx.x] = slog;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double wk = qs / n;
    w[k] = wk;
    ck[k] = -0.5 * static_cast<double>(D) * log(2.0 * M_PI) - 0.5 * red[0] + log(wk);
  }
}

// per-chunk column minima and maxima: part[(2 b) D + d] = min, part[(2 b + 1) D + d] = max over rows [b rpb, (b + 1) rpb)
__global__ void col_minmax_kernel(const float* __restrict__ X, int64_t ldx, int64_t n, int D, int64_t rpb, double* __restrict__ part) {
  const int64_t r0 = blockIdx.x * rpb, r1 = min(n, r0 + rpb);
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    double lo = INFINITY, hi = -INFINITY;
    for (int64_t r = r0; r < r1; ++r) {
      const double v = static_cast<double>(X[r * ldx + d]);
      lo = fmin(lo, v);
      hi = fmax(hi, v);
    }
    part[2LL * blockIdx.x * D + d] = lo;
    part[(2LL * blockIdx.x + 1) * D + d] = hi;
  }
}

__global__ void fill_f64_kernel(double* __restrict__ p, int64_t n, double v) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) p[i] = v;
}

// out row i = in row rows[i], padding columns included (they are zero in both)
__global__ void gather_rows_kernel(const float* __restrict__ in, int64_t ldi, const int64_t* __restrict__ rows, int64_t n,
                                   float* __restrict__ out, int64_t ldo) {
  const int64_t total = n * ldo;
  for (int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; t < total; t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t i = t / ldo, c = t - i * ldo;
    out[t] = c < ldi ? in[rows[i] * ldi + c] : 0.f;
  }
}

// ------------------------------------------------------------------------------------------------------------------ host
static unsigned grid_for(int64_t work, const Ctx& c) {
  return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((work + 255) / 256, 32LL * c.num_sms)));
}

enum GmmPhase { GP_SEED = 0, GP_INIT, GP_ESTEP, GP_STATS, GP_MSTEP, GP_COUNT };

// event pairs per phase, summed when the fit ends
struct PhaseTimer {
  Ctx& c;
  std::vector<std::pair<int, std::pair<cudaEvent_t, cudaEvent_t>>> spans;
  int open = -1;
  explicit PhaseTimer(Ctx& cc) : c(cc) {}
  ~PhaseTimer() {
    for (auto& s : spans) {
      cudaEventDestroy(s.second.first);
      cudaEventDestroy(s.second.second);
    }
  }
  void begin(int ph) {
    end();
    cudaEvent_t a, b;
    KS_CUDA(cudaEventCreate(&a));
    KS_CUDA(cudaEventCreate(&b));
    KS_CUDA(cudaEventRecord(a, c.st));
    spans.push_back({ph, {a, b}});
    open = ph;
  }
  void end() {
    if (open < 0) return;
    KS_CUDA(cudaEventRecord(spans.back().second.second, c.st));
    open = -1;
  }
  void collect(double ms[GP_COUNT]) {
    end();
    KS_CUDA(cudaStreamSynchronize(c.st));
    for (int i = 0; i < GP_COUNT; ++i) ms[i] = 0.0;
    for (auto& s : spans) {
      float t = 0.f;
      KS_CUDA(cudaEventElapsedTime(&t, s.second.first, s.second.second));
      ms[s.first] += t;
    }
  }
};

// workspace of the statistics passes over X for a K-component parameter set
struct StatsPass {
  int D = 0, K = 0, m = 0;
  int64_t n = 0, chunk = 0, P = 1, nchunks = 0;
  DevBuf offs, Q, part, acc, rowv, red;  // acc: m K statistics, then one slot for the row-value sum
  void init(Ctx& c, const Matrix& X, int64_t k) {
    D = static_cast<int>(X.cols);
    K = static_cast<int>(k);
    m = 2 * D + 1;
    n = X.rows;
    Gmm probe;
    probe.k = k;
    chunk = std::min(n, posterior_chunk_rows(probe));
    nchunks = (n + chunk - 1) / chunk;
    // pseudo-items per chunk: about four CTAs per SM of statistics tiles, at least 64 rows each
    P = std::max<int64_t>(1, std::min<int64_t>({4LL * c.num_sms / fv_stats_tiles(D, K), (chunk + 63) / 64, 65535}));
    std::vector<int64_t> h(static_cast<size_t>(nchunks * P + 1));
    for (int64_t ci = 0; ci < nchunks; ++ci) {
      const int64_t r0 = ci * chunk, nr = std::min(chunk, n - r0);
      for (int64_t p = 0; p < P; ++p) h[ci * P + p] = r0 + nr * p / P;
    }
    h.back() = n;
    offs.alloc(sizeof(int64_t) * h.size());
    KS_CUDA(cudaMemcpyAsync(offs.p, h.data(), sizeof(int64_t) * h.size(), cudaMemcpyHostToDevice, c.st));
    KS_CUDA(cudaStreamSynchronize(c.st));  // h is a local
    Q.alloc(sizeof(double) * static_cast<size_t>(chunk * K));
    part.alloc(sizeof(double) * static_cast<size_t>(P * m * K));
    acc.alloc(sizeof(double) * static_cast<size_t>(m * K + 1));
    rowv.alloc(sizeof(double) * static_cast<size_t>(n));
    red.alloc(sizeof(double) * static_cast<size_t>(2 * ((n + kSumRows - 1) / kSumRows + 1)));
  }
  double* stats() const { return acc.as<double>(); }
  double* row_sum() const { return acc.as<double>() + static_cast<int64_t>(m) * K; }

  // statistics of chunk ci from the Q the posterior kernel left
  void reduce_chunk(Ctx& c, const Matrix& X, int64_t ci) {
    const int64_t r0 = ci * chunk;
    launch_fv_stats(c, X, Q.as<double>(), K, r0, offs.as<int64_t>() + ci * P, P, D, K, part.as<double>());
    const int64_t per = static_cast<int64_t>(m) * K;
    stats_sum_kernel<<<grid_for(per, c), 256, 0, c.st>>>(part.as<double>(), static_cast<int>(P), per, stats(), ci > 0 ? 1 : 0);
    c.launches += 1;
  }
  // *row_sum() = sum of rowv[0, n) by block tree sums, level by level
  void sum_rows(Ctx& c) {
    const double* src = rowv.as<double>();
    int64_t len = n;
    double* bufs[2] = {red.as<double>(), red.as<double>() + (n + kSumRows - 1) / kSumRows + 1};
    int which = 0;
    do {
      const int64_t nb = (len + kSumRows - 1) / kSumRows;
      double* dst = nb == 1 ? row_sum() : bufs[which];
      block_sum_kernel<<<static_cast<unsigned>(nb), kSumRows, 0, c.st>>>(src, len, dst);
      c.launches += 1;
      src = dst;
      len = nb;
      which ^= 1;
    } while (len > 1);
  }
  // one pass: E-step (epilogue epi) and statistics, chunk by chunk, then the row-value sum
  void run(Ctx& c, const Gmm& g, const Matrix& X, int epi, PhaseTimer& tm) {
    for (int64_t ci = 0; ci < nchunks; ++ci) {
      const int64_t r0 = ci * chunk, nr = std::min(chunk, n - r0);
      tm.begin(GP_ESTEP);
      launch_gmm_estep(c, g, X, r0, nr, Q.as<double>(), nullptr, 0, epi, rowv.as<double>());
      tm.begin(GP_STATS);
      reduce_chunk(c, X, ci);
    }
    tm.begin(GP_ESTEP);
    sum_rows(c);
  }
};

static std::unique_ptr<Gmm> new_gmm(int64_t dim, int64_t k, double thr) {
  auto g = std::make_unique<Gmm>();
  g->dim = dim;
  g->k = k;
  g->thr = thr;
  g->buf.alloc(sizeof(double) * static_cast<size_t>(4 * dim * k + 2 * k));
  return g;
}
static double* mut(const double* p) { return const_cast<double*>(p); }

static void check_shape(const Matrix& X, int64_t k, const char* who) {
  if (k <= 0) throw KsError{KS_ERR_INVALID, std::string(who) + ": the number of centres must be > 0"};
  if (X.cols <= 0 || X.cols > 1024) throw KsError{KS_ERR_INVALID, std::string(who) + ": dim must be in [1, 1024]"};
  if (X.rows < k) throw KsError{KS_ERR_INVALID, std::string(who) + ": fewer rows than centres"};
  if (X.rows > (int64_t(1) << 40)) throw KsError{KS_ERR_INVALID, std::string(who) + ": too many rows"};
}

// global sums [sum x | sum x^2 | N] through the statistics path with K = 1, Q = 1; throws on non-finite input
static std::vector<double> global_sums(Ctx& c, const Matrix& X, const char* who) {
  StatsPass sp;
  sp.init(c, X, 1);
  fill_f64_kernel<<<grid_for(sp.chunk, c), 256, 0, c.st>>>(sp.Q.as<double>(), sp.chunk, 1.0);
  c.launches += 1;
  for (int64_t ci = 0; ci < sp.nchunks; ++ci) sp.reduce_chunk(c, X, ci);
  std::vector<double> h(static_cast<size_t>(sp.m));
  KS_CUDA(cudaMemcpyAsync(h.data(), sp.stats(), sizeof(double) * h.size(), cudaMemcpyDeviceToHost, c.st));
  c.check_async(who);
  for (double v : h)
    if (!std::isfinite(v)) throw KsError{KS_ERR_INVALID, std::string(who) + ": the input has non-finite values"};
  return h;
}

// k-means++ seeding (KMeansPlusPlus.scala:100-124) with the draw rule of the header; seeds: device array of k rows
static std::vector<int64_t> kmpp_seed(Ctx& c, const Matrix& X, int64_t k, const double* u, int64_t* seeds, const char* who) {
  const int64_t n = X.rows, nb = (n + kSumRows - 1) / kSumRows;
  for (int64_t j = 0; j < k; ++j)
    if (!(u[j] >= 0.0 && u[j] < 1.0)) throw KsError{KS_ERR_INVALID, std::string(who) + ": uniforms must lie in [0, 1)"};
  const int64_t s0 = std::min<int64_t>(static_cast<int64_t>(std::floor(u[0] * static_cast<double>(n))), n - 1);
  KS_CUDA(cudaMemcpyAsync(seeds, &s0, sizeof(int64_t), cudaMemcpyHostToDevice, c.st));
  DevBuf dist, part;
  dist.alloc(sizeof(double) * static_cast<size_t>(n));
  part.alloc(sizeof(double) * static_cast<size_t>(nb));
  HostBuf hp;
  hp.alloc(sizeof(double) * static_cast<size_t>(nb));
  const double* B = static_cast<const double*>(hp.p);
  const size_t smem = sizeof(double) * static_cast<size_t>(X.cols);
  for (int64_t j = 1; j < k; ++j) {
    kmpp_update_kernel<<<static_cast<unsigned>(nb), kSumRows, smem, c.st>>>(X.d, X.ld, n, static_cast<int>(X.cols), seeds,
                                                                            static_cast<int>(j - 1), j == 1 ? 1 : 0, dist.as<double>(),
                                                                            part.as<double>());
    KS_CUDA(cudaMemcpyAsync(hp.p, part.p, sizeof(double) * static_cast<size_t>(nb), cudaMemcpyDeviceToHost, c.st));
    c.launches += 1;
    c.check_async(who);
    double W = 0.0;
    for (int64_t b = 0; b < nb; ++b) W = W + B[b];
    if (!(W > 0.0))
      throw KsError{KS_ERR_INVALID, std::string(who) + ": fewer distinct points than centres (no point left to draw centre " +
                                        std::to_string(j) + " from)"};
    const double target = u[j] * W;
    int64_t pick = -1, last = -1;
    double base = 0.0, pbase = 0.0, lbase = 0.0;
    for (int64_t b = 0; b < nb && pick < 0; ++b) {
      const double next = base + B[b];
      if (B[b] > 0.0) {
        last = b;
        lbase = base;
      }
      if (next > target) {
        pick = b;
        pbase = base;
      }
      base = next;
    }
    if (pick < 0) {
      pick = last;
      pbase = lbase;
    }
    kmpp_pick_kernel<<<1, 1, 0, c.st>>>(dist.as<double>(), n, pick, pbase, target, seeds, static_cast<int>(j));
    c.launches += 1;
  }
  std::vector<int64_t> h(static_cast<size_t>(k));
  KS_CUDA(cudaMemcpyAsync(h.data(), seeds, sizeof(int64_t) * h.size(), cudaMemcpyDeviceToHost, c.st));
  c.check_async(who);
  return h;
}

// counts S[2D][k] and the row-value sum of the last pass; throws naming an empty cluster
static std::vector<double> read_counts(Ctx& c, const StatsPass& sp, const char* who, const char* what) {
  std::vector<double> h(static_cast<size_t>(sp.K + 1));
  KS_CUDA(cudaMemcpyAsync(h.data(), sp.stats() + 2LL * sp.D * sp.K, sizeof(double) * h.size(), cudaMemcpyDeviceToHost, c.st));
  c.check_async(who);
  if (what)
    for (int k = 0; k < sp.K; ++k)
      if (!(h[k] > 0.0)) throw KsError{KS_ERR_INVALID, std::string(who) + ": cluster " + std::to_string(k) + " is empty " + what};
  return h;
}

static std::string json_doubles(const std::vector<double>& v) {
  std::ostringstream o;
  o.precision(17);
  o << "[";
  for (size_t i = 0; i < v.size(); ++i) o << (i ? "," : "") << v[i];
  o << "]";
  return o.str();
}

static void write_fit_stats(Ctx& c, const char* solver, const Matrix& X, int64_t k, int iters, const char* reason,
                            const std::vector<double>& costs, const std::vector<int64_t>& seeds, PhaseTimer& tm, int64_t launches0,
                            const std::chrono::steady_clock::time_point& t0) {
  double ms[GP_COUNT];
  tm.collect(ms);
  std::ostringstream js;
  js.precision(17);
  js << "{\"solver\":\"" << solver << "\",\"n\":" << X.rows << ",\"d\":" << X.cols << ",\"k\":" << k << ",\"iterations\":" << iters
     << ",\"stop_reason\":\"" << reason << "\",\"cost_history\":" << json_doubles(costs) << ",\"seed_rows\":[";
  for (size_t i = 0; i < seeds.size(); ++i) js << (i ? "," : "") << seeds[i];
  js << "],\"seeding_ms\":" << ms[GP_SEED] << ",\"init_ms\":" << ms[GP_INIT] << ",\"estep_ms\":" << ms[GP_ESTEP]
     << ",\"stats_ms\":" << ms[GP_STATS] << ",\"mstep_ms\":" << ms[GP_MSTEP] << ",\"launches\":" << (c.launches - launches0)
     << ",\"host_ms\":" << std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count() << "}";
  c.stats_json = js.str();
}

// unit-variance parameters for hard assignment, centres from seeds (device) or left for the caller
static std::unique_ptr<Gmm> unit_gmm(Ctx& c, const Matrix& X, int64_t k, const int64_t* seeds) {
  auto g = new_gmm(X.cols, k, 0.0);
  unit_gmm_kernel<<<grid_for(X.cols * k, c), 256, 0, c.st>>>(X.d, X.ld, seeds, static_cast<int>(X.cols), static_cast<int>(k), mut(g->mu()),
                                                             mut(g->hiv()), mut(g->ck()));
  c.launches += 1;
  return g;
}

static void kmeans_update(Ctx& c, const StatsPass& sp, Gmm& g) {
  kmeans_means_kernel<<<grid_for(static_cast<int64_t>(sp.D) * sp.K, c), 256, 0, c.st>>>(sp.stats(), sp.D, sp.K, mut(g.mu()));
  c.launches += 1;
}

KmeansResult kmeans_fit(Ctx& c, Matrix& X, int64_t k, int max_iter, double tol, const double* uniforms) {
  const char* who = "KMeansPlusPlusEstimator";
  check_shape(X, k, who);
  if (max_iter < 1) throw KsError{KS_ERR_INVALID, "KMeansPlusPlusEstimator: maxIterations must be >= 1"};
  if (!uniforms) throw KsError{KS_ERR_INVALID, "KMeansPlusPlusEstimator: null uniforms"};
  const auto t0 = std::chrono::steady_clock::now();
  const int64_t launches0 = c.launches;
  PhaseTimer tm(c);
  tm.begin(GP_INIT);
  global_sums(c, X, who);
  DevBuf seeds;
  seeds.alloc(sizeof(int64_t) * static_cast<size_t>(k));
  tm.begin(GP_SEED);
  KmeansResult r;
  r.seeds = kmpp_seed(c, X, k, uniforms, seeds.as<int64_t>(), who);
  auto g = unit_gmm(c, X, k, seeds.as<int64_t>());
  StatsPass sp;
  sp.init(c, X, k);
  std::vector<double> costs;
  const char* reason = "max_iterations";
  // Lloyd passes (KMeansPlusPlus.scala:130-177): the means are updated in every pass, the stopping one included
  while (r.iterations < max_iter) {
    sp.run(c, *g, X, kEpiAssign, tm);
    tm.begin(GP_MSTEP);
    kmeans_update(c, sp, *g);
    const auto h = read_counts(c, sp, who, "after a Lloyd pass");
    costs.push_back(h[k] / static_cast<double>(X.rows));
    ++r.iterations;
    const size_t it = costs.size() - 1;
    if (it > 0 && !((costs[it - 1] - costs[it]) >= tol * std::fabs(costs[it - 1]))) {
      reason = "cost";
      break;
    }
  }
  std::vector<double> mu(static_cast<size_t>(X.cols * k));
  KS_CUDA(cudaMemcpyAsync(mu.data(), g->mu(), sizeof(double) * mu.size(), cudaMemcpyDeviceToHost, c.st));
  c.check_async(who);
  r.means.resize(mu.size());
  for (int64_t d = 0; d < X.cols; ++d)
    for (int64_t j = 0; j < k; ++j) r.means[j * X.cols + d] = mu[d * k + j];
  write_fit_stats(c, "kmeans", X, k, r.iterations, reason, costs, r.seeds, tm, launches0, t0);
  return r;
}

std::unique_ptr<Matrix> kmeans_assign(Ctx& c, Matrix& X, const double* means, int64_t k, int64_t dim) {
  if (!means || k <= 0) throw KsError{KS_ERR_INVALID, "KMeansModel: null means or k <= 0"};
  if (dim != X.cols) throw KsError{KS_ERR_INVALID, "KMeansModel.apply: input columns != model dimension"};
  if (dim > 1024) throw KsError{KS_ERR_INVALID, "KMeansModel: dim must be <= 1024"};
  std::vector<double> h(static_cast<size_t>(dim * k));
  for (int64_t j = 0; j < k; ++j)
    for (int64_t d = 0; d < dim; ++d) {
      const double v = means[j * dim + d];
      if (!std::isfinite(v)) throw KsError{KS_ERR_INVALID, "KMeansModel: means must be finite"};
      h[d * k + j] = v;
    }
  auto g = unit_gmm(c, X, k, nullptr);
  KS_CUDA(cudaMemcpyAsync(mut(g->mu()), h.data(), sizeof(double) * h.size(), cudaMemcpyHostToDevice, c.st));
  auto out = new_matrix(X.rows, k);
  if (out->ld != k) KS_CUDA(cudaMemsetAsync(out->d, 0, out->buf.bytes, c.st));
  const int64_t chunk = std::min(std::max<int64_t>(X.rows, 1), posterior_chunk_rows(*g));
  DevBuf Q, dist;
  Q.alloc(sizeof(double) * static_cast<size_t>(chunk * k));
  dist.alloc(sizeof(double) * static_cast<size_t>(std::max<int64_t>(X.rows, 1)));
  for (int64_t r0 = 0; r0 < X.rows; r0 += chunk)
    launch_gmm_estep(c, *g, X, r0, std::min(chunk, X.rows - r0), Q.as<double>(), out->d + r0 * out->ld, out->ld, kEpiAssign, dist.as<double>());
  c.check_async("KMeansModel.apply");  // h is a local
  return out;
}

int64_t gmm_fit(Ctx& c, Matrix& X, const GmmFitArgs& a, double* means_out, double* vars_out, double* weights_out, int* iterations) {
  const char* who = "GaussianMixtureModelEstimator";
  const int64_t k = a.k, D = X.cols, N = X.rows;
  check_shape(X, k, who);
  if (a.max_iter < 1) throw KsError{KS_ERR_INVALID, "GaussianMixtureModelEstimator: maxIterations must be > 0"};
  if (!(a.min_cluster > 0)) throw KsError{KS_ERR_INVALID, "GaussianMixtureModelEstimator: minClusterSize must be > 0"};
  if (!(a.thr >= 0.0 && a.thr < 1.0 / static_cast<double>(k)))
    throw KsError{KS_ERR_INVALID, "GaussianMixtureModelEstimator: weightThreshold must lie in [0, 1/k) (at or above 1/k a row can be zeroed)"};
  if (!std::isfinite(a.tol) || !std::isfinite(a.small_var) || !(a.abs_var > 0.0) || !std::isfinite(a.abs_var))
    throw KsError{KS_ERR_INVALID, "GaussianMixtureModelEstimator: thresholds must be finite, absoluteVarianceThreshold > 0"};
  if (a.init != 0 && a.init != 1) throw KsError{KS_ERR_INVALID, "GaussianMixtureModelEstimator: unknown initialization method"};
  if (!a.uniforms || !means_out || !vars_out || !weights_out) throw KsError{KS_ERR_INVALID, "GaussianMixtureModelEstimator: null arrays"};
  const auto t0 = std::chrono::steady_clock::now();
  const int64_t launches0 = c.launches;
  PhaseTimer tm(c);
  tm.begin(GP_INIT);
  // global mean and variance (GaussianMixtureModelEstimator.scala:60-64) -> variance floor
  const auto gs = global_sums(c, X, who);
  std::vector<double> lb(static_cast<size_t>(D));
  for (int64_t d = 0; d < D; ++d) {
    const double mean = gs[d] / static_cast<double>(N), var = gs[D + d] / static_cast<double>(N) - mean * mean;
    lb[d] = std::max(a.small_var * var, a.abs_var);
  }
  DevBuf dlb;
  dlb.alloc(sizeof(double) * static_cast<size_t>(D));
  KS_CUDA(cudaMemcpyAsync(dlb.p, lb.data(), sizeof(double) * lb.size(), cudaMemcpyHostToDevice, c.st));
  auto cur = new_gmm(D, k, a.thr), cand = new_gmm(D, k, a.thr);
  auto mstep = [&](const StatsPass& sp, Gmm& g) {
    gmm_mstep_kernel<<<static_cast<unsigned>(k), 256, 0, c.st>>>(sp.stats(), static_cast<int>(D), static_cast<int>(k), static_cast<double>(N),
                                                                dlb.as<double>(), mut(g.mu()), mut(g.var()), mut(g.hiv()), mut(g.ck()),
                                                                mut(g.w()));
    c.launches += 1;
  };
  StatsPass sp;
  sp.init(c, X, k);
  std::vector<int64_t> seeds_h;
  if (a.init == 0) {
    // KMeansPlusPlusEstimator(k, 1).fit(X), then the hard assignment to its updated means (:69-77)
    DevBuf seeds;
    seeds.alloc(sizeof(int64_t) * static_cast<size_t>(k));
    tm.begin(GP_SEED);
    seeds_h = kmpp_seed(c, X, k, a.uniforms, seeds.as<int64_t>(), who);
    auto g = unit_gmm(c, X, k, seeds.as<int64_t>());
    tm.begin(GP_INIT);
    sp.run(c, *g, X, kEpiAssign, tm);
    tm.begin(GP_INIT);
    kmeans_update(c, sp, *g);
    read_counts(c, sp, who, "after the k-means++ Lloyd pass");
    sp.run(c, *g, X, kEpiAssign, tm);
    tm.begin(GP_INIT);
    read_counts(c, sp, who, "in the k-means++ initialisation (the reference divides by zero here)");
    mstep(sp, *cur);
  } else {
    // colMin + U range, 0.1 range^2, 1/k (:81-96), floored (:100-103)
    const double* u = a.uniforms;
    for (int64_t i = 0; i < k * D; ++i)
      if (!(u[i] >= 0.0 && u[i] < 1.0)) throw KsError{KS_ERR_INVALID, "GaussianMixtureModelEstimator: uniforms must lie in [0, 1)"};
    const int64_t nb = std::min<int64_t>(4LL * c.num_sms, N), rpb = (N + nb - 1) / nb, nblk = (N + rpb - 1) / rpb;
    DevBuf part;
    part.alloc(sizeof(double) * static_cast<size_t>(2 * nblk * D));
    col_minmax_kernel<<<static_cast<unsigned>(nblk), 256, 0, c.st>>>(X.d, X.ld, N, static_cast<int>(D), rpb, part.as<double>());
    c.launches += 1;
    std::vector<double> hp(static_cast<size_t>(2 * nblk * D));
    KS_CUDA(cudaMemcpyAsync(hp.data(), part.p, sizeof(double) * hp.size(), cudaMemcpyDeviceToHost, c.st));
    c.check_async(who);
    std::vector<double> lo(static_cast<size_t>(D), INFINITY), hi(static_cast<size_t>(D), -INFINITY);
    for (int64_t b = 0; b < nblk; ++b)
      for (int64_t d = 0; d < D; ++d) {
        lo[d] = std::min(lo[d], hp[2 * b * D + d]);
        hi[d] = std::max(hi[d], hp[(2 * b + 1) * D + d]);
      }
    std::vector<double> h(static_cast<size_t>(4 * D * k + 2 * k));
    double *hmu = h.data(), *hvar = hmu + D * k, *hhiv = hvar + D * k, *hck = hhiv + D * k, *hw = hck + k;
    for (int64_t j = 0; j < k; ++j) {
      double slog = 0.0;
      for (int64_t d = 0; d < D; ++d) {
        const double range = hi[d] - lo[d];
        const double var = std::max(0.1 * (range * range), lb[d]);
        hmu[d * k + j] = u[j * D + d] * range + lo[d];
        hvar[d * k + j] = var;
        hhiv[d * k + j] = 0.5 / var;
        slog += log(var);
      }
      hw[j] = 1.0 / static_cast<double>(k);
      hck[j] = -0.5 * static_cast<double>(D) * log(2.0 * M_PI) - 0.5 * slog + log(hw[j]);
    }
    KS_CUDA(cudaMemcpyAsync(cur->buf.p, h.data(), sizeof(double) * h.size(), cudaMemcpyHostToDevice, c.st));
    c.check_async(who);  // h is a local
  }
  // EM (:106-190)
  std::vector<double> costs;
  const char* reason = "max_iterations";
  int iter = 0;
  std::vector<double> h(static_cast<size_t>(k + 1));
  while (iter < a.max_iter) {
    sp.run(c, *cur, X, kEpiLse, tm);
    tm.begin(GP_MSTEP);
    mstep(sp, *cand);
    KS_CUDA(cudaMemcpyAsync(h.data(), sp.stats() + 2 * D * k, sizeof(double) * h.size(), cudaMemcpyDeviceToHost, c.st));
    c.check_async(who);
    const double cost = h[k] / static_cast<double>(N);
    costs.push_back(cost);
    ++iter;
    if (iter > 1 && !((cost - costs[iter - 2]) >= a.tol * std::fabs(costs[iter - 2]))) {
      reason = "cost";
      break;
    }
    bool small = false;
    for (int64_t j = 0; j < k; ++j) small = small || h[j] < a.min_cluster;
    if (small) {
      reason = "min_cluster_size";
      break;
    }
    std::swap(cur, cand);
  }
  tm.end();
  // the model: GaussianMixtureModel(means.t, vars.t, weights) with the default weightThreshold (:192)
  std::vector<double> p(static_cast<size_t>(2 * D * k + k));
  KS_CUDA(cudaMemcpyAsync(p.data(), cur->mu(), sizeof(double) * 2 * D * k, cudaMemcpyDeviceToHost, c.st));
  KS_CUDA(cudaMemcpyAsync(p.data() + 2 * D * k, cur->w(), sizeof(double) * k, cudaMemcpyDeviceToHost, c.st));
  c.check_async(who);
  for (int64_t d = 0; d < D; ++d)
    for (int64_t j = 0; j < k; ++j) {
      means_out[d + D * j] = p[d * k + j];
      vars_out[d + D * j] = p[D * k + d * k + j];
    }
  for (int64_t j = 0; j < k; ++j) weights_out[j] = p[2 * D * k + j];
  if (iterations) *iterations = iter;
  write_fit_stats(c, "gmm", X, k, iter, reason, costs, seeds_h, tm, launches0, t0);
  return gmm_create(c, means_out, vars_out, weights_out, D, k, 1e-4);
}

std::unique_ptr<Matrix> gather_rows(Ctx& c, Matrix& X, const int64_t* rows, int64_t n) {
  if (n < 0 || (n > 0 && !rows)) throw KsError{KS_ERR_INVALID, "gather_rows: null rows or negative count"};
  for (int64_t i = 0; i < n; ++i)
    if (rows[i] < 0 || rows[i] >= X.rows) throw KsError{KS_ERR_INVALID, "gather_rows: row index out of range"};
  auto out = new_matrix(n, X.cols);
  if (n > 0) {
    DevBuf d;
    d.alloc(sizeof(int64_t) * static_cast<size_t>(n));
    KS_CUDA(cudaMemcpyAsync(d.p, rows, sizeof(int64_t) * static_cast<size_t>(n), cudaMemcpyHostToDevice, c.st));
    gather_rows_kernel<<<grid_for(n * out->ld, c), 256, 0, c.st>>>(X.d, X.ld, d.as<int64_t>(), n, out->d, out->ld);
    c.launches += 1;
  }
  c.check_async("ColumnSampler");
  return out;
}

}  // namespace ks
