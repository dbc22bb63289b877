// BlockWeightedLeastSquaresEstimator on the device.
//
// Restates K/nodes/learning/BlockWeightedLeastSquares.scala:102-321 (trainWithL2) with the same per-block statistics,
// computed from class-contiguous row ranges instead of one-class-per-partition RDDs:
//   * groupByClasses (:333-370)  -> stable sort of the rows by class on the host + device row gather (only when the
//                                   rows are not already class-contiguous with every class in one run, :111-131)
//   * (A^T A, A^T R) treeReduce (:212-214) and the per-class covariances (:248-251)
//                                -> ONE Gram pass per class row range with the tensor-core Gram kernel; the population
//                                   Gram is the sum of the class Grams (the reference computes both separately)
//   * per-class  W_c = (jointXTX + lambda I) \ (jointXTR - lambda W_old[:, c])  (:259-273)
//                                -> fp64 assembly kernels + cuSOLVER Cholesky, one b x b system per class
//   * residual update (:287-290) -> the same EPI_UPDATE GEMM as BlockLS
// Features are shifted by an estimate m of the population mean before the (tf32) Gram; every quantity the reference
// defines on raw features is recovered exactly in fp64 from (m, column sums, Gram of the shifted block).
// Multi-rank: rows are sharded BY CLASS (each class on exactly one rank, checked); population statistics and the solved
// columns are all-reduced.  Class Grams of one block are kept resident (classes_on_rank * b * b * 4 bytes).
// Operand modes: KS_PRECISION_TF32 (one tf32 MMA per product; KS_PRECISION_F16 is accepted and computes the same way) and
// KS_PRECISION_F16X2, the parity mode: slab, residual and increment are carried as tf32 hi + lo pairs (products keep
// hi*hi + hi*lo + lo*hi; generated features come from the split fp16 projection), which doubles the resident class Grams;
// the diagonals of the class and population Grams are then taken in fp64 from the pairs (launch_colsumsq_pair).
// The per-class Cholesky solves are independent: they run on kSolveLanes streams with one cuSOLVER handle each.
#include "engine.h"

#include <algorithm>
#include <numeric>

namespace ks {

// ------------------------------------------------------------------------------------ kernels
__global__ void gather_rows_kernel(const float* __restrict__ src, int64_t ld, const int32_t* __restrict__ perm,
                                   float* __restrict__ dst, int64_t rows) {
  const int64_t total = rows * (ld / 4);
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / (ld / 4), c4 = i - r * (ld / 4);
    reinterpret_cast<float4*>(dst + r * ld)[c4] = reinterpret_cast<const float4*>(src + static_cast<int64_t>(perm[r]) * ld)[c4];
  }
}
// out[f] = sum_ci parts[ci][f]   (parts: n rows of ld doubles)
__global__ void sum_parts_f64_kernel(const double* __restrict__ parts, int n, int64_t ld, double* __restrict__ out, int b) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= b) return;
  double s = 0.0;
  for (int i = 0; i < n; ++i) s += parts[static_cast<int64_t>(i) * ld + f];
  out[f] = s;
}
__global__ void add_f32_kernel(const float* __restrict__ a, float* __restrict__ acc, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    acc[i] += a[i];
}
// Cpop += Ctmp ; xtr[f] = Ctmp[f][c]
__global__ void bwls_accum_kernel(const float* __restrict__ Ctmp, float* __restrict__ Cpop, int ldc, float* __restrict__ xtr,
                                  int c, int b, int k) {
  const int64_t total = static_cast<int64_t>(b) * ldc;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float v = Ctmp[i];
    Cpop[i] += v;
    const int f = static_cast<int>(i / ldc), col = static_cast<int>(i - static_cast<int64_t>(f) * ldc);
    if (col == c) xtr[f] = v;
  }
}
// delta vectors from column sums (fp64 sums, count)
__global__ void bwls_means_kernel(const double* __restrict__ sum, double count, double* __restrict__ out, int b) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < b) out[i] = sum[i] / count;
}
// H = (1-w) (Gpop/N - dp dp^T) + w (Gc/nc - dc dc^T) + w(1-w) (dc-dp)(dc-dp)^T + lam I     (:216, :248-261, :272)
// Xpop / Xc (split-operand mode, else null): full b x b cross Grams S_hi^T S_lo; the Gram of S = S_hi + S_lo is
// S_hi^T S_hi + X + X^T (the lo x lo term, ~2^-22 of the diagonal, is dropped)
// diag_pop / diag_c (split-operand mode, else null): the Gram diagonals in fp64 (launch_colsumsq_pair), used instead of the
// tensor core's, whose all-positive accumulation chains are biased low
__global__ void bwls_build_kernel(const float* __restrict__ Gpop, const float* __restrict__ Gc, int ldg,
                                  const double* __restrict__ dp, const double* __restrict__ dc, double N, double nc, double w,
                                  double lam, double* __restrict__ H, int b, const float* __restrict__ Xpop,
                                  const float* __restrict__ Xc, const double* __restrict__ diag_pop,
                                  const double* __restrict__ diag_c) {
  const int64_t total = static_cast<int64_t>(b) * b;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i / b), r = static_cast<int>(i - static_cast<int64_t>(c) * b);
    const int lo = min(r, c), hi = max(r, c);
    const int64_t gi = static_cast<int64_t>(lo) * ldg + hi;
    double gp = static_cast<double>(Gpop[gi]), gc = static_cast<double>(Gc[gi]);
    if (Xpop) {
      const int64_t a = static_cast<int64_t>(r) * ldg + c, t = static_cast<int64_t>(c) * ldg + r;
      gp += static_cast<double>(Xpop[a]) + static_cast<double>(Xpop[t]);
      gc += static_cast<double>(Xc[a]) + static_cast<double>(Xc[t]);
    }
    if (diag_pop && r == c) {
      gp = diag_pop[r];
      gc = diag_c[r];
    }
    const double pop = gp / N - dp[r] * dp[c];
    const double cls = gc / nc - dc[r] * dc[c];
    const double md = (dc[r] - dp[r]) * (dc[c] - dp[c]);
    H[i] = (1.0 - w) * pop + w * cls + w * (1.0 - w) * md + (r == c ? lam : 0.0);
  }
}
// rhs = (1-w) popXTR[:,c] + w classXTR - jointMean * meanMixtureWt - lam Wold[:,c]                      (:263-273)
// with raw-feature quantities rebuilt from the shifted block:  F^T r = S^T r + m * sum(r)
__global__ void bwls_rhs_kernel(const float* __restrict__ Cpop, int ldc, const float* __restrict__ xtr,
                                const float* __restrict__ m, const double* __restrict__ dp, const double* __restrict__ dc,
                                double N, double nc, const double* __restrict__ rsum_all, const double* __restrict__ rsum_cls,
                                double w, double lam, const double* __restrict__ Wold_col, double* __restrict__ rhs,
                                double* __restrict__ jm_row, int c, int b) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= b) return;
  const double rsum_all_c = rsum_all[c], rsum_cls_c = rsum_cls[c];
  const double mf = static_cast<double>(m[f]);
  const double pop_xtr = (static_cast<double>(Cpop[static_cast<int64_t>(f) * ldc + c]) + mf * rsum_all_c) / N;
  const double cls_xtr = (static_cast<double>(xtr[f]) + mf * rsum_cls_c) / nc;
  const double joint_mean = mf + w * dc[f] + (1.0 - w) * dp[f];  // w classMean + (1-w) popMean   (:201-204)
  const double mix = (rsum_all_c / N) * (1.0 - w) + w * (rsum_cls_c / nc);
  rhs[f] = (1.0 - w) * pop_xtr + w * cls_xtr - joint_mean * mix - lam * Wold_col[f];
  if (jm_row) jm_row[f] = joint_mean;
}
__global__ void copy_col_kernel(const double* __restrict__ src, double* __restrict__ dst, int b) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < b) dst[i] = src[i];
}
__global__ void neg_f32_to_f64_kernel(const float* __restrict__ src, double* __restrict__ dst, int b) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < b) dst[i] = -static_cast<double>(src[i]);
}
// acc[c] += sum_f jm[c][f] * W[f][c]   (W column-major b x k, jm row-major k x b)                       (:316)
__global__ void bwls_final_b_kernel(const double* __restrict__ jm, const double* __restrict__ W, double* __restrict__ acc,
                                    int b, int k) {
  const int c = blockIdx.x;
  __shared__ double red[256];
  double s = 0;
  for (int f = threadIdx.x; f < b; f += blockDim.x) s += jm[static_cast<int64_t>(c) * b + f] * W[static_cast<int64_t>(c) * b + f];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int t = blockDim.x / 2; t > 0; t >>= 1) {
    if (threadIdx.x < t) red[threadIdx.x] += red[threadIdx.x + t];
    __syncthreads();
  }
  if (threadIdx.x == 0) acc[c] += red[0];
}
__global__ void bwls_init_residual_kernel(const float* __restrict__ Y, int64_t ldy, const double* __restrict__ jlm,
                                          float* __restrict__ R, int64_t ldr, int64_t rows, int k) {
  const int64_t total = rows * ldr;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / ldr;
    const int c = static_cast<int>(i - r * ldr);
    R[i] = c < k ? static_cast<float>(static_cast<double>(Y[r * ldy + c]) - jlm[c]) : 0.f;
  }
}
__global__ void final_b_finish_kernel(const double* __restrict__ jlm, const double* __restrict__ acc, double* __restrict__ out, int k) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < k) out[i] = jlm[i] - acc[i];
}

static unsigned grid1d(int64_t n, int threads = 256) {
  int64_t g = (n + threads - 1) / threads;
  return static_cast<unsigned>(std::min<int64_t>(std::max<int64_t>(g, 1), 132 * 16));
}

// ------------------------------------------------------------------------------------ fit
int64_t fit_bwls(Ctx& c, FeatSrc& src, Matrix& Y, int bs, int num_iter, double lam, double w, int64_t nf_opt, int precision) {
  // ks_debug_bwls_capture arms one fit: take the request and disarm before anything can throw
  const int cap_block = c.bwls_cap_block, cap_cls = c.bwls_cap_cls;
  double* const cap_H = c.bwls_cap_H;
  double* const cap_rhs = c.bwls_cap_rhs;
  c.bwls_cap_block = c.bwls_cap_cls = -1;
  c.bwls_cap_H = c.bwls_cap_rhs = nullptr;
  if (bs <= 0 || num_iter < 1) throw KsError{KS_ERR_INVALID, "blockSize must be > 0 and numIter >= 1"};
  if (Y.rows != src.n_rows) throw KsError{KS_ERR_INVALID, "features and labels have different row counts"};
  // Multi-rank: every rank passes the rows of the classes it owns; each class must live on exactly one rank (the
  // reference's one-class-per-partition precondition, :111-124, lifted to ranks).  N is this rank's row count, Ntot the
  // global one; population statistics are all-reduced, per-class statistics and solves stay local, the solved columns are
  // all-reduced into the full dW (the `collect` + `broadcast` of :276, :285).
  const int64_t N = Y.rows;
  const int k = static_cast<int>(Y.cols);
  const int64_t D = nf_opt > 0 ? nf_opt : src.D;
  if (D > src.D || D <= 0 || N < 0) throw KsError{KS_ERR_INVALID, "bad problem size"};
  const int nb = static_cast<int>((D + bs - 1) / bs);
  const int bmax = static_cast<int>(std::min<int64_t>(bs, D));
  const int64_t lds = round_up(bmax, 32), kpad = round_up(k, 32);
  const int ldg = static_cast<int>(lds), ldc = static_cast<int>(kpad);
  cudaStream_t st = c.st;
  const int64_t launches0 = c.launches;
  cudaEvent_t ev0 = c.get_event(), ev1 = c.get_event();
  KS_CUDA(cudaEventRecord(ev0, st));

  // ---- class of every row (argmax of the +-1 indicators, :133-139) and the class-contiguous row order
  DevBuf cls_d;
  cls_d.alloc(sizeof(int32_t) * N);
  launch_argmax_rows(Y.d, Y.ld, N, k, cls_d.as<int32_t>(), st);
  c.launches += 1;
  std::vector<int32_t> cls(N);
  KS_CUDA(cudaMemcpyAsync(cls.data(), cls_d.p, sizeof(int32_t) * N, cudaMemcpyDeviceToHost, st));
  KS_CUDA(cudaStreamSynchronize(st));
  std::vector<int64_t> count(k, 0);
  for (int64_t i = 0; i < N; ++i) {
    if (cls[i] < 0 || cls[i] >= k) throw KsError{KS_ERR_INVALID, "label row " + std::to_string(i) + " has no valid class"};
    count[cls[i]]++;
  }
  // global class sizes / ownership check / global row count
  std::vector<double> gcount(k, 0.0);
  double Ntot_d = static_cast<double>(N);
  {
    std::vector<double> h(2 * k + 1, 0.0);
    for (int cc = 0; cc < k; ++cc) {
      h[cc] = static_cast<double>(count[cc]);
      h[k + cc] = count[cc] > 0 ? 1.0 : 0.0;
    }
    h[2 * k] = static_cast<double>(N);
    if (c.world > 1) {
      DevBuf tmp;
      tmp.alloc(sizeof(double) * h.size());
      KS_CUDA(cudaMemcpyAsync(tmp.p, h.data(), sizeof(double) * h.size(), cudaMemcpyHostToDevice, st));
      c.allreduce_f64(tmp.as<double>(), h.size());
      KS_CUDA(cudaMemcpyAsync(h.data(), tmp.p, sizeof(double) * h.size(), cudaMemcpyDeviceToHost, st));
      KS_CUDA(cudaStreamSynchronize(st));
    }
    for (int cc = 0; cc < k; ++cc) {
      gcount[cc] = h[cc];
      if (h[k + cc] > 1.5)
        throw KsError{KS_ERR_INVALID, "ks_blockwls_fit: class " + std::to_string(cc) + " has rows on more than one rank; every class "
                                      "must be owned by exactly one rank (shard the rows by class)"};
    }
    Ntot_d = h[2 * k];
  }
  if (Ntot_d < 1) throw KsError{KS_ERR_INVALID, "no training rows"};
  bool contiguous = true;  // every class forms one run
  {
    std::vector<char> seen(k, 0);
    for (int64_t i = 0; i < N; ++i)
      if (i == 0 || cls[i] != cls[i - 1]) {
        if (seen[cls[i]]) { contiguous = false; break; }
        seen[cls[i]] = 1;
      }
  }
  std::vector<int32_t> perm(N);
  std::iota(perm.begin(), perm.end(), 0);
  std::stable_sort(perm.begin(), perm.end(), [&](int32_t a, int32_t b) { return cls[a] < cls[b]; });  // groupByClasses
  struct Range { int cls; int64_t off, n; };
  std::vector<Range> ranges;
  {
    int64_t off = 0;
    for (int cc = 0; cc < k; ++cc) {
      if (count[cc] > 0) ranges.push_back({cc, off, count[cc]});
      off += count[cc];
    }
  }
  bool sorted_already = contiguous;
  if (contiguous)  // contiguous runs may still be in a different class order: keep the given order, recompute offsets
  {
    ranges.clear();
    int64_t i = 0;
    while (i < N) {
      int64_t j = i;
      while (j < N && cls[j] == cls[i]) ++j;
      ranges.push_back({cls[i], i, j - i});
      i = j;
    }
  }
  // gathered copies when a reshuffle is needed
  const bool x2 = precision == KS_PRECISION_F16X2;
  Matrix Yg, Xg, Fg;
  Matrix* Yp = &Y;
  FeatSrc gsrc;
  FeatSrc* sp = &src;
  DevBuf perm_d;
  if (!sorted_already) {
    perm_d.alloc(sizeof(int32_t) * N);
    KS_CUDA(cudaMemcpyAsync(perm_d.p, perm.data(), sizeof(int32_t) * N, cudaMemcpyHostToDevice, st));
    auto gather = [&](Matrix& in, Matrix& out) {
      out.rows = in.rows; out.cols = in.cols; out.ld = in.ld;
      out.buf.alloc(sizeof(float) * static_cast<size_t>(in.rows * in.ld));
      out.d = out.buf.as<float>();
      gather_rows_kernel<<<grid1d(in.rows * (in.ld / 4)), 256, 0, st>>>(in.d, in.ld, perm_d.as<int32_t>(), out.d, in.rows);
      c.launches += 1;
    };
    gather(Y, Yg);
    Yp = &Yg;
    if (src.F) {
      gather(*src.F, Fg);
      gsrc.F = &Fg;
      gsrc.D = src.D;
      gsrc.n_rows = src.n_rows;
      gsrc.zeros.alloc(src.zeros.bytes);
      KS_CUDA(cudaMemsetAsync(gsrc.zeros.p, 0, gsrc.zeros.bytes, st));
    } else {
      gather(*src.X, Xg);
      derive_feat_src(c, src, &Xg, gsrc, precision);  // the same feature map (kind included) over the gathered rows
    }
    sp = &gsrc;
  }
  const int ncls = static_cast<int>(ranges.size());
  const size_t g_elems = static_cast<size_t>(bmax) * ldg, c_elems = static_cast<size_t>(bmax) * ldc;
  if (static_cast<double>(g_elems) * 4.0 * ncls * (x2 ? 2 : 1) > 120e9)
    throw KsError{KS_ERR_INVALID, "ks_blockwls_fit: class Grams of one block exceed the resident budget (k * b^2 * 4 B > 120 GB)"};

  // ---- jointLabelMean (:148-156), residual = labels - jointLabelMean (:167-169)
  std::vector<double> jlm(k, 0.0);
  for (int cc = 0; cc < k; ++cc)
    if (gcount[cc] > 0) jlm[cc] = 2 * w + (2 * (1.0 - w) * gcount[cc] / Ntot_d) - 1;
  DevBuf jlm_d, R, Rr, Rlo, slab, slab_lo, sf32, Gcls, Xcls, Gpop, Xpop, Ctmp, Cpop, xtr, shift, negm, psum, csum, rsum_all, rsum_cls,
      dp, dcs, dW, bop, bop_lo, cbias, fsum, facc, fail, diag_cls, diag_pop;
  jlm_d.alloc(sizeof(double) * k);
  KS_CUDA(cudaMemcpyAsync(jlm_d.p, jlm.data(), sizeof(double) * k, cudaMemcpyHostToDevice, st));
  R.alloc(sizeof(float) * static_cast<size_t>(std::max<int64_t>(N, 1) * kpad));
  Rr.alloc(R.bytes);
  bwls_init_residual_kernel<<<grid1d(N * kpad), 256, 0, st>>>(Yp->d, Yp->ld, jlm_d.as<double>(), R.as<float>(), kpad, N, k);
  c.launches += 1;
  slab.alloc(sizeof(float) * static_cast<size_t>(std::max<int64_t>(N, 1) * lds));
  Gcls.alloc(sizeof(float) * g_elems * std::max(ncls, 1));
  Gpop.alloc(sizeof(float) * g_elems);
  if (x2) {
    Rlo.alloc(R.bytes);
    slab_lo.alloc(slab.bytes);
    if (!sp->F) sf32.alloc(slab.bytes);
    Xcls.alloc(Gcls.bytes);
    Xpop.alloc(Gpop.bytes);
    diag_cls.alloc(sizeof(double) * static_cast<size_t>(std::max(ncls, 1)) * lds);
    diag_pop.alloc(sizeof(double) * lds);
  }
  Ctmp.alloc(sizeof(float) * c_elems);
  Cpop.alloc(sizeof(float) * c_elems);
  xtr.alloc(sizeof(float) * static_cast<size_t>(std::max(ncls, 1)) * lds);
  shift.alloc(sizeof(float) * lds);
  negm.alloc(sizeof(double) * lds);
  psum.alloc(sizeof(double) * lds);
  csum.alloc(sizeof(double) * static_cast<size_t>(std::max(ncls, 1)) * lds);
  rsum_all.alloc(sizeof(double) * kpad);
  rsum_cls.alloc(sizeof(double) * static_cast<size_t>(std::max(ncls, 1)) * kpad);
  dp.alloc(sizeof(double) * lds);
  dcs.alloc(sizeof(double) * static_cast<size_t>(std::max(ncls, 1)) * lds);
  dW.alloc(sizeof(double) * (static_cast<size_t>(bmax) * k + 1));  // + one slot: the collective "a Cholesky failed" flag
  bop.alloc(sizeof(float) * static_cast<size_t>(kpad) * lds);
  if (x2) bop_lo.alloc(bop.bytes);
  cbias.alloc(sizeof(float) * kpad);
  facc.alloc(sizeof(double) * k);
  KS_CUDA(cudaMemsetAsync(facc.p, 0, facc.bytes, st));
  if (sp->F) {
    fsum.alloc(sizeof(double) * static_cast<size_t>(sp->F->ld));
    KS_CUDA(cudaMemsetAsync(fsum.p, 0, fsum.bytes, st));
    launch_colsum(sp->F->d, nullptr, sp->F->ld, N, static_cast<int>(sp->F->cols), fsum.as<double>(), st);
    c.launches += 1;
    c.allreduce_f64(fsum.as<double>(), static_cast<size_t>(sp->F->cols));
  }
  // per-class solves: independent b x b systems, spread over the context's solve lanes (stream + cuSOLVER handle each)
  const int nlanes = std::max(1, std::min(c.solve_lanes, std::max(ncls, 1)));
  c.ensure_lanes(nlanes);
  std::unique_ptr<DevBuf[]> laneH(new DevBuf[nlanes]), laneRhs(new DevBuf[nlanes]);
  for (int q = 0; q < nlanes; ++q) {
    laneH[q].alloc(sizeof(double) * static_cast<size_t>(bmax) * bmax);
    laneRhs[q].alloc(sizeof(double) * bmax);
  }
  cudaEvent_t ev_stats = c.get_event();
  std::vector<cudaEvent_t> ev_lane(nlanes);
  for (int q = 0; q < nlanes; ++q) ev_lane[q] = c.get_event();
  c.fit_events.push_back(ev_stats);
  for (auto e : ev_lane) c.fit_events.push_back(e);

  auto model = std::make_unique<Model>();
  model->block_size = bs;
  model->k = k;
  model->has_mean = false;  // means are folded into the intercept (:316-320)
  model->has_intercept = true;
  model->intercept.alloc(sizeof(double) * k);
  std::vector<std::unique_ptr<DevBuf>> shifts(nb), jms(nb);
  // the three product terms of the split mode (hi*hi, lo*hi, hi*lo); plain modes run the first only
  auto gram_c = [&](const float* A, int64_t off, int64_t n, int b, const float* Rop, float* Cout) {
    launch_gram_block(c, A + off * lds, lds, n, b, Rop + off * kpad, kpad, k, nullptr, 0, Cout, ldc, false, true, st, false,
                      x2 ? 2048 : 0);
  };

  for (int it = 0; it < num_iter; ++it) {
    for (int j = 0; j < nb; ++j) {
      const int64_t c0 = static_cast<int64_t>(j) * bs;
      const int b = static_cast<int>(std::min<int64_t>(D, c0 + bs) - c0);
      // ---------------- shift estimate (pass 0) and the shifted, rounded slab over all (class-sorted) rows
      if (it == 0) {
        shifts[j] = std::make_unique<DevBuf>();
        shifts[j]->alloc(sizeof(float) * lds);
        KS_CUDA(cudaMemsetAsync(shifts[j]->p, 0, shifts[j]->bytes, st));
        if (sp->F) {
          // exact population mean of the block
          DevBuf cnt;
          cnt.alloc(sizeof(double));
          const double nd = Ntot_d;
          KS_CUDA(cudaMemcpyAsync(cnt.p, &nd, sizeof(double), cudaMemcpyHostToDevice, st));
          launch_divide_by_count(fsum.as<double>() + c0, cnt.as<double>(), shifts[j]->as<float>(), nullptr, b, st);
          KS_CUDA(cudaStreamSynchronize(st));
          c.launches += 1;
        } else {
          // 16 row segments spread over the (class-sorted) rows so that every region of the data contributes
          const int nseg = 16;
          const int64_t seg = std::max<int64_t>(1, std::min<int64_t>(N, c.sample_rows) / nseg);
          DevBuf s32, cnt;
          s32.alloc(sizeof(float) * lds);
          cnt.alloc(sizeof(double));
          KS_CUDA(cudaMemsetAsync(s32.p, 0, s32.bytes, st));
          int64_t total = 0;
          for (int sgi = 0; sgi < nseg && N > 0; ++sgi) {
            const int64_t r0 = std::min<int64_t>(N - 1, (N * sgi) / nseg);
            const int64_t nr = std::min<int64_t>(seg, N - r0);
            produce_slab(c, *sp, c0, b, sp->zeros.as<float>(), slab.as<float>() + r0 * lds, lds, r0, nr, false, s32.as<float>(), st);
            total += nr;
          }
          launch_f32_to_f64_rows(s32.as<float>(), lds, psum.as<double>(), lds, 1, b, st);
          const double nd = static_cast<double>(total);
          KS_CUDA(cudaMemcpyAsync(cnt.p, &nd, sizeof(double), cudaMemcpyHostToDevice, st));
          c.allreduce_f64(psum.as<double>(), static_cast<size_t>(b));
          c.allreduce_f64(cnt.as<double>(), 1);
          launch_divide_by_count(psum.as<double>(), cnt.as<double>(), shifts[j]->as<float>(), nullptr, b, st);
          KS_CUDA(cudaStreamSynchronize(st));
          c.launches += 2;
        }
        auto W = std::make_unique<DevBuf>();
        W->alloc(sizeof(double) * static_cast<size_t>(b) * k);
        KS_CUDA(cudaMemsetAsync(W->p, 0, W->bytes, st));
        model->brows.push_back(b);
        model->W.push_back(std::move(W));
        jms[j] = std::make_unique<DevBuf>();
        jms[j]->alloc(sizeof(double) * static_cast<size_t>(k) * b);
        KS_CUDA(cudaMemsetAsync(jms[j]->p, 0, jms[j]->bytes, st));
      }
      const float* m = shifts[j]->as<float>();
      if (x2 && sp->F) {
        launch_center_round(sp->F->d, sp->F->ld, static_cast<int>(c0), m, slab.as<float>(), nullptr, lds, N, b, st, slab_lo.as<float>());
        c.launches += 1;
      } else if (x2) {
        produce_slab(c, *sp, c0, b, m, sf32.p, lds, 0, N, /*round_out=*/false, nullptr, st, false, true);
        launch_center_round(sf32.as<float>(), lds, 0, sp->zeros.as<float>(), slab.as<float>(), nullptr, lds, N, b, st, slab_lo.as<float>());
        c.launches += 1;
      } else {
        produce_slab(c, *sp, c0, b, m, slab.as<float>(), lds, 0, N, true, nullptr, st);
      }

      // ---------------- residual: rounded operand copy, column sums over all rows and per class (means, :171, :263)
      KS_CUDA(cudaMemsetAsync(rsum_all.p, 0, rsum_all.bytes, st));
      launch_round_colsum(R.as<float>(), Rr.as<float>(), kpad, N, k, rsum_all.as<double>(), st, x2 ? Rlo.as<float>() : nullptr);
      KS_CUDA(cudaMemsetAsync(rsum_cls.p, 0, rsum_cls.bytes, st));
      KS_CUDA(cudaMemsetAsync(csum.p, 0, csum.bytes, st));
      KS_CUDA(cudaMemsetAsync(psum.p, 0, psum.bytes, st));
      for (int ci = 0; ci < ncls; ++ci) {
        const Range& rg = ranges[ci];
        launch_colsum(R.as<float>() + rg.off * kpad, nullptr, kpad, rg.n, k, rsum_cls.as<double>() + static_cast<size_t>(ci) * kpad, st);
        launch_colsum(slab.as<float>() + rg.off * lds, x2 ? slab_lo.as<float>() + rg.off * lds : nullptr, lds, rg.n, b,
                      csum.as<double>() + static_cast<size_t>(ci) * lds, st);
      }
      launch_colsum(slab.as<float>(), x2 ? slab_lo.as<float>() : nullptr, lds, N, b, psum.as<double>(), st);
      c.launches += 2 + 2 * ncls;
      c.allreduce_f64(psum.as<double>(), static_cast<size_t>(b));
      c.allreduce_f64(rsum_all.as<double>(), static_cast<size_t>(k));
      if (x2) {  // exact Gram diagonals (fp64) of every class range; the population's is their sum over all ranks
        KS_CUDA(cudaMemsetAsync(diag_cls.p, 0, diag_cls.bytes, st));
        for (int ci = 0; ci < ncls; ++ci) {
          const Range& rg = ranges[ci];
          launch_colsumsq_pair(slab.as<float>() + rg.off * lds, slab_lo.as<float>() + rg.off * lds, false, lds, rg.n, b,
                               diag_cls.as<double>() + static_cast<size_t>(ci) * lds, st);
        }
        sum_parts_f64_kernel<<<(b + 255) / 256, 256, 0, st>>>(diag_cls.as<double>(), ncls, lds, diag_pop.as<double>(), b);
        c.launches += ncls + 1;
        c.allreduce_f64(diag_pop.as<double>(), static_cast<size_t>(b));
      }

      // ---------------- class Grams (one tensor-core pass per class row range); population = sum of classes
      KS_CUDA(cudaMemsetAsync(Gcls.p, 0, Gcls.bytes, st));
      KS_CUDA(cudaMemsetAsync(Gpop.p, 0, Gpop.bytes, st));
      KS_CUDA(cudaMemsetAsync(Cpop.p, 0, Cpop.bytes, st));
      if (x2) {
        KS_CUDA(cudaMemsetAsync(Xcls.p, 0, Xcls.bytes, st));
        KS_CUDA(cudaMemsetAsync(Xpop.p, 0, Xpop.bytes, st));
      }
      for (int ci = 0; ci < ncls; ++ci) {
        const Range& rg = ranges[ci];
        float* Gc = Gcls.as<float>() + static_cast<size_t>(ci) * g_elems;
        KS_CUDA(cudaMemsetAsync(Ctmp.p, 0, Ctmp.bytes, st));
        launch_gram_block(c, slab.as<float>() + rg.off * lds, lds, rg.n, b, Rr.as<float>() + rg.off * kpad, kpad, k, Gc, ldg,
                          Ctmp.as<float>(), ldc, true, true, st, false, x2 ? 2048 : 0);
        add_f32_kernel<<<grid1d(static_cast<int64_t>(g_elems)), 256, 0, st>>>(Gc, Gpop.as<float>(), static_cast<int64_t>(g_elems));
        if (x2) {
          float* Xc = Xcls.as<float>() + static_cast<size_t>(ci) * g_elems;
          // cross Gram S_hi^T S_lo (all tiles: the "C" slot with kcols = b), then the two remaining terms of S^T R
          launch_gram_block(c, slab.as<float>() + rg.off * lds, lds, rg.n, b, slab_lo.as<float>() + rg.off * lds, lds, b, nullptr, 0,
                            Xc, ldg, false, true, st, false, 2048);
          add_f32_kernel<<<grid1d(static_cast<int64_t>(g_elems)), 256, 0, st>>>(Xc, Xpop.as<float>(), static_cast<int64_t>(g_elems));
          gram_c(slab_lo.as<float>(), rg.off, rg.n, b, Rr.as<float>(), Ctmp.as<float>());
          gram_c(slab.as<float>(), rg.off, rg.n, b, Rlo.as<float>(), Ctmp.as<float>());
          c.launches += 1;
        }
        bwls_accum_kernel<<<grid1d(static_cast<int64_t>(c_elems)), 256, 0, st>>>(Ctmp.as<float>(), Cpop.as<float>(), ldc,
                                                                            xtr.as<float>() + static_cast<size_t>(ci) * lds,
                                                                            rg.cls, b, k);
        c.launches += 2;
      }
      c.allreduce_f32(Gpop.as<float>(), g_elems);   // population statistics over all ranks (treeReduce, :212-214)
      if (x2) c.allreduce_f32(Xpop.as<float>(), g_elems);
      c.allreduce_f32(Cpop.as<float>(), c_elems);

      // ---------------- per class: joint second moments, fp64 Cholesky solve (:241-276), spread over the solve lanes
      bwls_means_kernel<<<(b + 255) / 256, 256, 0, st>>>(psum.as<double>(), Ntot_d, dp.as<double>(), b);
      KS_CUDA(cudaMemsetAsync(dW.p, 0, dW.bytes, st));
      KS_CUDA(cudaEventRecord(ev_stats, st));
      for (int q = 0; q < nlanes; ++q) KS_CUDA(cudaStreamWaitEvent(c.lanes[q]->s, ev_stats, 0));
      for (int ci = 0; ci < ncls; ++ci) {
        const Range& rg = ranges[ci];
        const int q = ci % nlanes;
        cudaStream_t ls = c.lanes[q]->s;
        const double nc = static_cast<double>(rg.n);
        double* dc = dcs.as<double>() + static_cast<size_t>(ci) * lds;
        double* Hq = laneH[q].as<double>();
        double* rq = laneRhs[q].as<double>();
        bwls_means_kernel<<<(b + 255) / 256, 256, 0, ls>>>(csum.as<double>() + static_cast<size_t>(ci) * lds, nc, dc, b);
        bwls_build_kernel<<<grid1d(static_cast<int64_t>(b) * b), 256, 0, ls>>>(
            Gpop.as<float>(), Gcls.as<float>() + static_cast<size_t>(ci) * g_elems, ldg, dp.as<double>(), dc, Ntot_d, nc, w, lam, Hq, b,
            x2 ? Xpop.as<float>() : nullptr, x2 ? Xcls.as<float>() + static_cast<size_t>(ci) * g_elems : nullptr,
            x2 ? diag_pop.as<double>() : nullptr, x2 ? diag_cls.as<double>() + static_cast<size_t>(ci) * lds : nullptr);
        bwls_rhs_kernel<<<(b + 255) / 256, 256, 0, ls>>>(Cpop.as<float>(), ldc, xtr.as<float>() + static_cast<size_t>(ci) * lds, m,
                                                       dp.as<double>(), dc, Ntot_d, nc, rsum_all.as<double>(),
                                                       rsum_cls.as<double>() + static_cast<size_t>(ci) * kpad, w, lam,
                                                       model->W[j]->as<double>() + static_cast<size_t>(rg.cls) * b, rq,
                                                       it == 0 ? jms[j]->as<double>() + static_cast<size_t>(rg.cls) * b : nullptr, rg.cls, b);
        c.launches += 3;
        if (it == 0 && j == cap_block && rg.cls == cap_cls) {  // pageable destinations: these copies complete before they return
          if (cap_H) KS_CUDA(cudaMemcpyAsync(cap_H, Hq, sizeof(double) * static_cast<size_t>(b) * b, cudaMemcpyDeviceToHost, ls));
          if (cap_rhs) KS_CUDA(cudaMemcpyAsync(cap_rhs, rq, sizeof(double) * b, cudaMemcpyDeviceToHost, ls));
        }
        c.lane_potrf_potrs(q, Hq, b, rq, 1, ci);
        copy_col_kernel<<<(b + 255) / 256, 256, 0, ls>>>(rq, dW.as<double>() + static_cast<size_t>(rg.cls) * b, b);
        c.launches += 1;
      }
      for (int q = 0; q < nlanes; ++q) {
        KS_CUDA(cudaEventRecord(ev_lane[q], c.lanes[q]->s));
        KS_CUDA(cudaStreamWaitEvent(st, ev_lane[q], 0));
      }
      // a failed factorisation must stop EVERY rank (the next collective would hang otherwise): the flag travels with dW
      double* flag = dW.as<double>() + static_cast<size_t>(bmax) * k;
      c.infos_to_flag(std::min(ncls, 4096), flag, st);
      c.allreduce_f64(dW.as<double>(), static_cast<size_t>(b) * k);  // every rank contributes the columns of its classes
      c.allreduce_f64(flag, 1);
      double h_flag = 0;
      KS_CUDA(cudaMemcpyAsync(&h_flag, flag, sizeof(double), cudaMemcpyDeviceToHost, st));
      // ---------------- W_j += dW ; R -= F dW = S dW + 1 (m^T dW)   (:278-294)
      neg_f32_to_f64_kernel<<<(b + 255) / 256, 256, 0, st>>>(m, negm.as<double>(), b);
      launch_pack_update(dW.as<double>(), model->W[j]->as<double>(), negm.as<double>(), bop.as<float>(), x2 ? bop_lo.as<float>() : nullptr,
                         static_cast<int>(lds), cbias.as<float>(), b, k, static_cast<int>(kpad), st);
      c.launches += 2;
      launch_update(c, slab.as<float>(), lds, N, b, bop.as<float>(), lds, k, R.as<float>(), kpad, cbias.as<float>(), EPI_UPDATE, true, st);
      if (x2) {
        launch_update(c, slab_lo.as<float>(), lds, N, b, bop.as<float>(), lds, k, R.as<float>(), kpad, nullptr, EPI_UPDATE, true, st);
        launch_update(c, slab.as<float>(), lds, N, b, bop_lo.as<float>(), lds, k, R.as<float>(), kpad, nullptr, EPI_UPDATE, true, st);
      }
      KS_CUDA(cudaStreamSynchronize(st));
      if (h_flag != 0)
        throw KsError{KS_ERR_NOT_SPD, "BlockWeightedLeastSquares: a per-class Cholesky failed in block " + std::to_string(j) +
                                          " (the regularised joint covariance is not positive definite; lambda too small?)"};
    }
  }
  // ---------------- finalB = jointLabelMean - sum_rows(jointMeansCombined^T .* finalFullModel)   (:314-319)
  for (int j = 0; j < nb; ++j) {
    bwls_final_b_kernel<<<k, 256, 0, st>>>(jms[j]->as<double>(), model->W[j]->as<double>(), facc.as<double>(),
                                           static_cast<int>(model->brows[j]), k);
    c.launches += 1;
  }
  c.allreduce_f64(facc.as<double>(), static_cast<size_t>(k));  // joint means exist only on the rank that owns the class
  final_b_finish_kernel<<<(k + 255) / 256, 256, 0, st>>>(jlm_d.as<double>(), facc.as<double>(), model->intercept.as<double>(), k);
  c.launches += 1;
  KS_CUDA(cudaEventRecord(ev1, st));
  c.check_async("BlockWeightedLeastSquaresEstimator.fit");
  float total_ms = 0;
  cudaEventElapsedTime(&total_ms, ev0, ev1);
  c.event_pool.push_back(ev0);
  c.event_pool.push_back(ev1);
  for (cudaEvent_t e : c.fit_events) c.event_pool.push_back(e);
  c.fit_events.clear();
  c.stats_json = "{\"solver\":\"blockwls\",\"world\":" + std::to_string(c.world) + ",\"n_local\":" + std::to_string(N) +
                 ",\"n_total\":" + std::to_string(static_cast<int64_t>(Ntot_d)) + ",\"d\":" + std::to_string(D) + ",\"k\":" +
                 std::to_string(k) + ",\"classes_present\":" + std::to_string(ncls) + ",\"block_size\":" + std::to_string(bs) +
                 ",\"num_iter\":" + std::to_string(num_iter) + ",\"reshuffled\":" + (sorted_already ? "0" : "1") +
                 ",\"mma\":\"" + (x2 ? "tf32x2" : "tf32x1") + "\",\"solve_lanes\":" + std::to_string(nlanes) +
                 ",\"total_ms\":" + std::to_string(total_ms) + ",\"launches\":" + std::to_string(c.launches - launches0) + "}";
  return c.add(std::move(model));
}

}  // namespace ks
