// The LCS branch of the ImageNet / VOC Fisher-vector pipelines on the device: LCSExtractor, GaussianMixtureModel.apply (posteriors),
// FisherVector(gmm), NormalizeRows and the signed square root of (Batch)SignedHellingerMapper
// (K/nodes/images/{LCSExtractor,FisherVector}.scala, K/nodes/learning/GaussianMixtureModel.scala, K/nodes/stats/). DESIGN.md section 16.
//
//   LCS        window sums and variances in fp64, rounded once to fp32.  Only the windows the keypoints use are computed (one
//              thread per distinct window centre and channel), then gathered into descriptor rows.
//   Posterior  fp64 log-likelihoods (x - mu)^2 / (2 sigma^2) on CUDA cores, row max / exp / normalise / threshold / normalise in
//              fp64 with fixed-order warp reductions.
//   FV         [X | X o X | 1]^T Q per item on the DMMA tensor core (mma.sync.m8n8k4.f64), every item of a batch in one launch,
//              then an elementwise epilogue; no float atomics anywhere, so every result repeats bit for bit.
#include "engine.h"

#include <math.h>

#include <algorithm>
#include <vector>

namespace ks {

// ------------------------------------------------------------------------------------------------------------------- LCS
// stats[((i C + c) ncy + iy) ncx + ix] = (mean, std) of the s x s window around (cx[ix], cy[iy]) of channel c of image i, zeros
// outside the image: rows [cx - lo, cx + hi], columns [cy - lo, cy + hi] (ImageUtils.conv2D with a length-s box filter).
__global__ void lcs_window_kernel(const float* __restrict__ img, int64_t ldi, int64_t n_img, int x_dim, int y_dim, int ch,
                                  const int* __restrict__ cx, int ncx, const int* __restrict__ cy, int ncy, int s, int lo,
                                  float2* __restrict__ stats) {
  const int64_t total = n_img * ch * ncy * ncx;
  const double inv = 1.0 / (static_cast<double>(s) * s);
  for (int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; t < total; t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int ix = static_cast<int>(t % ncx);
    int64_t r = t / ncx;
    const int iy = static_cast<int>(r % ncy);
    r /= ncy;
    const int c = static_cast<int>(r % ch);
    const int64_t i = r / ch;
    const int x0 = max(cx[ix] - lo, 0), x1 = min(cx[ix] - lo + s, x_dim);
    const int y0 = max(cy[iy] - lo, 0), y1 = min(cy[iy] - lo + s, y_dim);
    const float* im = img + i * ldi + c;
    double sum = 0.0, sq = 0.0;
    for (int y = y0; y < y1; ++y)
      for (int x = x0; x < x1; ++x) {
        const double v = static_cast<double>(im[(static_cast<int64_t>(y) * x_dim + x) * ch]);
        sum += v;
        sq += v * v;
      }
    const double mean = sum * inv;
    stats[t] = make_float2(static_cast<float>(mean), static_cast<float>(sqrt(fmax(sq * inv - mean * mean, 0.0))));
  }
}

// out row i nkp + xk nky + yk, column ((c nn + a) nn + b) 2 + {0: mean, 1: std}; wx[xk nn + a] / wy[yk nn + b]: window index
__global__ void lcs_gather_kernel(const float2* __restrict__ stats, int64_t n_img, int ch, int ncx, int ncy, const int* __restrict__ wx,
                                  const int* __restrict__ wy, int nkx, int nky, int nn, float* __restrict__ out, int64_t ldo) {
  const int cols = ch * nn * nn * 2;
  const int64_t total = n_img * nkx * nky * static_cast<int64_t>(cols);
  for (int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; t < total; t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int col = static_cast<int>(t % cols);
    const int64_t row = t / cols;
    const int kp = static_cast<int>(row % (static_cast<int64_t>(nkx) * nky));
    const int64_t i = row / (static_cast<int64_t>(nkx) * nky);
    const int xk = kp / nky, yk = kp % nky;
    const int m = col & 1, b = (col >> 1) % nn, a = (col >> 1) / nn % nn, c = (col >> 1) / (nn * nn);
    const float2 v = stats[((i * ch + c) * ncy + wy[yk * nn + b]) * ncx + wx[xk * nn + a]];
    out[row * ldo + col] = m ? v.y : v.x;
  }
}

// -------------------------------------------------------------------------------------------------------- GMM posteriors
static constexpr int kGR = 32;        // rows per CTA (one per lane)
static constexpr int kGThreads = 256; // 8 warps: warp w owns components k0 + w + 8 j, j < 4, of each 32-component chunk
static constexpr int kGSLd = kGR + 1;
static constexpr int kEpiPosterior = 0, kEpiPosteriorLse = 1, kEpiAssign = 2;

// Q[row][k] (fp64, ldq) and / or out (fp32, ldo) = thresholded, renormalised posteriors of rows [32 blockIdx.x, +32) of X (N x D).
// mu / hiv: [d][k] = mean, 0.5 / variance; ck[k] = log w_k - 1/2 sum_d log var_dk - D/2 log 2 pi.
// The epilogue is a compile-time choice (one kernel, so the three share the load phase and the log-likelihood loop exactly):
//   kEpiPosterior     the posteriors (GaussianMixtureModel.apply, FisherVector);
//   kEpiPosteriorLse  the same, and first row_out[row] = the reference's incremental ("Xerox") log-sum-exp of the row's raw
//                     log-likelihoods, one lane per row over k in order (GaussianMixtureModelEstimator.scala:127-148);
//   kEpiAssign        hard assignment: Q row (and out) = one-hot at the first argmax of the log-likelihood, row_out[row] = -max.  With
//                     hiv = 1/2 and ck = 0 that is the first argmin of 1/2 |x - c|^2 and the distance itself (KMeansModel.apply).
template <int kEpi>
__global__ void __launch_bounds__(kGThreads) gmm_posterior_kernel(const float* __restrict__ X, int64_t ldx, int64_t rows, int D, int K,
                                                                  const double* __restrict__ mu, const double* __restrict__ hiv,
                                                                  const double* __restrict__ ck, double thr, double* __restrict__ Q,
                                                                  int64_t ldq, float* __restrict__ out, int64_t ldo,
                                                                  double* __restrict__ row_out) {
  extern __shared__ float sx[];  // [D][kGSLd]: this CTA's rows, transposed
  __shared__ double smu[32][32], shv[32][32];
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * kGR;
  const int nr = static_cast<int>(min(static_cast<int64_t>(kGR), rows - r0));
  for (int e = threadIdx.x; e < kGR * D; e += kGThreads) {
    const int r = e / D, d = e - r * D;
    sx[d * kGSLd + r] = r < nr ? X[(r0 + r) * ldx + d] : 0.f;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k0 = 0; k0 < K; k0 += 32) {
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    for (int d0 = 0; d0 < D; d0 += 32) {
      __syncthreads();
      for (int e = threadIdx.x; e < 32 * 32; e += kGThreads) {
        const int dd = e >> 5, kk = e & 31;
        const bool in = d0 + dd < D && k0 + kk < K;
        smu[dd][kk] = in ? mu[static_cast<int64_t>(d0 + dd) * K + k0 + kk] : 0.0;
        shv[dd][kk] = in ? hiv[static_cast<int64_t>(d0 + dd) * K + k0 + kk] : 0.0;
      }
      __syncthreads();
      const int dn = min(32, D - d0);
      for (int dd = 0; dd < dn; ++dd) {
        const double x = static_cast<double>(sx[(d0 + dd) * kGSLd + lane]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const double t = x - smu[dd][warp + 8 * j];
          acc[j] = fma(t * t, shv[dd][warp + 8 * j], acc[j]);
        }
      }
    }
    if (lane < nr)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int k = k0 + warp + 8 * j;
        if (k < K) Q[(r0 + lane) * ldq + k] = ck[k] - acc[j];
      }
  }
  __syncthreads();  // the log-likelihoods of the CTA's rows are in Q
  if constexpr (kEpi == kEpiAssign) {
    for (int r = warp; r < nr; r += kGThreads / 32) {
      double* q = Q + (r0 + r) * ldq;
      double m = -INFINITY;
      int best = K;
      for (int k = lane; k < K; k += 32)
        if (q[k] > m) {  // strict: the first of equal values within the lane
          m = q[k];
          best = k;
        }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double om = __shfl_xor_sync(0xffffffffu, m, o);
        const int ob = __shfl_xor_sync(0xffffffffu, best, o);
        if (om > m || (om == m && ob < best)) {
          m = om;
          best = ob;
        }
      }
      for (int k = lane; k < K; k += 32) {
        q[k] = k == best ? 1.0 : 0.0;
        if (out) out[(r0 + r) * ldo + k] = k == best ? 1.f : 0.f;
      }
      if (lane == 0) row_out[r0 + r] = -m;
    }
    return;
  }
  if constexpr (kEpi == kEpiPosteriorLse) {
    if (threadIdx.x < nr) {
      const double* q = Q + (r0 + threadIdx.x) * ldq;
      double lse = q[0];
      for (int k = 1; k < K; ++k) {
        const double l = q[k], delta = lse - l;
        double inc = 0.0;  // delta <= -30 adds no weight
        if (delta > 30.0) inc = delta;
        else if (delta > -30.0) inc = log(exp(delta) + 1.0);
        lse = inc + l;
      }
      row_out[r0 + threadIdx.x] = lse;
    }
    __syncthreads();  // the raw log-likelihoods are read before the exp pass overwrites them
  }
  for (int r = warp; r < nr; r += kGThreads / 32) {
    double* q = Q + (r0 + r) * ldq;
    double m = -INFINITY;
    for (int k = lane; k < K; k += 32) m = fmax(m, q[k]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    double s = 0.0;
    for (int k = lane; k < K; k += 32) {
      const double e = exp(q[k] - m);
      q[k] = e;
      s += e;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    double t = 0.0;
    for (int k = lane; k < K; k += 32) {
      const double p = q[k] / s;
      const double kept = p > thr ? p : 0.0;
      q[k] = kept;
      t += kept;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    for (int k = lane; k < K; k += 32) {
      const double p = q[k] / t;
      q[k] = p;
      if (out) out[(r0 + r) * ldo + k] = static_cast<float>(p);
    }
  }
}

// ------------------------------------------------------------------------------------------------- Fisher-vector statistics
static constexpr int kFT = 64;          // output tile (rows of [X | X o X | 1]^T x components)
static constexpr int kFK = 32;          // descriptors per shared-memory stage
static constexpr int kFLd = kFT + 4;    // == 4 (mod 16) doubles: conflict-free fragment loads
static constexpr int kFThreads = 128;   // 4 warps, 32 x 32 outputs each
static constexpr int kFLoads = kFK * kFT / kFThreads;

__device__ __forceinline__ void fv_dmma(double (&d)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(d[0]), "+d"(d[1])
               : "d"(a), "d"(b));
}

// S[item][c][k] = sum over the item's descriptors n of a_c(x_n) q_nk with a_c = x_c (c < D), x_{c-D}^2 (c < 2D), 1 (c = 2D).
// blockIdx.y: item of the batch (descriptor rows [offs[y], offs[y + 1])); blockIdx.x: 64 x 64 tile.  Q row 0 is descriptor q_row0.
__global__ void __launch_bounds__(kFThreads) fv_stats_kernel(const float* __restrict__ X, int64_t ldx, const double* __restrict__ Q,
                                                             int64_t ldq, int64_t q_row0, const int64_t* __restrict__ offs, int D, int K,
                                                             double* __restrict__ S) {
  __shared__ double sA[kFK * kFLd], sB[kFK * kFLd];
  const int m = 2 * D + 1, ntn = (K + kFT - 1) / kFT;
  const int bi = blockIdx.x / ntn, bj = blockIdx.x % ntn;
  const int64_t r0 = offs[blockIdx.y], r1 = offs[blockIdx.y + 1];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wm = warp >> 1, wn = warp & 1;
  const int col = threadIdx.x & (kFT - 1), ca = bi * kFT + col, kb = bj * kFT + col;
  const int xd = ca < D ? ca : ca - D;
  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
  double pa[kFLoads], pb[kFLoads];
  auto load = [&](int64_t r) {
#pragma unroll
    for (int u = 0; u < kFLoads; ++u) {
      const int64_t row = r + (threadIdx.x >> 6) + 2 * u;
      double a = 0.0, b = 0.0;
      if (row < r1) {
        if (ca < 2 * D) {
          const double x = static_cast<double>(X[row * ldx + xd]);
          a = ca < D ? x : x * x;
        } else if (ca == 2 * D) {
          a = 1.0;
        }
        if (kb < K) b = Q[(row - q_row0) * ldq + kb];
      }
      pa[u] = a;
      pb[u] = b;
    }
  };
  load(r0);
  for (int64_t r = r0; r < r1; r += kFK) {
#pragma unroll
    for (int u = 0; u < kFLoads; ++u) {
      sA[((threadIdx.x >> 6) + 2 * u) * kFLd + col] = pa[u];
      sB[((threadIdx.x >> 6) + 2 * u) * kFLd + col] = pb[u];
    }
    __syncthreads();
    if (r + kFK < r1) load(r + kFK);  // the next stage's loads are in flight during this stage's MMAs
    const int kk = lane & 3, q = lane >> 2;
#pragma unroll
    for (int k = 0; k < kFK; k += 4) {
      double a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = sA[(k + kk) * kFLd + wm * 32 + i * 8 + q];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = sB[(k + kk) * kFLd + wn * 32 + j * 8 + q];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) fv_dmma(acc[i][j], a[i], b[j]);
    }
    __syncthreads();
  }
  double* Si = S + static_cast<int64_t>(blockIdx.y) * m * K;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int gi = bi * kFT + wm * 32 + i * 8 + (lane >> 2), gj = bj * kFT + wn * 32 + j * 8 + (lane & 3) * 2 + e;
        if (gi < m && gj < K) Si[static_cast<int64_t>(gi) * K + gj] = acc[i][j][e];
      }
}

// out[item][d + D j] (MatrixVectorizer order of the D x 2K matrix [fv1 | fv2]) with s0 = S[2D][k] / n, s1 = S[d][k] / n,
// s2 = S[D + d][k] / n:  fv1 = (s1 - mu s0) / (sigma sqrt(w)),  fv2 = (s2 - 2 mu s1 + (mu^2 - var) s0) / (var sqrt(2 w)).
__global__ void fv_finalize_kernel(const double* __restrict__ S, const int64_t* __restrict__ offs, int64_t n_items, int D, int K,
                                   const double* __restrict__ mu, const double* __restrict__ var, const double* __restrict__ w,
                                   float* __restrict__ out, int64_t ldo) {
  const int64_t per = 2LL * D * K, total = n_items * per;
  for (int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; t < total; t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t i = t / per;
    const int e = static_cast<int>(t - i * per), d = e % D, j = e / D, k = j % K;
    const double inv_n = 1.0 / static_cast<double>(offs[i + 1] - offs[i]);
    const double* Si = S + i * (2LL * D + 1) * K;
    const double s0 = Si[2LL * D * K + k] * inv_n, s1 = Si[static_cast<int64_t>(d) * K + k] * inv_n;
    const double m = mu[static_cast<int64_t>(d) * K + k], v = var[static_cast<int64_t>(d) * K + k];
    double r;
    if (j < K) {
      r = (s1 - m * s0) / (sqrt(v) * sqrt(w[k]));
    } else {
      const double s2 = Si[static_cast<int64_t>(D + d) * K + k] * inv_n;
      r = (s2 - 2.0 * m * s1 + (m * m - v) * s0) / (v * sqrt(2.0 * w[k]));
    }
    out[i * ldo + e] = static_cast<float>(r);
  }
}

// ----------------------------------------------------------------------------------------- NormalizeRows, signed square root
// one CTA per row: norm in fp64 (fixed-order tree), out = x / max(norm, 2.2e-16) rounded once; padding columns stay zero
__global__ void __launch_bounds__(256) normalize_rows_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t ld, int cols) {
  __shared__ double red[256];
  const float* x = in + blockIdx.x * ld;
  double s = 0.0;
  for (int c = threadIdx.x; c < cols; c += 256) {
    const double v = static_cast<double>(x[c]);
    s = fma(v, v, s);
  }
  red[threadIdx.x] = s;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  const double den = fmax(sqrt(red[0]), 2.2e-16);
  float* y = out + blockIdx.x * ld;
  for (int64_t c = threadIdx.x; c < ld; c += 256) y[c] = c < cols ? static_cast<float>(static_cast<double>(x[c]) / den) : 0.f;
}

// sign(v) sqrt(|v|) (BatchSignedHellingerMapper: math.sqrt in fp64, then toFloat)
__global__ void signed_sqrt_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float v = in[i];
    const float r = static_cast<float>(sqrt(fabs(static_cast<double>(v))));
    out[i] = v > 0.f ? r : v < 0.f ? -r : 0.f;
  }
}

// ------------------------------------------------------------------------------------------------------------- launchers
static unsigned grid_of(int64_t work, int threads, const Ctx& c) {
  return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((work + threads - 1) / threads, 32LL * c.num_sms)));
}

// ImageUtils.conv2D pads floor((s - 1) / 2) before and ceil((s - 1) / 2) after, so window (x) covers [x - lo, x - lo + s)
std::unique_ptr<Matrix> lcs_extract(Ctx& c, Matrix& im, int x_dim, int y_dim, int ch, int stride, int start, int s) {
  if (x_dim <= 0 || y_dim <= 0 || ch <= 0 || stride <= 0 || start < 0 || s <= 0)
    throw KsError{KS_ERR_INVALID, "LCSExtractor: dimensions, stride and subPatchSize must be positive, strideStart >= 0"};
  if (im.cols != static_cast<int64_t>(x_dim) * y_dim * ch) throw KsError{KS_ERR_INVALID, "LCSExtractor: image size does not match the matrix"};
  // keypoints strideStart until dim - strideStart by stride; neighbour offsets -2s + s/2 - 1 to s + s/2 - 1 by s (LCSExtractor.scala:56-71)
  auto grid = [&](int dim) {
    std::vector<int> v;
    for (int p = start; p < dim - start; p += stride) v.push_back(p);
    return v;
  };
  const std::vector<int> kx = grid(x_dim), ky = grid(y_dim);
  std::vector<int> nb;
  for (int o = -2 * s + s / 2 - 1; o <= s + s / 2 - 1; o += s) nb.push_back(o);
  if (kx.empty() || ky.empty()) throw KsError{KS_ERR_INVALID, "LCSExtractor: no keypoint fits the image (strideStart too large)"};
  if (kx.front() + nb.front() < 0 || ky.front() + nb.front() < 0 || kx.back() + nb.back() >= x_dim || ky.back() + nb.back() >= y_dim)
    throw KsError{KS_ERR_INVALID, "LCSExtractor: keypoint neighbourhoods leave the image (raise strideStart or lower subPatchSize)"};
  const int nn = static_cast<int>(nb.size());
  // distinct window centres per axis and the window index of every (keypoint, neighbour)
  auto centres = [&](const std::vector<int>& kp, std::vector<int>& ctr, std::vector<int>& widx) {
    for (int p : kp)
      for (int o : nb) ctr.push_back(p + o);
    std::sort(ctr.begin(), ctr.end());
    ctr.erase(std::unique(ctr.begin(), ctr.end()), ctr.end());
    for (int p : kp)
      for (int o : nb) widx.push_back(static_cast<int>(std::lower_bound(ctr.begin(), ctr.end(), p + o) - ctr.begin()));
  };
  std::vector<int> cx, cy, wx, wy;
  centres(kx, cx, wx);
  centres(ky, cy, wy);
  const int nkx = static_cast<int>(kx.size()), nky = static_cast<int>(ky.size()), ncx = static_cast<int>(cx.size()),
            ncy = static_cast<int>(cy.size());
  const int64_t nkp = static_cast<int64_t>(nkx) * nky, cols = static_cast<int64_t>(ch) * nn * nn * 2;
  auto out = new_matrix(im.rows * nkp, cols);
  if (out->ld != cols) KS_CUDA(cudaMemsetAsync(out->d, 0, out->buf.bytes, c.st));
  std::vector<int> tab;
  for (auto* v : {&cx, &cy, &wx, &wy}) tab.insert(tab.end(), v->begin(), v->end());
  DevBuf dtab, stats;
  dtab.alloc(sizeof(int) * tab.size());
  KS_CUDA(cudaMemcpyAsync(dtab.p, tab.data(), sizeof(int) * tab.size(), cudaMemcpyHostToDevice, c.st));
  const int* dcx = dtab.as<int>();
  const int *dcy = dcx + ncx, *dwx = dcy + ncy, *dwy = dwx + wx.size();
  // image chunks bound the window statistics to 16 MB
  const int64_t per_img = static_cast<int64_t>(ch) * ncx * ncy;
  const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(im.rows, (int64_t(16) << 20) / (8 * per_img)));
  stats.alloc(sizeof(float2) * static_cast<size_t>(chunk * per_img));
  for (int64_t i0 = 0; i0 < im.rows; i0 += chunk) {
    const int64_t ni = std::min(chunk, im.rows - i0);
    lcs_window_kernel<<<grid_of(ni * per_img, 256, c), 256, 0, c.st>>>(im.d + i0 * im.ld, im.ld, ni, x_dim, y_dim, ch, dcx, ncx, dcy, ncy, s,
                                                                       (s - 1) / 2, stats.as<float2>());
    lcs_gather_kernel<<<grid_of(ni * nkp * cols, 256, c), 256, 0, c.st>>>(stats.as<float2>(), ni, ch, ncx, ncy, dwx, dwy, nkx, nky, nn,
                                                                          out->d + i0 * nkp * out->ld, out->ld);
    c.launches += 2;
  }
  c.check_async("LCSExtractor.apply");
  return out;
}

int64_t gmm_create(Ctx& c, const double* means, const double* vars, const double* w, int64_t dim, int64_t k, double thr) {
  if (!means || !vars || !w || dim <= 0 || k <= 0) throw KsError{KS_ERR_INVALID, "GaussianMixtureModel: null arrays or empty shape"};
  if (dim > 1024) throw KsError{KS_ERR_INVALID, "GaussianMixtureModel: dim must be <= 1024"};
  if (!(thr >= 0.0 && thr < 1.0 / static_cast<double>(k)))
    throw KsError{KS_ERR_INVALID, "GaussianMixtureModel: weightThreshold must lie in [0, 1/k) (at or above 1/k a row can be zeroed)"};
  const int64_t n = dim * k;
  auto g = std::make_unique<Gmm>();
  g->dim = dim;
  g->k = k;
  g->thr = thr;
  std::vector<double> h(4 * n + 2 * k);  // [mu | var | hiv][d][k] (row-major d x k), ck, w
  double* hmu = h.data();
  double* hvar = hmu + n;
  double* hhiv = hvar + n;
  double* hck = hhiv + n;
  double* hw = hck + k;
  for (int64_t kk = 0; kk < k; ++kk) {
    if (!std::isfinite(w[kk]) || !(w[kk] > 0.0)) throw KsError{KS_ERR_INVALID, "GaussianMixtureModel: weights must be finite and > 0"};
    double slog = 0.0;
    for (int64_t d = 0; d < dim; ++d) {
      const double m = means[d + dim * kk], v = vars[d + dim * kk];  // column-major D x K
      if (!std::isfinite(m)) throw KsError{KS_ERR_INVALID, "GaussianMixtureModel: means must be finite"};
      if (!std::isfinite(v) || !(v > 0.0)) throw KsError{KS_ERR_INVALID, "GaussianMixtureModel: variances must be finite and > 0"};
      hmu[d * k + kk] = m;
      hvar[d * k + kk] = v;
      hhiv[d * k + kk] = 0.5 / v;
      slog += log(v);
    }
    hck[kk] = -0.5 * static_cast<double>(dim) * log(2.0 * M_PI) - 0.5 * slog + log(w[kk]);
    hw[kk] = w[kk];
  }
  g->buf.alloc(sizeof(double) * h.size());
  KS_CUDA(cudaMemcpyAsync(g->buf.p, h.data(), sizeof(double) * h.size(), cudaMemcpyHostToDevice, c.st));
  c.check_async("GaussianMixtureModel");
  const int64_t id = c.next_id++;
  c.gmms[id] = std::move(g);
  return id;
}

template <int kEpi>
static void launch_posterior_epi(Ctx& c, const Gmm& g, const Matrix& X, int64_t row0, int64_t rows, double* Q, int64_t ldq, float* out,
                                 int64_t ldo, double* row_out) {
  if (rows == 0) return;
  const int64_t blocks = (rows + kGR - 1) / kGR;
  if (blocks > 0x7fffffffLL) throw KsError{KS_ERR_INVALID, "GaussianMixtureModel: too many rows"};
  const size_t smem = sizeof(float) * static_cast<size_t>(g.dim) * kGSLd;
  KS_CUDA(cudaFuncSetAttribute(gmm_posterior_kernel<kEpi>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  gmm_posterior_kernel<kEpi><<<static_cast<unsigned>(blocks), kGThreads, smem, c.st>>>(
      X.d + row0 * X.ld, X.ld, rows, static_cast<int>(g.dim), static_cast<int>(g.k), g.mu(), g.hiv(), g.ck(), g.thr, Q, ldq, out, ldo,
      row_out ? row_out + row0 : nullptr);
  c.launches += 1;
}

// posteriors of rows [row0, row0 + rows) of X into Q (fp64, ldq) and / or out (fp32)
static void launch_posteriors(Ctx& c, const Gmm& g, const Matrix& X, int64_t row0, int64_t rows, double* Q, int64_t ldq, float* out,
                              int64_t ldo) {
  launch_posterior_epi<kEpiPosterior>(c, g, X, row0, rows, Q, ldq, out, ldo, nullptr);
}

void launch_gmm_estep(Ctx& c, const Gmm& g, const Matrix& X, int64_t row0, int64_t rows, double* Q, float* out, int64_t ldo, int epi,
                      double* row_out) {
  if (epi == kEpiPosteriorLse) launch_posterior_epi<kEpiPosteriorLse>(c, g, X, row0, rows, Q, g.k, out, ldo, row_out);
  else if (epi == kEpiAssign) launch_posterior_epi<kEpiAssign>(c, g, X, row0, rows, Q, g.k, out, ldo, row_out);
  else throw KsError{KS_ERR_INVALID, "launch_gmm_estep: unknown epilogue"};
}

void launch_fv_stats(Ctx& c, const Matrix& X, const double* Q, int64_t ldq, int64_t q_row0, const int64_t* d_offs, int64_t n_items, int D,
                     int K, double* S) {
  const int m = 2 * D + 1;
  const unsigned tiles = static_cast<unsigned>(((m + kFT - 1) / kFT) * ((K + kFT - 1) / kFT));
  fv_stats_kernel<<<dim3(tiles, static_cast<unsigned>(n_items)), kFThreads, 0, c.st>>>(X.d, X.ld, Q, ldq, q_row0, d_offs, D, K, S);
  c.launches += 1;
}

int64_t fv_stats_tiles(int D, int K) { return static_cast<int64_t>((2 * D + 1 + kFT - 1) / kFT) * ((K + kFT - 1) / kFT); }

// the fp64 posterior scratch of one launch is bounded to 256 MB of rows
int64_t posterior_chunk_rows(const Gmm& g) { return std::max<int64_t>(kGR, ((int64_t(256) << 20) / (8 * g.k)) / kGR * kGR); }

std::unique_ptr<Matrix> gmm_posteriors(Ctx& c, const Gmm& g, Matrix& X) {
  if (X.cols != g.dim) throw KsError{KS_ERR_INVALID, "GaussianMixtureModel.apply: input columns != model dimension"};
  auto out = new_matrix(X.rows, g.k);
  if (out->ld != g.k) KS_CUDA(cudaMemsetAsync(out->d, 0, out->buf.bytes, c.st));
  const int64_t chunk = std::min(std::max<int64_t>(X.rows, 1), posterior_chunk_rows(g));
  DevBuf Q;
  Q.alloc(sizeof(double) * static_cast<size_t>(chunk * g.k));
  for (int64_t r0 = 0; r0 < X.rows; r0 += chunk) {
    const int64_t nr = std::min(chunk, X.rows - r0);
    launch_posteriors(c, g, X, r0, nr, Q.as<double>(), g.k, out->d + r0 * out->ld, out->ld);
  }
  c.check_async("GaussianMixtureModel.apply");
  return out;
}

std::unique_ptr<Matrix> fisher_vector_apply(Ctx& c, const Gmm& g, Matrix& X, const int64_t* offs, int64_t n_items) {
  if (n_items <= 0 || !offs) throw KsError{KS_ERR_INVALID, "FisherVector: no items"};
  if (X.cols != g.dim) throw KsError{KS_ERR_INVALID, "FisherVector: descriptor columns != GMM dimension"};
  if (offs[0] != 0 || offs[n_items] != X.rows) throw KsError{KS_ERR_INVALID, "FisherVector: offsets must start at 0 and end at the row count"};
  for (int64_t i = 0; i < n_items; ++i)
    if (offs[i + 1] <= offs[i]) throw KsError{KS_ERR_INVALID, "FisherVector: offsets must increase strictly (an empty item has no Fisher vector)"};
  const int D = static_cast<int>(g.dim), K = static_cast<int>(g.k), m = 2 * D + 1;
  const int64_t per = 2LL * D * K;
  auto out = new_matrix(n_items, per);
  if (out->ld != per) KS_CUDA(cudaMemsetAsync(out->d, 0, out->buf.bytes, c.st));
  // item batches: the posterior scratch (rows x K) and the statistics (items x (2D + 1) x K) stay within 256 MB each (an item larger
  // than that is a batch of its own)
  const int64_t budget = (int64_t(256) << 20) / 8;
  std::vector<std::pair<int64_t, int64_t>> batches;
  int64_t max_rows = 0, max_items = 0;
  for (int64_t i0 = 0; i0 < n_items;) {
    int64_t i1 = i0 + 1;
    while (i1 < n_items && i1 - i0 < 65535 && (offs[i1 + 1] - offs[i0]) * K <= budget && (i1 + 1 - i0) * m * K <= budget) ++i1;
    batches.push_back({i0, i1});
    max_rows = std::max(max_rows, offs[i1] - offs[i0]);
    max_items = std::max(max_items, i1 - i0);
    i0 = i1;
  }
  DevBuf doffs, Q, S;
  doffs.alloc(sizeof(int64_t) * static_cast<size_t>(n_items + 1));
  KS_CUDA(cudaMemcpyAsync(doffs.p, offs, sizeof(int64_t) * static_cast<size_t>(n_items + 1), cudaMemcpyHostToDevice, c.st));
  Q.alloc(sizeof(double) * static_cast<size_t>(max_rows * K));
  S.alloc(sizeof(double) * static_cast<size_t>(max_items * m * K));
  const unsigned tiles = static_cast<unsigned>(((m + kFT - 1) / kFT) * ((K + kFT - 1) / kFT));
  for (auto [i0, i1] : batches) {
    const int64_t q0 = offs[i0], ni = i1 - i0;
    launch_posteriors(c, g, X, q0, offs[i1] - q0, Q.as<double>(), K, nullptr, 0);
    fv_stats_kernel<<<dim3(tiles, static_cast<unsigned>(ni)), kFThreads, 0, c.st>>>(X.d, X.ld, Q.as<double>(), K, q0, doffs.as<int64_t>() + i0,
                                                                                    D, K, S.as<double>());
    fv_finalize_kernel<<<grid_of(ni * per, 256, c), 256, 0, c.st>>>(S.as<double>(), doffs.as<int64_t>() + i0, ni, D, K, g.mu(), g.var(),
                                                                     g.w(), out->d + i0 * out->ld, out->ld);
    c.launches += 2;
  }
  c.check_async("FisherVector.apply");
  return out;
}

std::unique_ptr<Matrix> normalize_rows(Ctx& c, Matrix& in) {
  auto out = new_matrix(in.rows, in.cols);
  if (in.rows > 0x7fffffffLL) throw KsError{KS_ERR_INVALID, "NormalizeRows: too many rows"};
  if (in.rows > 0) {
    normalize_rows_kernel<<<static_cast<unsigned>(in.rows), 256, 0, c.st>>>(in.d, out->d, in.ld, static_cast<int>(in.cols));
    c.launches += 1;
  }
  c.check_async("NormalizeRows");
  return out;
}

void launch_signed_sqrt(Ctx& c, const float* in, float* out, int64_t n) {
  if (n == 0) return;
  signed_sqrt_kernel<<<grid_of(n, 256, c), 256, 0, c.st>>>(in, out, n);
  c.launches += 1;
}

}  // namespace ks
