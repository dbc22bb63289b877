// The CIFAR random-patch front end and test-time augmentation on the device (DESIGN.md section 21):
//   image views   Windower, Cropper, RandomPatcher, CenterCornerPatcher and RandomImageTransformer as one gather.  A view is
//                 (src_row, x0, y0, flip) with a fixed out_x x out_y size; in ImageVectorizer order (value (x, y, c) at
//                 c + x C + y C xDim) every y-line of a crop is one contiguous span of out_x C floats of the source, and
//                 ImageUtils.flipHorizontal (which reverses y) only reorders the spans.  One CTA per view copies them.
//   normalizeRows Stats.normalizeRows(mat, alpha): per row, fp64 mean and sample variance by a fixed tree, rounded once to fp32.
//   scaler        StandardScaler: fp64 column sums over fixed row chunks, then the chunks added in order (no float atomics,
//                 so a refit is bit-identical), summed over the ranks; apply (x - mean) / std in fp64, rounded once.
//   evaluator     AugmentedExamplesEvaluator: one CTA per group of views adds the average or Borda scores in view order, takes
//                 the first maximum and counts it into the confusion matrix with integer atomics.
#include "engine.h"

#include <math.h>

#include <algorithm>
#include <vector>

namespace ks {

static constexpr int kScalerChunk = 1024;  // rows per partial column sum of the scaler fit
static constexpr int kMaxEvalClasses = 4096;

static unsigned grid_for(int64_t work, int threads, const Ctx& c) {
  return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((work + threads - 1) / threads, 32LL * c.num_sms)));
}

// ------------------------------------------------------------------------------------------------------------------ views
// out row v = view v: element (x, y, c) at c + x C + y C out_x, read from source (x0 + x, y0 + (flip ? out_y - 1 - y : y), c)
__global__ void __launch_bounds__(256) image_views_kernel(const float* __restrict__ src, int64_t lds, int x_dim, int ch,
                                                          const int4* __restrict__ views, int out_x, int out_y,
                                                          float* __restrict__ out, int64_t ldo) {
  const int4 v = views[blockIdx.x];
  const int span = out_x * ch;
  const float* s = src + static_cast<int64_t>(v.x) * lds + static_cast<int64_t>(v.y) * ch;
  float* o = out + static_cast<int64_t>(blockIdx.x) * ldo;
  const int64_t n = static_cast<int64_t>(span) * out_y;
  for (int64_t t = threadIdx.x; t < ldo; t += blockDim.x) {
    if (t < n) {
      const int y = static_cast<int>(t / span), r = static_cast<int>(t - static_cast<int64_t>(y) * span);
      const int ys = v.z + (v.w ? out_y - 1 - y : y);
      o[t] = s[static_cast<int64_t>(ys) * x_dim * ch + r];
    } else {
      o[t] = 0.f;
    }
  }
}

void check_views(const int32_t* views, int64_t n_views, int64_t n_images, int x_dim, int y_dim, int out_x, int out_y) {
  if (n_views < 0 || (n_views > 0 && !views)) throw KsError{KS_ERR_INVALID, "image views: null view table or negative count"};
  if (n_views > 0x7fffffffLL) throw KsError{KS_ERR_INVALID, "image views: more than 2^31 - 1 views"};
  if (out_x < 1 || out_y < 1 || out_x > x_dim || out_y > y_dim)
    throw KsError{KS_ERR_INVALID, "image views: the view size must lie in [1, x_dim] x [1, y_dim]"};
  for (int64_t i = 0; i < n_views; ++i) {
    const int32_t* v = views + 4 * i;
    // ImageUtils.crop: 0 <= start <= end <= dim on both axes
    if (v[0] < 0 || v[0] >= n_images) throw KsError{KS_ERR_INVALID, "image views: view " + std::to_string(i) + " names no source image"};
    if (v[1] < 0 || v[1] > x_dim - out_x) throw KsError{KS_ERR_INVALID, "image views: view " + std::to_string(i) + " leaves the image in x"};
    if (v[2] < 0 || v[2] > y_dim - out_y) throw KsError{KS_ERR_INVALID, "image views: view " + std::to_string(i) + " leaves the image in y"};
    if (v[3] != 0 && v[3] != 1) throw KsError{KS_ERR_INVALID, "image views: flip must be 0 or 1"};
  }
}

static void check_image_batch(const Matrix& images, int x_dim, int y_dim, int ch) {
  if (x_dim < 1 || y_dim < 1 || ch < 1 || static_cast<int64_t>(x_dim) * y_dim * ch != images.cols)
    throw KsError{KS_ERR_INVALID, "image views: x_dim * y_dim * channels must equal the image matrix's columns"};
}

void launch_image_views(Ctx& c, const Matrix& images, int x_dim, int ch, const int32_t* d_views, int64_t n, int out_x, int out_y,
                        float* out, int64_t ldo) {
  if (n == 0) return;
  image_views_kernel<<<static_cast<unsigned>(n), 256, 0, c.st>>>(images.d, images.ld, x_dim, ch, reinterpret_cast<const int4*>(d_views),
                                                                  out_x, out_y, out, ldo);
  c.launches += 1;
}

std::unique_ptr<Matrix> image_views(Ctx& c, Matrix& images, int x_dim, int y_dim, int ch, const int32_t* views, int64_t n_views, int out_x,
                                    int out_y) {
  check_image_batch(images, x_dim, y_dim, ch);
  check_views(views, n_views, images.rows, x_dim, y_dim, out_x, out_y);
  auto out = new_matrix(n_views, static_cast<int64_t>(out_x) * out_y * ch);
  DevBuf dv;
  if (n_views > 0) {
    dv.alloc(sizeof(int32_t) * 4 * static_cast<size_t>(n_views));
    KS_CUDA(cudaMemcpyAsync(dv.p, views, sizeof(int32_t) * 4 * n_views, cudaMemcpyHostToDevice, c.st));
  }
  launch_image_views(c, images, x_dim, ch, dv.as<int32_t>(), n_views, out_x, out_y, out->d, out->ld);
  c.check_async("image views");
  return out;
}

// ------------------------------------------------------------------------------------------------------------ normalizeRows
__device__ __forceinline__ double block_sum_256(double v, double* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + h]);
    __syncthreads();
  }
  const double s = red[0];
  __syncthreads();
  return s;
}

__global__ void __launch_bounds__(256) stats_normalize_rows_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t ld,
                                                                   int cols, double alpha) {
  __shared__ double red[256];
  const float* x = in + blockIdx.x * ld;
  double s = 0.0;
  for (int c = threadIdx.x; c < cols; c += 256) s = __dadd_rn(s, static_cast<double>(x[c]));
  double mean = __ddiv_rn(block_sum_256(s, red), static_cast<double>(cols));
  if (isnan(mean)) mean = 0.0;
  double q = 0.0;
  for (int c = threadIdx.x; c < cols; c += 256) {
    const double d = __dsub_rn(static_cast<double>(x[c]), mean);
    q = __dadd_rn(q, __dmul_rn(d, d));
  }
  const double var = __ddiv_rn(block_sum_256(q, red), static_cast<double>(cols) - 1.0);
  double sd = __dsqrt_rn(__dadd_rn(var, alpha));
  if (isnan(sd)) sd = sqrt(alpha);
  float* y = out + blockIdx.x * ld;
  for (int64_t c = threadIdx.x; c < ld; c += 256)
    y[c] = c < cols ? __double2float_rn(__ddiv_rn(__dsub_rn(static_cast<double>(x[c]), mean), sd)) : 0.f;
}

std::unique_ptr<Matrix> stats_normalize_rows(Ctx& c, Matrix& in, double alpha) {
  if (!std::isfinite(alpha)) throw KsError{KS_ERR_INVALID, "normalizeRows: alpha must be finite"};
  if (in.rows > 0x7fffffffLL) throw KsError{KS_ERR_INVALID, "normalizeRows: too many rows"};
  auto out = new_matrix(in.rows, in.cols);
  if (in.rows > 0) {
    stats_normalize_rows_kernel<<<static_cast<unsigned>(in.rows), 256, 0, c.st>>>(in.d, out->d, in.ld, static_cast<int>(in.cols), alpha);
    c.launches += 1;
  }
  c.check_async("normalizeRows");
  return out;
}

// ------------------------------------------------------------------------------------------------------------ StandardScaler
// part[chunk][col] = sum over the chunk's rows r (in order per thread row, then the 8 thread rows in order) of f(x[r][col]), where
// f(v) = v (shift null) or (v - shift[col])^2.  CTA: 32 columns x 8 thread rows, one chunk of kScalerChunk rows.
__global__ void __launch_bounds__(256) scaler_partial_kernel(const float* __restrict__ x, int64_t ld, int64_t rows, int64_t cols,
                                                             const double* __restrict__ shift, double* __restrict__ part) {
  __shared__ double red[8][33];
  const int64_t col = static_cast<int64_t>(blockIdx.x) * 32 + threadIdx.x;
  const int64_t r0 = static_cast<int64_t>(blockIdx.y) * kScalerChunk;
  const int64_t r1 = min(rows, r0 + kScalerChunk);
  double s = 0.0;
  if (col < cols) {
    const double m = shift ? shift[col] : 0.0;
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
      const double v = static_cast<double>(x[r * ld + col]);
      if (shift) {
        const double d = __dsub_rn(v, m);
        s = __dadd_rn(s, __dmul_rn(d, d));
      } else {
        s = __dadd_rn(s, v);
      }
    }
  }
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && col < cols) {
    double t = red[0][threadIdx.x];
    for (int i = 1; i < 8; ++i) t = __dadd_rn(t, red[i][threadIdx.x]);
    part[static_cast<int64_t>(blockIdx.y) * cols + col] = t;
  }
}

// sum[col] = the chunks' partials added in chunk order
__global__ void scaler_chunks_kernel(const double* __restrict__ part, int64_t n_chunks, int64_t cols, double* __restrict__ sum) {
  for (int64_t col = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; col < cols; col += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    double t = 0.0;
    for (int64_t k = 0; k < n_chunks; ++k) t = __dadd_rn(t, part[k * cols + col]);
    sum[col] = t;
  }
}

// buf = [column sums (cols) | local row count]; after the all-reduce: mean = sum / N (stage 0), or std from the squared deviations
// with MLlib's unbiased variance and the guard of StandardScaler.scala:45-59 (stage 1)
__global__ void scaler_finish_kernel(double* __restrict__ buf, int64_t cols, double eps, int stage, double* __restrict__ res) {
  const double n = buf[cols];
  for (int64_t col = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; col < cols; col += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    if (stage == 0) {
      res[col] = __ddiv_rn(buf[col], n);
    } else {
      const double var = n > 1.0 ? __ddiv_rn(buf[col], __dsub_rn(n, 1.0)) : 0.0;
      const double sd = __dsqrt_rn(var);
      res[col] = (isnan(sd) || isinf(sd) || fabs(sd) < eps) ? 1.0 : sd;
    }
  }
}

static void scaler_column_sums(Ctx& c, const Matrix& X, const double* shift, DevBuf& part, double* buf) {
  const int64_t n_chunks = std::max<int64_t>(1, (X.rows + kScalerChunk - 1) / kScalerChunk);
  if (n_chunks > 65535) throw KsError{KS_ERR_INVALID, "StandardScaler: more than 65535 * 1024 rows on one rank"};
  part.alloc(sizeof(double) * static_cast<size_t>(n_chunks * std::max<int64_t>(X.cols, 1)));
  const dim3 grid(static_cast<unsigned>((X.cols + 31) / 32), static_cast<unsigned>(n_chunks));
  scaler_partial_kernel<<<grid, dim3(32, 8), 0, c.st>>>(X.d, X.ld, X.rows, X.cols, shift, part.as<double>());
  scaler_chunks_kernel<<<grid_for(X.cols, 256, c), 256, 0, c.st>>>(part.as<double>(), n_chunks, X.cols, buf);
  c.launches += 2;
}

void standard_scaler_fit(Ctx& c, Matrix& X, int normalize_std, double eps, double* mean_out, double* std_out) {
  if (!mean_out || (normalize_std && !std_out)) throw KsError{KS_ERR_INVALID, "StandardScaler: null output"};
  if (normalize_std != 0 && normalize_std != 1) throw KsError{KS_ERR_INVALID, "StandardScaler: normalize_std must be 0 or 1"};
  if (!(eps >= 0.0) || !std::isfinite(eps)) throw KsError{KS_ERR_INVALID, "StandardScaler: eps must be finite and >= 0"};
  if (X.cols < 1) throw KsError{KS_ERR_INVALID, "StandardScaler: no columns"};
  const int64_t d = X.cols;
  DevBuf part, buf, mean, sd;
  buf.alloc(sizeof(double) * static_cast<size_t>(d + 1));
  mean.alloc(sizeof(double) * static_cast<size_t>(d));
  double* b = buf.as<double>();
  scaler_column_sums(c, X, nullptr, part, b);
  launch_set_f64(b + d, static_cast<double>(X.rows), c.st);
  c.allreduce_f64(b, static_cast<size_t>(d + 1));
  double n_total = 0;
  KS_CUDA(cudaMemcpyAsync(&n_total, b + d, sizeof(double), cudaMemcpyDeviceToHost, c.st));
  KS_CUDA(cudaStreamSynchronize(c.st));
  if (n_total < 1) throw KsError{KS_ERR_INVALID, "StandardScaler: no rows on any rank"};
  scaler_finish_kernel<<<grid_for(d, 256, c), 256, 0, c.st>>>(b, d, eps, 0, mean.as<double>());
  c.launches += 2;
  if (normalize_std) {
    sd.alloc(sizeof(double) * static_cast<size_t>(d));
    scaler_column_sums(c, X, mean.as<double>(), part, b);
    launch_set_f64(b + d, n_total, c.st);   // the global count; only the deviations are summed over the ranks
    c.allreduce_f64(b, static_cast<size_t>(d));
    scaler_finish_kernel<<<grid_for(d, 256, c), 256, 0, c.st>>>(b, d, eps, 1, sd.as<double>());
    c.launches += 2;
    KS_CUDA(cudaMemcpyAsync(std_out, sd.p, sizeof(double) * d, cudaMemcpyDeviceToHost, c.st));
  }
  KS_CUDA(cudaMemcpyAsync(mean_out, mean.p, sizeof(double) * d, cudaMemcpyDeviceToHost, c.st));
  c.check_async("StandardScaler.fit");
}

__global__ void scaler_apply_kernel(const float* __restrict__ x, float* __restrict__ out, int64_t ld, int64_t rows, int64_t cols,
                                    const double* __restrict__ mean, const double* __restrict__ sd) {
  const int64_t total = rows * ld;
  for (int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; t < total; t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t col = t % ld;
    if (col < cols) {
      const double v = __dsub_rn(static_cast<double>(x[t]), mean[col]);
      out[t] = __double2float_rn(sd ? __ddiv_rn(v, sd[col]) : v);
    } else {
      out[t] = 0.f;
    }
  }
}

std::unique_ptr<Matrix> standard_scaler_apply(Ctx& c, Matrix& X, const double* mean, const double* std_or_null) {
  if (!mean) throw KsError{KS_ERR_INVALID, "StandardScalerModel: null mean"};
  const int64_t d = X.cols;
  for (int64_t j = 0; j < d; ++j)
    if (!std::isfinite(mean[j]) || (std_or_null && !(std::isfinite(std_or_null[j]) && std_or_null[j] != 0.0)))
      throw KsError{KS_ERR_INVALID, "StandardScalerModel: the mean must be finite and the std finite and non-zero"};
  auto out = new_matrix(X.rows, d);
  DevBuf ms;
  ms.alloc(sizeof(double) * static_cast<size_t>(2 * std::max<int64_t>(d, 1)));
  KS_CUDA(cudaMemcpyAsync(ms.p, mean, sizeof(double) * d, cudaMemcpyHostToDevice, c.st));
  if (std_or_null) KS_CUDA(cudaMemcpyAsync(ms.as<double>() + d, std_or_null, sizeof(double) * d, cudaMemcpyHostToDevice, c.st));
  if (X.rows > 0) {
    scaler_apply_kernel<<<grid_for(X.rows * X.ld, 256, c), 256, 0, c.st>>>(X.d, out->d, X.ld, X.rows, d, ms.as<double>(),
                                                                            std_or_null ? ms.as<double>() + d : nullptr);
    c.launches += 1;
  }
  c.check_async("StandardScalerModel.apply");
  return out;
}

// ------------------------------------------------------------------------------------------------- AugmentedExamplesEvaluator
// One CTA per group g: views rows[offs[g] .. offs[g+1]) in that order.  Thread j owns class j: average adds the score, borda the
// rank of class j in the view's ascending stable sort (the classes i with s_i < s_j, or s_i == s_j and i < j).  Average then
// divides by the view count.  Thread 0 takes the first maximum and counts (label, prediction).
__global__ void __launch_bounds__(256) grouped_confusion_kernel(const float* __restrict__ scores, int64_t ld, const int64_t* __restrict__ rows,
                                                                const int64_t* __restrict__ offs, const int32_t* __restrict__ glabel, int k,
                                                                int policy, unsigned long long* __restrict__ counts) {
  extern __shared__ double acc[];
  const int64_t g = blockIdx.x;
  const int64_t v0 = offs[g], v1 = offs[g + 1];
  for (int j = threadIdx.x; j < k; j += blockDim.x) {
    double a = 0.0;
    for (int64_t v = v0; v < v1; ++v) {
      const float* s = scores + rows[v] * ld;
      if (policy == 0) {
        a = __dadd_rn(a, static_cast<double>(s[j]));
      } else {
        const float sj = s[j];
        int rank = 0;
        for (int i = 0; i < k; ++i) {
          const float si = s[i];
          rank += (si < sj || (si == sj && i < j)) ? 1 : 0;
        }
        a = __dadd_rn(a, static_cast<double>(rank));
      }
    }
    acc[j] = policy == 0 ? __ddiv_rn(a, static_cast<double>(v1 - v0)) : a;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int best = 0;
    for (int j = 1; j < k; ++j)
      if (acc[j] > acc[best]) best = j;
    atomicAdd(counts + static_cast<int64_t>(glabel[g]) * k + best, 1ULL);
  }
}

void grouped_confusion_matrix(Ctx& c, Matrix& scores, const int64_t* rows, const int64_t* group_offsets, int64_t n_groups,
                              const int32_t* labels, int64_t k, int policy, double* out) {
  if (!rows || !group_offsets || !labels || !out) throw KsError{KS_ERR_INVALID, "grouped confusion matrix: null argument"};
  if (policy != 0 && policy != 1) throw KsError{KS_ERR_INVALID, "grouped confusion matrix: policy must be 0 (average) or 1 (borda)"};
  if (k < 1 || k > kMaxEvalClasses || k != scores.cols)
    throw KsError{KS_ERR_INVALID, "grouped confusion matrix: k must equal the score columns and lie in [1, 4096]"};
  if (n_groups < 0 || n_groups > 0x7fffffffLL) throw KsError{KS_ERR_INVALID, "grouped confusion matrix: bad group count"};
  const int64_t n = scores.rows;
  if (group_offsets[0] != 0 || group_offsets[n_groups] != n)
    throw KsError{KS_ERR_INVALID, "grouped confusion matrix: group offsets must run from 0 to the score rows"};
  std::vector<char> seen(static_cast<size_t>(n), 0);
  std::vector<int32_t> glabel(static_cast<size_t>(n_groups));
  for (int64_t g = 0; g < n_groups; ++g) {
    if (group_offsets[g + 1] <= group_offsets[g]) throw KsError{KS_ERR_INVALID, "grouped confusion matrix: an empty or decreasing group"};
    for (int64_t v = group_offsets[g]; v < group_offsets[g + 1]; ++v) {
      const int64_t r = rows[v];
      if (r < 0 || r >= n || seen[r]) throw KsError{KS_ERR_INVALID, "grouped confusion matrix: rows must be a permutation of the score rows"};
      seen[r] = 1;
      if (labels[r] < 0 || labels[r] >= k) throw KsError{KS_ERR_INVALID, "grouped confusion matrix: a label outside [0, k)"};
      if (labels[r] != labels[rows[group_offsets[g]]])
        throw KsError{KS_ERR_INVALID, "grouped confusion matrix: the views of group " + std::to_string(g) + " carry different labels"};
    }
    glabel[g] = labels[rows[group_offsets[g]]];
  }
  DevBuf d_rows, d_offs, d_lab, d_cnt;
  d_rows.alloc(sizeof(int64_t) * static_cast<size_t>(n));
  d_offs.alloc(sizeof(int64_t) * static_cast<size_t>(n_groups + 1));
  d_lab.alloc(sizeof(int32_t) * static_cast<size_t>(n_groups));
  d_cnt.alloc(sizeof(unsigned long long) * static_cast<size_t>(k * k));
  KS_CUDA(cudaMemcpyAsync(d_rows.p, rows, sizeof(int64_t) * n, cudaMemcpyHostToDevice, c.st));
  KS_CUDA(cudaMemcpyAsync(d_offs.p, group_offsets, sizeof(int64_t) * (n_groups + 1), cudaMemcpyHostToDevice, c.st));
  KS_CUDA(cudaMemcpyAsync(d_lab.p, glabel.data(), sizeof(int32_t) * n_groups, cudaMemcpyHostToDevice, c.st));
  KS_CUDA(cudaMemsetAsync(d_cnt.p, 0, d_cnt.bytes, c.st));
  if (n_groups > 0) {
    const size_t smem = sizeof(double) * static_cast<size_t>(k);
    if (smem > 48 * 1024) KS_CUDA(cudaFuncSetAttribute(grouped_confusion_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    grouped_confusion_kernel<<<static_cast<unsigned>(n_groups), 256, smem, c.st>>>(scores.d, scores.ld, d_rows.as<int64_t>(), d_offs.as<int64_t>(),
                                                                                   d_lab.as<int32_t>(), static_cast<int>(k), policy,
                                                                                   d_cnt.as<unsigned long long>());
    c.launches += 1;
  }
  std::vector<unsigned long long> cnt(static_cast<size_t>(k * k));
  KS_CUDA(cudaMemcpyAsync(cnt.data(), d_cnt.p, d_cnt.bytes, cudaMemcpyDeviceToHost, c.st));
  c.check_async("AugmentedExamplesEvaluator");
  for (int64_t i = 0; i < k * k; ++i) out[i] = static_cast<double>(cnt[i]);
}

}  // namespace ks
