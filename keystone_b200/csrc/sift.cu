// Dense multi-scale SIFT on the device: PixelScaler, GrayScaler and SIFTExtractor (K/nodes/images/{PixelScaler,GrayScaler}.scala,
// K/nodes/images/external/SIFTExtractor.scala and its vlfeat driver VLFeat.cxx).  DESIGN.md section 18.
//
// Per scale s (bin b = bin + 2s, step step + s scaleStep), for a chunk of equal-size images at once (the image is a grid dimension):
//   smooth      the ORIGINAL gray image by a Gaussian of sigma b / 6 (radius ceil(4 sigma), continuity padding), column pass then row
//               pass, taps accumulated in ascending source order (vl_imsmooth_f);
//   gradients   central differences, vl_fast_sqrt_f / vl_fast_atan2_f, the magnitude split between the two nearest of 8 orientation
//               planes;
//   triangle    each plane convolved along y then along x by the unit-area triangle max(b - |t|, 0) / b^2, from two running sums in
//               vlfeat's order (vl_imconvcoltri_f), one thread per line;
//   descriptor  one warp per keypoint, 4 values per lane: the window-weighted samples, the mass, L2 normalise / clamp at 0.2 /
//               normalise, the contrast threshold, vl_dsift_transpose_descriptor and min((unsigned)(512 v), 255).
// Every rounding step is an explicit __f*_rn / __d*_rn intrinsic, so nothing is contracted to an FMA and the result is the fp32
// operation sequence of vlfeat's x86 build; the sums a descriptor needs are taken sequentially in vlfeat's order.  No float
// atomics: a repeated call returns identical bits.
//
// vlfeat works on the image transposed: the reference passes width = xDim (the Image's rows) and a float array with x fastest, which
// is exactly the ImageVectorizer row of a one-channel image.  So "W" below is x_dim, "H" is y_dim, and pixel (vx, vy) is at vx + vy W.
#include "engine.h"

#include <float.h>
#include <math.h>

#include <algorithm>
#include <vector>

namespace ks {

static constexpr int kNumBinT = 8, kNumBinXY = 4, kDescr = 128;
static constexpr int kDescWarps = 8;  // keypoints per 256-thread CTA

// ------------------------------------------------------------------------------------------------------ image preparation
// out (fp32) = in / 255.0 in fp64, rounded once (PixelScaler without a following GrayScaler)
__global__ void pixel_scale_kernel(const float* __restrict__ in, int64_t ldi, int64_t cols, float* __restrict__ out, int64_t ldo) {
  const int64_t i = blockIdx.y;
  for (int64_t j = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; j < cols; j += static_cast<int64_t>(gridDim.x) * blockDim.x)
    out[i * ldo + j] = __double2float_rn(__ddiv_rn(static_cast<double>(in[i * ldi + j]), 255.0));
}

// GrayScaler (ImageUtils.toGrayScale) in fp64, optionally after PixelScaler's x / 255.0, rounded once to fp32.  Three channels (BGR):
// 0.2989 R + 0.5870 G + 0.1140 B left to right; otherwise sqrt(sum_c v^2 / C).  Pixel p (= x + y x_dim) at in[p C + c].
__global__ void grayscale_kernel(const float* __restrict__ in, int64_t ldi, int64_t npx, int ch, int scale, float* __restrict__ out,
                                 int64_t ldo) {
  const int64_t i = blockIdx.y;
  for (int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; p < npx; p += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float* px = in + i * ldi + p * ch;
    auto val = [&](int c) {
      const double v = static_cast<double>(px[c]);
      return scale ? __ddiv_rn(v, 255.0) : v;
    };
    double g;
    if (ch == 3) {
      g = __dadd_rn(__dadd_rn(__dmul_rn(0.2989, val(2)), __dmul_rn(0.5870, val(1))), __dmul_rn(0.1140, val(0)));
    } else {
      double acc = 0.0;
      for (int c = 0; c < ch; ++c) acc = __dadd_rn(acc, __dmul_rn(val(c), val(c)));
      g = __dsqrt_rn(__ddiv_rn(acc, static_cast<double>(ch)));
    }
    out[i * ldo + p] = __double2float_rn(g);
  }
}

// bad[0] |= 1 if any of the first `cols` values of a row is not finite
__global__ void nonfinite_kernel(const float* __restrict__ in, int64_t ld, int64_t cols, unsigned* __restrict__ bad) {
  const int64_t i = blockIdx.y;
  unsigned any = 0;
  for (int64_t j = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; j < cols; j += static_cast<int64_t>(gridDim.x) * blockDim.x)
    any |= !isfinite(in[i * ld + j]);
  if (__any_sync(0xffffffffu, any) && (threadIdx.x & 31) == 0) atomicOr(bad, 1u);
}

// --------------------------------------------------------------------------------------------------------------- smoothing
// vl_imconvcol_f with continuity padding along y (along_x = 0) or x: out[v] = sum over p = v - r .. v + r, ascending, of
// in[clamp(p)] f[p - v + r], accumulated from 0.  Image i at in + i ldi, out + i ldo.
__global__ void smooth_kernel(const float* __restrict__ in, int64_t ldi, float* __restrict__ out, int64_t ldo, int H, int W,
                              const float* __restrict__ f, int r, int along_x) {
  const int64_t i = blockIdx.y, npx = static_cast<int64_t>(H) * W;
  const float* src = in + i * ldi;
  for (int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; p < npx; p += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(p % W), y = static_cast<int>(p / W);
    float acc = 0.f;
    for (int k = -r; k <= r; ++k) {
      const float v = along_x ? src[static_cast<int64_t>(y) * W + min(max(x + k, 0), W - 1)]
                              : src[static_cast<int64_t>(min(max(y + k, 0), H - 1)) * W + x];
      acc = __fadd_rn(acc, __fmul_rn(v, f[k + r]));
    }
    out[i * ldo + p] = acc;
  }
}

// --------------------------------------------------------------------------------------------------------------- gradients
__device__ __forceinline__ float fast_sqrt(float x) {  // vl_fast_sqrt_f (the 1e-8 literal is a double)
  if (static_cast<double>(x) < 1e-8) return 0.f;
  const float xhalf = __fmul_rn(0.5f, x);
  float y = __int_as_float(0x5f3759df - (__float_as_int(x) >> 1));
  y = __fmul_rn(y, __fsub_rn(1.5f, __fmul_rn(__fmul_rn(xhalf, y), y)));
  y = __fmul_rn(y, __fsub_rn(1.5f, __fmul_rn(__fmul_rn(xhalf, y), y)));
  return __fmul_rn(x, y);
}

__device__ __forceinline__ float fast_atan2(float y, float x) {  // vl_fast_atan2_f
  const float abs_y = __fadd_rn(fabsf(y), FLT_EPSILON);
  float r, angle;
  if (x >= 0.f) {
    r = __fdiv_rn(__fsub_rn(x, abs_y), __fadd_rn(x, abs_y));
    angle = static_cast<float>(M_PI / 4);
  } else {
    r = __fdiv_rn(__fadd_rn(x, abs_y), __fsub_rn(abs_y, x));
    angle = static_cast<float>(3 * M_PI / 4);
  }
  angle = __fadd_rn(angle, __fmul_rn(__fsub_rn(__fmul_rn(__fmul_rn(0.1821f, r), r), 0.9675f), r));
  return y < 0.f ? -angle : angle;
}

// planes[(i 8 + t) H W + p] = the part of the gradient magnitude of pixel p that falls in orientation bin t (vl_dsift_process)
__global__ void gradient_bin_kernel(const float* __restrict__ im, int64_t ldi, int H, int W, float* __restrict__ planes) {
  const int64_t i = blockIdx.y, npx = static_cast<int64_t>(H) * W;
  const float* a = im + i * ldi;
  for (int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; p < npx; p += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(p % W), y = static_cast<int>(p / W);
    float gy, gx;
    if (y == 0) gy = __fsub_rn(a[p + W], a[p]);
    else if (y == H - 1) gy = __fsub_rn(a[p], a[p - W]);
    else gy = __fmul_rn(0.5f, __fsub_rn(a[p + W], a[p - W]));
    if (x == 0) gx = __fsub_rn(a[p + 1], a[p]);
    else if (x == W - 1) gx = __fsub_rn(a[p], a[p - 1]);
    else gx = __fmul_rn(0.5f, __fsub_rn(a[p + 1], a[p - 1]));
    float angle = fast_atan2(gy, gx);
    const float mod = fast_sqrt(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)));
    const float two_pi = static_cast<float>(2 * M_PI);
    while (angle > two_pi) angle = __fsub_rn(angle, two_pi);  // vl_mod_2pi_f
    while (angle < 0.f) angle = __fadd_rn(angle, two_pi);
    const float nt = __double2float_rn(__dmul_rn(static_cast<double>(angle), kNumBinT / (2 * M_PI)));
    const int bint = static_cast<int>(floorf(nt));
    const float rbint = __fsub_rn(nt, static_cast<float>(bint));
    const int t0 = bint % kNumBinT, t1 = (bint + 1) % kNumBinT;
    const float v0 = __fmul_rn(__fsub_rn(1.f, rbint), mod), v1 = __fmul_rn(rbint, mod);
    float* out = planes + i * kNumBinT * npx + p;
#pragma unroll
    for (int t = 0; t < kNumBinT; ++t) out[t * npx] = t == t0 ? v0 : (t == t1 ? v1 : 0.f);
  }
}

// ---------------------------------------------------------------------------------------------------------- triangle filter
// vl_imconvcoltri_f with continuity padding along each line of every plane (blockIdx.y): element e of line l of plane q at
// q plane_stride + l line_stride + e elem_stride (same layout in and out).  S [q][len + F][n_lines] holds the backward integral,
// overwritten in place by the forward one:
//   B[j] (j = len + F - 1 down to 0) = sum of ext[j..], ext[j] = in[j - F] for j >= F, in[0] below;
//   R[j] = B[j] - B[j + F] for j < len, B[j] - in[len - 1] (len - j) above;  C = running sum of R;  out[e] = (C[e + F] - C[e]) / F^2.
__global__ void tri_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t plane_stride, int n_lines, int len,
                           int line_stride, int elem_stride, int F, float scale, float* __restrict__ S) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= n_lines) return;
  const int64_t q = blockIdx.y;
  const float* src = in + q * plane_stride + static_cast<int64_t>(l) * line_stride;
  float* dst = out + q * plane_stride + static_cast<int64_t>(l) * line_stride;
  float* s = S + q * static_cast<int64_t>(len + F) * n_lines + l;
  const float last = src[static_cast<int64_t>(len - 1) * elem_stride], first = src[0];
  float acc = last;
  s[static_cast<int64_t>(len + F - 1) * n_lines] = acc;
  for (int j = len + F - 2; j >= 0; --j) {
    acc = __fadd_rn(acc, j >= F ? src[static_cast<int64_t>(j - F) * elem_stride] : first);
    s[static_cast<int64_t>(j) * n_lines] = acc;
  }
  float c = 0.f;
  for (int j = 0; j < len + F; ++j) {
    const float b = s[static_cast<int64_t>(j) * n_lines];
    const float r = j < len ? __fsub_rn(b, s[static_cast<int64_t>(j + F) * n_lines])
                            : __fsub_rn(b, __fmul_rn(last, static_cast<float>(len - j)));
    c = j == 0 ? r : __fadd_rn(c, r);
    s[static_cast<int64_t>(j) * n_lines] = c;
    if (j >= F) dst[static_cast<int64_t>(j - F) * elem_stride] = __fmul_rn(scale, __fsub_rn(c, s[static_cast<int64_t>(j - F) * n_lines]));
  }
}

// ------------------------------------------------------------------------------------------------------------- descriptors
struct DescGeom {
  int b, st, lo, nfx, nfy;
  float norm_const;  // (3 b + 1)^2
};

// the sum of the 128 values (lane l holds 4l .. 4l + 3) in index order, identical on every lane
__device__ __forceinline__ float ordered_sum(const float (&v)[4]) {
  float s = 0.f;
  for (int L = 0; L < 32; ++L)
#pragma unroll
    for (int k = 0; k < 4; ++k) s = __fadd_rn(s, __shfl_sync(0xffffffffu, v[k], L));
  return s;
}

__device__ __forceinline__ void normalize(float (&v)[4]) {  // _vl_dsift_normalize_histogram
  float sq[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) sq[k] = __fmul_rn(v[k], v[k]);
  const float n = __fadd_rn(fast_sqrt(ordered_sum(sq)), FLT_EPSILON);
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = __fdiv_rn(v[k], n);
}

// One warp per keypoint (frames vy-outer, vx-inner); w[by 4 + bx] = (wx b) (wy b), the window means times the bin size.  Raw layout t + 8 bx + 32 by: lane l holds by = l / 8, bx = (l / 2) % 4,
// t = 4 (l % 2) + k.  Writes row (i rows_per_image + row0 + kp) of out, values min((unsigned)(512 v), 255) in transposed order.
__global__ void __launch_bounds__(32 * kDescWarps) descriptor_kernel(const float* __restrict__ planes, int H, int W, DescGeom g,
                                                                    const float* __restrict__ w,
                                                                    float* __restrict__ out, int64_t ldo, int64_t rows_per_image,
                                                                    int64_t row0) {
  const int lane = threadIdx.x & 31;
  const int64_t kp = static_cast<int64_t>(blockIdx.x) * kDescWarps + (threadIdx.x >> 5);
  const int64_t nkp = static_cast<int64_t>(g.nfx) * g.nfy;
  if (kp >= nkp) return;
  const int64_t i = blockIdx.y, npx = static_cast<int64_t>(H) * W;
  const int fy = static_cast<int>(kp / g.nfx), fx = static_cast<int>(kp % g.nfx);
  const int by = lane >> 3, bx = (lane >> 1) & 3;
  const int y = g.lo + fy * g.st + by * g.b, x = g.lo + fx * g.st + bx * g.b;
  const float wt = w[by * kNumBinXY + bx];
  const float* src = planes + (i * kNumBinT + 4 * (lane & 1)) * npx + static_cast<int64_t>(y) * W + x;
  float v[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = __fmul_rn(wt, src[k * npx]);
  const float mass = __fdiv_rn(ordered_sum(v), g.norm_const);
  normalize(v);
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = v[k] > 0.2f ? 0.2f : v[k];
  normalize(v);
  const bool keep = !(mass < 0.005f);
  // vl_dsift_transpose_descriptor(., 8, 4, 4): output j = 8 (y + 4 x) + tT takes raw 8 (x + 4 y) + (10 - tT) % 8
  float o[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int j = 4 * lane + k, yy = (j >> 3) & 3, xx = j >> 5, t = (10 - (j & 7)) & 7;
    const int p = kNumBinT * (xx + kNumBinXY * yy) + t;
    float a[4];
#pragma unroll
    for (int m = 0; m < 4; ++m) a[m] = __shfl_sync(0xffffffffu, v[m], p >> 2);
    const int m = p & 3;
    const float d = m == 0 ? a[0] : m == 1 ? a[1] : m == 2 ? a[2] : a[3];
    const unsigned u = __float2uint_rz(__fmul_rn(512.f, d));
    o[k] = keep ? static_cast<float>(u < 255u ? u : 255u) : 0.f;
  }
  *reinterpret_cast<float4*>(out + (i * rows_per_image + row0 + kp) * ldo + 4 * lane) = make_float4(o[0], o[1], o[2], o[3]);
}

// ------------------------------------------------------------------------------------------------------------------ host side
static unsigned blocks_for(int64_t work, int threads, const Ctx& c) {
  return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((work + threads - 1) / threads, 8LL * c.num_sms)));
}

std::vector<SiftScale> sift_geometry(int x_dim, int y_dim, int step, int bin, int scales, int scale_step) {
  if (x_dim <= 0 || y_dim <= 0) throw KsError{KS_ERR_INVALID, "SIFTExtractor: image dimensions must be positive"};
  if (step < 1 || bin < 1 || scales < 1 || scale_step < 0)
    throw KsError{KS_ERR_INVALID, "SIFTExtractor: stepSize, binSize and scales must be >= 1, scaleStep >= 0"};
  if (step > (1 << 16) || bin > (1 << 12) || scales > 256 || scale_step > (1 << 16))
    throw KsError{KS_ERR_INVALID, "SIFTExtractor: stepSize, scaleStep <= 65536, binSize <= 4096, scales <= 256"};
  std::vector<SiftScale> g(static_cast<size_t>(scales));
  for (int s = 0; s < scales; ++s) {
    SiftScale& q = g[static_cast<size_t>(s)];
    q.b = bin + 2 * s;
    q.st = step + s * scale_step;
    q.lo = std::max(1 + 2 * scales - 3 * s, 0);  // VLFeat.cxx:93-95; vl_dsift_set_bounds clamps a negative minimum to 0
    auto frames = [&](int dim) {
      const int range = (dim - 1) - q.lo - (kNumBinXY - 1) * q.b;
      return range >= 0 ? range / q.st + 1 : 0;
    };
    q.nfx = frames(x_dim);
    q.nfy = frames(y_dim);
  }
  return g;
}

static float bin_window_mean(int bin, int index) {  // _vl_dsift_get_bin_window_mean with windowSize 1.5
  const float delta = static_cast<float>(bin) * (static_cast<float>(index) - 0.5f * static_cast<float>(kNumBinXY - 1));
  const float sigma = static_cast<float>(bin) * 1.5f;
  float acc = 0.f;
  for (int x = -bin + 1; x <= bin - 1; ++x) {
    const float z = (static_cast<float>(x) - delta) / sigma;
    const float e = (-0.5f * z) * z;
    acc = static_cast<float>(static_cast<double>(acc) + std::exp(static_cast<double>(e)));
  }
  return acc / static_cast<float>(2 * bin - 1);
}

void check_finite(Ctx& c, const Matrix& m, int64_t cols, const char* who) {
  if (m.rows == 0) return;
  DevBuf flag;
  flag.alloc(sizeof(unsigned));
  KS_CUDA(cudaMemsetAsync(flag.p, 0, sizeof(unsigned), c.st));
  for (int64_t i0 = 0; i0 < m.rows; i0 += 65535) {
    const int64_t ni = std::min<int64_t>(65535, m.rows - i0);
    nonfinite_kernel<<<dim3(blocks_for(cols, 256, c), static_cast<unsigned>(ni)), 256, 0, c.st>>>(m.d + i0 * m.ld, m.ld, cols,
                                                                                                  flag.as<unsigned>());
    c.launches += 1;
  }
  unsigned h = 0;
  KS_CUDA(cudaMemcpyAsync(&h, flag.p, sizeof(unsigned), cudaMemcpyDeviceToHost, c.st));
  c.check_async(who);
  if (h) throw KsError{KS_ERR_INVALID, std::string(who) + ": the images have non-finite pixels"};
}

std::unique_ptr<Matrix> image_pixel_scale(Ctx& c, Matrix& im) {
  check_finite(c, im, im.cols, "PixelScaler");
  auto out = new_matrix(im.rows, im.cols);
  if (out->ld != im.cols) KS_CUDA(cudaMemsetAsync(out->d, 0, out->buf.bytes, c.st));
  for (int64_t i0 = 0; i0 < im.rows; i0 += 65535) {
    const int64_t ni = std::min<int64_t>(65535, im.rows - i0);
    pixel_scale_kernel<<<dim3(blocks_for(im.cols, 256, c), static_cast<unsigned>(ni)), 256, 0, c.st>>>(im.d + i0 * im.ld, im.ld, im.cols,
                                                                                                      out->d + i0 * out->ld, out->ld);
    c.launches += 1;
  }
  c.check_async("PixelScaler.apply");
  return out;
}

std::unique_ptr<Matrix> image_grayscale(Ctx& c, Matrix& im, int x_dim, int y_dim, int ch, int pixel_scale) {
  if (x_dim <= 0 || y_dim <= 0 || ch <= 0) throw KsError{KS_ERR_INVALID, "GrayScaler: dimensions and channels must be positive"};
  const int64_t npx = static_cast<int64_t>(x_dim) * y_dim;
  if (im.cols != npx * ch) throw KsError{KS_ERR_INVALID, "GrayScaler: image size does not match the matrix"};
  if (pixel_scale != 0 && pixel_scale != 1) throw KsError{KS_ERR_INVALID, "GrayScaler: pixel_scale must be 0 or 1"};
  check_finite(c, im, im.cols, "GrayScaler");
  auto out = new_matrix(im.rows, npx);
  if (out->ld != npx) KS_CUDA(cudaMemsetAsync(out->d, 0, out->buf.bytes, c.st));
  for (int64_t i0 = 0; i0 < im.rows; i0 += 65535) {
    const int64_t ni = std::min<int64_t>(65535, im.rows - i0);
    grayscale_kernel<<<dim3(blocks_for(npx, 256, c), static_cast<unsigned>(ni)), 256, 0, c.st>>>(im.d + i0 * im.ld, im.ld, npx, ch,
                                                                                                 pixel_scale, out->d + i0 * out->ld, out->ld);
    c.launches += 1;
  }
  c.check_async("GrayScaler.apply");
  return out;
}

std::unique_ptr<Matrix> sift_extract(Ctx& c, Matrix& im, int x_dim, int y_dim, int step, int bin, int scales, int scale_step) {
  const std::vector<SiftScale> geo = sift_geometry(x_dim, y_dim, step, bin, scales, scale_step);
  const int W = x_dim, H = y_dim;
  const int64_t npx = static_cast<int64_t>(W) * H;
  if (im.cols != npx) throw KsError{KS_ERR_INVALID, "SIFTExtractor: the images must have one channel of x_dim * y_dim pixels"};
  check_finite(c, im, im.cols, "SIFTExtractor");
  int64_t nkp = 0;
  int max_f = 0;
  std::vector<int64_t> row0;
  std::vector<float> taps;
  std::vector<int> tap0, w0;  // per scale: offsets of the smoothing taps and of the bin weights in `taps`
  for (const SiftScale& q : geo) {
    row0.push_back(nkp);
    nkp += static_cast<int64_t>(q.nfx) * q.nfy;
    max_f = std::max(max_f, q.b);
    // vl_imsmooth_f's kernel: radius ceil(4 sigma), exp in fp64 stored as fp32, divided by the fp32 sum of the taps in order
    const double sigma = q.b / 6.0;
    const int r = static_cast<int>(std::ceil(sigma * 4.0));
    tap0.push_back(static_cast<int>(taps.size()));
    float mass = 0.f;
    for (int j = 0; j <= 2 * r; ++j) {
      const double x = (j - r) / sigma;
      taps.push_back(static_cast<float>(std::exp(-0.5 * x * x)));
      mass = mass + taps.back();
    }
    for (int j = 0; j <= 2 * r; ++j) taps[static_cast<size_t>(tap0.back() + j)] /= mass;
    // the spatial-bin weights w[by 4 + bx] = (wx b) (wy b) of _vl_dsift_with_flat_window
    float wm[kNumBinXY];
    for (int k = 0; k < kNumBinXY; ++k) wm[k] = bin_window_mean(q.b, k) * static_cast<float>(q.b);
    w0.push_back(static_cast<int>(taps.size()));
    for (int by = 0; by < kNumBinXY; ++by)
      for (int bx = 0; bx < kNumBinXY; ++bx) taps.push_back(wm[bx] * wm[by]);
  }
  auto out = new_matrix(im.rows * nkp, kDescr);
  if (nkp == 0 || im.rows == 0) return out;
  DevBuf dtaps;
  dtaps.alloc(sizeof(float) * taps.size());
  KS_CUDA(cudaMemcpyAsync(dtaps.p, taps.data(), sizeof(float) * taps.size(), cudaMemcpyHostToDevice, c.st));
  // scratch per image: planes A and B (8 H W each; B also holds the smoothing passes) and the running sums of the triangle filter
  const int64_t per_plane_s = npx + static_cast<int64_t>(max_f) * std::max(H, W);
  const int64_t per_img = 2 * kNumBinT * npx + kNumBinT * per_plane_s;
  const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>({im.rows, (int64_t(256) << 20) / (4 * per_img), 8191}));
  DevBuf scratch;
  scratch.alloc(sizeof(float) * static_cast<size_t>(chunk * per_img));
  float* A = scratch.as<float>();
  float* B = A + chunk * kNumBinT * npx;
  float* S = B + chunk * kNumBinT * npx;
  const int64_t ld_b = kNumBinT * npx;  // image stride of the smoothing buffers inside B
  for (int64_t i0 = 0; i0 < im.rows; i0 += chunk) {
    const int64_t ni = std::min(chunk, im.rows - i0);
    const unsigned gpx = blocks_for(npx, 256, c);
    for (size_t s = 0; s < geo.size(); ++s) {
      const SiftScale& q = geo[s];
      if (static_cast<int64_t>(q.nfx) * q.nfy == 0) continue;  // a scale without frames contributes no rows
      const int r = static_cast<int>(std::ceil(q.b / 6.0 * 4.0));
      const float* f = dtaps.as<float>() + tap0[s];
      smooth_kernel<<<dim3(gpx, static_cast<unsigned>(ni)), 256, 0, c.st>>>(im.d + i0 * im.ld, im.ld, B, ld_b, H, W, f, r, 0);
      smooth_kernel<<<dim3(gpx, static_cast<unsigned>(ni)), 256, 0, c.st>>>(B, ld_b, B + npx, ld_b, H, W, f, r, 1);
      gradient_bin_kernel<<<dim3(gpx, static_cast<unsigned>(ni)), 256, 0, c.st>>>(B + npx, ld_b, H, W, A);
      const float scale = static_cast<float>(1.0 / (static_cast<double>(q.b) * static_cast<double>(q.b)));
      const unsigned planes = static_cast<unsigned>(ni * kNumBinT);
      tri_kernel<<<dim3((W + 127) / 128, planes), 128, 0, c.st>>>(A, B, npx, W, H, 1, W, q.b, scale, S);  // along y, one line per x
      tri_kernel<<<dim3((H + 127) / 128, planes), 128, 0, c.st>>>(B, A, npx, H, W, W, 1, q.b, scale, S);  // along x, one line per y
      DescGeom g;
      g.b = q.b;
      g.st = q.st;
      g.lo = q.lo;
      g.nfx = q.nfx;
      g.nfy = q.nfy;
      g.norm_const = static_cast<float>((3 * q.b + 1) * (3 * q.b + 1));
      const int64_t n = static_cast<int64_t>(q.nfx) * q.nfy;
      descriptor_kernel<<<dim3(static_cast<unsigned>((n + kDescWarps - 1) / kDescWarps), static_cast<unsigned>(ni)), 32 * kDescWarps, 0,
                          c.st>>>(A, H, W, g, dtaps.as<float>() + w0[s], out->d + i0 * nkp * out->ld, out->ld, nkp, row0[s]);
      c.launches += 6;
    }
  }
  c.check_async("SIFTExtractor.apply");
  return out;
}

}  // namespace ks
