// HOG and DAISY descriptors on the device: HogExtractor and DaisyExtractor (K/nodes/images/{HogExtractor,DaisyExtractor}.scala,
// ImageUtils.conv2D).  DESIGN.md section 19.
//
// HOG, for a chunk of equal-size three-channel images at once (the image is a grid dimension):
//   gradient   per pixel of the visible area, the channel with the largest dx^2 + dy^2 (scanned 2, 1, 0, strict >), its fp64
//              magnitude and its snap to one of 18 orientations; reads are the reference's unclamped flat reads c + x C + y C xDim;
//   histogram  a gather: one warp per cell, lane o < 18 owns bin o and walks the cell's support in the reference's pixel order
//              (x outer, y inner), so each fp32 bin receives its bilinear addends in the order the reference's scatter adds them;
//   norms      per cell, sum over o < 9 of (h_o + h_{o+9})^2 in fp32;
//   features   per interior cell, the 32 voc-release5 values in fp64 from fp32 histograms, rounded once.
// DAISY, on one-channel images, every plane fp64 with values (x, y) at x + y xDim:
//   gradients  conv2D with [1, 0, -1] / [1, 2, 1] (a pass along x, then along y, zero padding, reversed filters);
//   layers     per orientation a < H the rectified max(cos a ix + sin a iy, 0), fused into the first pass along x of the
//              Gaussian blur, then one separable blur per layer;
//   descriptor one warp per keypoint, lane j owns histogram j (the centre, then ring sample (t, l) at j = 1 + t Q + l, which is
//              also its column block), normalised in fp64 and stored once as fp32.
// Every rounding step is an explicit __f*_rn / __d*_rn intrinsic, so nothing is contracted to an FMA; every running sum is taken
// in the reference's order by one thread.  No float atomics: a repeated call returns identical bits.
#include "engine.h"

#include <math.h>

#include <algorithm>
#include <vector>

namespace ks {

static constexpr int kHogOri = 18, kHogFeatures = 32;
static constexpr int kCellWarps = 4;   // HOG cells per 128-thread CTA
static constexpr int kKpWarps = 8;     // DAISY keypoints per 256-thread CTA
static constexpr int64_t kScratchBytes = int64_t(256) << 20;

__constant__ double c_hog_uu[9] = {1.0000, 0.9397, 0.7660, 0.500, 0.1736, -0.1736, -0.5000, -0.7660, -0.9397};
__constant__ double c_hog_vv[9] = {0.0000, 0.3420, 0.6428, 0.8660, 0.9848, 0.9848, 0.8660, 0.6428, 0.3420};

static unsigned grid_for(int64_t work, int threads, const Ctx& c) {
  return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((work + threads - 1) / threads, 8LL * c.num_sms)));
}

// ------------------------------------------------------------------------------------------------------------------------ HOG
struct HogGeom {
  int x_dim, nx, ny, vx, vy, bin, scale;  // visible area vx = nx bin by vy = ny bin
};

// mag[p], ori[p] for p = x + y vx, 1 <= x < vx - 1, 1 <= y < vy - 1 (the reference's pixel loop).  Image i at in + i ldi.
__global__ void hog_gradient_kernel(const float* __restrict__ in, int64_t ldi, HogGeom g, double* __restrict__ mag,
                                    unsigned char* __restrict__ ori) {
  const int64_t i = blockIdx.y, w = g.vx - 2, n = w * static_cast<int64_t>(g.vy - 2), plane = static_cast<int64_t>(g.vx) * g.vy;
  const float* src = in + i * ldi;
  for (int64_t q = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; q < n; q += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int x = 1 + static_cast<int>(q % w), y = 1 + static_cast<int>(q / w);
    auto get = [&](int xx, int yy, int c) {  // ChannelMajorArrayVectorizedImage.get without bounds: c + x 3 + y 3 xDim
      const double v = static_cast<double>(src[c + 3 * static_cast<int64_t>(xx) + 3 * static_cast<int64_t>(yy) * g.x_dim]);
      return g.scale ? __ddiv_rn(v, 255.0) : v;
    };
    double best = -INFINITY, bdx = 0.0, bdy = 0.0;
    for (int c = 2; c >= 0; --c) {
      const double dx = __dsub_rn(get(x + 1, y, c), get(x - 1, y, c));
      const double dy = __dsub_rn(get(x, y + 1, c), get(x, y - 1, c));
      const double m2 = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
      if (m2 > best) {
        best = m2;
        bdx = dx;
        bdy = dy;
      }
    }
    double bdot = 0.0;
    int o_best = 0;
#pragma unroll
    for (int o = 0; o < 9; ++o) {
      const double dot = __dadd_rn(__dmul_rn(c_hog_uu[o], bdy), __dmul_rn(c_hog_vv[o], bdx));
      if (dot > bdot) {
        o_best = o;
        bdot = dot;
      } else if (-dot > bdot) {
        o_best = o + 9;
        bdot = -dot;
      }
    }
    const int64_t p = i * plane + x + static_cast<int64_t>(y) * g.vx;
    mag[p] = __dsqrt_rn(best);
    ori[p] = static_cast<unsigned char>(o_best);
  }
}

// the bilinear position of pixel coordinate v: cell index floor((v + 0.5) / bin - 0.5) and the weight toward cell `cell`
// (1 - frac for the lower cell, frac for the upper); false when the pixel does not reach that cell
__device__ __forceinline__ bool hog_weight(int v, int bin, int cell, double* wgt) {
  const double p = __dsub_rn(__ddiv_rn(static_cast<double>(v) + 0.5, static_cast<double>(bin)), 0.5);
  const double f = floor(p);
  const int ip = static_cast<int>(f);
  const double v0 = __dsub_rn(p, f);
  if (ip == cell) {
    *wgt = __dsub_rn(1.0, v0);
    return true;
  }
  if (ip + 1 == cell) {
    *wgt = v0;
    return true;
  }
  return false;
}

// hist[i][o][cy nx + cx]: one warp per cell, lane o < 18 sums its bin over the support in pixel order (x outer, y inner).
__global__ void __launch_bounds__(32 * kCellWarps) hog_hist_kernel(const double* __restrict__ mag, const unsigned char* __restrict__ ori,
                                                                   HogGeom g, float* __restrict__ hist) {
  const int lane = threadIdx.x & 31;
  const int64_t cells = static_cast<int64_t>(g.nx) * g.ny;
  const int64_t cell = static_cast<int64_t>(blockIdx.x) * kCellWarps + (threadIdx.x >> 5);
  if (cell >= cells || lane >= kHogOri) return;
  const int cx = static_cast<int>(cell % g.nx), cy = static_cast<int>(cell / g.nx);
  const int64_t i = blockIdx.y, plane = static_cast<int64_t>(g.vx) * g.vy;
  const double* m = mag + i * plane;
  const unsigned char* r = ori + i * plane;
  // pixel v reaches cells floor((v + 0.5) / bin - 0.5) and the next one; these bounds hold that range with room to spare
  const int half = g.bin / 2;
  const int x0 = max(1, cx * g.bin - half - 1), x1 = min(g.vx - 2, cx * g.bin + g.bin + half + 1);
  const int y0 = max(1, cy * g.bin - half - 1), y1 = min(g.vy - 2, cy * g.bin + g.bin + half + 1);
  float acc = 0.f;
  for (int x = x0; x <= x1; ++x) {
    double wx;
    if (!hog_weight(x, g.bin, cx, &wx)) continue;
    for (int y = y0; y <= y1; ++y) {
      const int64_t p = x + static_cast<int64_t>(y) * g.vx;
      if (r[p] != lane) continue;
      double wy;
      if (!hog_weight(y, g.bin, cy, &wy)) continue;
      acc = __fadd_rn(acc, __double2float_rn(__dmul_rn(__dmul_rn(wy, wx), m[p])));
    }
  }
  hist[(i * kHogOri + lane) * cells + cell] = acc;
}

// norm[i][c] = sum over o < 9 of (h_o + h_{o+9})^2 in fp32, o ascending
__global__ void hog_norm_kernel(const float* __restrict__ hist, int64_t cells, float* __restrict__ norm) {
  const int64_t i = blockIdx.y;
  for (int64_t c = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; c < cells; c += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float* h = hist + i * kHogOri * cells + c;
    float n = 0.f;
    for (int o = 0; o < 9; ++o) {
      const float s = __fadd_rn(h[o * cells], h[(o + 9) * cells]);
      n = __fadd_rn(n, __fmul_rn(s, s));
    }
    norm[i * cells + c] = n;
  }
}

// 1 / sqrt(four fp32 norms added in fp32, then + 1e-4 in fp64) for the 2 x 2 block whose low corner is cell `off`
__device__ __forceinline__ double hog_block(const float* nm, int64_t off, int nx) {
  const float s = __fadd_rn(__fadd_rn(__fadd_rn(nm[off], nm[off + 1]), nm[off + nx]), nm[off + nx + 1]);
  return __ddiv_rn(1.0, __dsqrt_rn(__dadd_rn(static_cast<double>(s), 0.0001)));
}

__device__ __forceinline__ float hog_value(double v, const double (&n)[4], double (&h)[4]) {
#pragma unroll
  for (int k = 0; k < 4; ++k) h[k] = fmin(__dmul_rn(v, n[k]), 0.2);
  return __double2float_rn(__dmul_rn(0.5, __dadd_rn(__dadd_rn(__dadd_rn(h[0], h[1]), h[2]), h[3])));
}

// one thread per interior cell; row y + x (ny - 2) of image i holds its 32 features
__global__ void hog_feature_kernel(const float* __restrict__ hist, const float* __restrict__ norm, HogGeom g, float* __restrict__ out,
                                   int64_t ldo) {
  const int64_t i = blockIdx.y, cells = static_cast<int64_t>(g.nx) * g.ny;
  const int fy = g.ny - 2;
  const int64_t rows = static_cast<int64_t>(g.nx - 2) * fy;
  for (int64_t r = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; r < rows; r += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(r / fy), y = static_cast<int>(r % fy);
    const float* nm = norm + i * cells;
    const double n[4] = {hog_block(nm, static_cast<int64_t>(y + 1) * g.nx + x + 1, g.nx), hog_block(nm, static_cast<int64_t>(y + 1) * g.nx + x, g.nx),
                         hog_block(nm, static_cast<int64_t>(y) * g.nx + x + 1, g.nx), hog_block(nm, static_cast<int64_t>(y) * g.nx + x, g.nx)};
    const float* h = hist + i * kHogOri * cells + static_cast<int64_t>(y + 1) * g.nx + x + 1;
    float* dst = out + (i * rows + r) * ldo;
    double t[4] = {0.0, 0.0, 0.0, 0.0}, hv[4];
    for (int o = 0; o < kHogOri; ++o) {
      dst[o] = hog_value(static_cast<double>(h[o * cells]), n, hv);
#pragma unroll
      for (int k = 0; k < 4; ++k) t[k] = __dadd_rn(t[k], hv[k]);
    }
    for (int o = 0; o < 9; ++o) dst[kHogOri + o] = hog_value(static_cast<double>(__fadd_rn(h[o * cells], h[(o + 9) * cells])), n, hv);
#pragma unroll
    for (int k = 0; k < 4; ++k) dst[27 + k] = __double2float_rn(__dmul_rn(0.2357, t[k]));
    dst[31] = 0.f;
  }
}

// ---------------------------------------------------------------------------------------------------------------------- DAISY
// One pass of ImageUtils.conv2D along x (along_x = 1) or y: out plane q (blockIdx.y) at out + q npx; its input is plane q / in_div
// at in + (q / in_div) ldi and its filter f + (q % nf) len.  out[v] = sum over k ascending of in[v + k - (len - 1) / 2] f[len - 1 - k],
// zero outside the image, accumulated from 0.0.
template <typename T>
__global__ void conv_pass_kernel(const T* __restrict__ in, int64_t ldi, int in_div, double* __restrict__ out, int X, int Y,
                                 const double* __restrict__ f, int len, int nf, int along_x) {
  const int64_t q = blockIdx.y, npx = static_cast<int64_t>(X) * Y;
  const T* src = in + (q / in_div) * ldi;
  const double* fq = f + (q % nf) * len;
  const int pad = (len - 1) / 2;
  for (int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; p < npx; p += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(p % X), y = static_cast<int>(p / X);
    double acc = 0.0;
    for (int k = 0; k < len; ++k) {
      double v = 0.0;
      if (along_x) {
        const int xx = x + k - pad;
        if (xx >= 0 && xx < X) v = static_cast<double>(src[static_cast<int64_t>(y) * X + xx]);
      } else {
        const int yy = y + k - pad;
        if (yy >= 0 && yy < Y) v = static_cast<double>(src[static_cast<int64_t>(yy) * X + x]);
      }
      acc = __dadd_rn(acc, __dmul_rn(v, fq[len - 1 - k]));
    }
    out[q * npx + p] = acc;
  }
}

// The first pass along x of layer 0 for orientation a = q % H of image q / H, on the rectified max(cs[2a] ix + cs[2a+1] iy, 0)
// computed per tap (grad holds ix, iy of image i as planes 2i, 2i + 1).
__global__ void orient_conv_x_kernel(const double* __restrict__ grad, int H, const double* __restrict__ cs, double* __restrict__ out,
                                     int X, int Y, const double* __restrict__ f, int len) {
  const int64_t q = blockIdx.y, npx = static_cast<int64_t>(X) * Y;
  const int64_t i = q / H;
  const int a = static_cast<int>(q % H);
  const double ca = cs[2 * a], sa = cs[2 * a + 1];
  const double* ix = grad + 2 * i * npx;
  const double* iy = ix + npx;
  const int pad = (len - 1) / 2;
  for (int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; p < npx; p += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(p % X), y = static_cast<int>(p / X);
    double acc = 0.0;
    for (int k = 0; k < len; ++k) {
      const int xx = x + k - pad;
      double v = 0.0;
      if (xx >= 0 && xx < X) {
        const int64_t s = static_cast<int64_t>(y) * X + xx;
        const double d = __dadd_rn(__dmul_rn(ca, ix[s]), __dmul_rn(sa, iy[s]));
        v = d > 0.0 ? d : 0.0;
      }
      acc = __dadd_rn(acc, __dmul_rn(v, f[len - 1 - k]));
    }
    out[q * npx + p] = acc;
  }
}

struct DaisyGeom {
  int X, Y, H, Q, n_hist;     // n_hist = 1 + T Q
  int kx0, ky0, nkx, nky, stride;
  int64_t layer_stride;       // distance between layer l and l + 1 inside the chunk's layer block
};

// One warp per keypoint (x outer, y inner).  samp[j] = (dx, dy, layer) of histogram j; lane j normalises histogram j in fp64 (norm
// sqrt of the squares summed in order, zero at or below 1e-8) and writes columns [j H, (j + 1) H) of row (i nkp + kp).
__global__ void __launch_bounds__(32 * kKpWarps) daisy_descriptor_kernel(const double* __restrict__ layers, DaisyGeom g,
                                                                         const int* __restrict__ samp, float* __restrict__ out,
                                                                         int64_t ldo) {
  const int lane = threadIdx.x & 31;
  const int64_t nkp = static_cast<int64_t>(g.nkx) * g.nky;
  const int64_t kp = static_cast<int64_t>(blockIdx.x) * kKpWarps + (threadIdx.x >> 5);
  if (kp >= nkp) return;
  const int64_t i = blockIdx.y, npx = static_cast<int64_t>(g.X) * g.Y;
  const int kx = g.kx0 + static_cast<int>(kp / g.nky) * g.stride, ky = g.ky0 + static_cast<int>(kp % g.nky) * g.stride;
  float* row = out + (i * nkp + kp) * ldo;
  for (int j = lane; j < g.n_hist; j += 32) {
    const int dx = samp[3 * j], dy = samp[3 * j + 1], l = samp[3 * j + 2];
    const double* v = layers + l * g.layer_stride + i * g.H * npx + (kx + dx) + static_cast<int64_t>(ky + dy) * g.X;
    double s = 0.0;
    for (int a = 0; a < g.H; ++a) s = __dadd_rn(s, __dmul_rn(v[a * npx], v[a * npx]));
    const double n = __dsqrt_rn(s);
    // at or below the threshold divide by +inf instead: the layers are sums of non-negative products, so that stores +0 (one
    // division site keeps the slow path of the fp64 division from spilling)
    const double d = n > 1e-8 ? n : __longlong_as_double(0x7ff0000000000000LL);
    float* dst = row + j * g.H;
    for (int a = 0; a < g.H; ++a, v += npx) dst[a] = __double2float_rn(__ddiv_rn(*v, d));
  }
}

// ------------------------------------------------------------------------------------------------------------------ host side
static std::unique_ptr<Matrix> zeroed_output(Ctx& c, int64_t rows, int64_t cols) {
  auto out = new_matrix(rows, cols);
  if (out->ld != cols && rows > 0) KS_CUDA(cudaMemsetAsync(out->d, 0, out->buf.bytes, c.st));
  return out;
}

HogShape hog_shape(int x_dim, int y_dim, int channels, int bin) {
  if (x_dim <= 0 || y_dim <= 0) throw KsError{KS_ERR_INVALID, "HogExtractor: image dimensions must be positive"};
  if (channels != 3) throw KsError{KS_ERR_INVALID, "HogExtractor: the images must have 3 channels (BGR)"};
  if (bin < 1 || bin > 1024) throw KsError{KS_ERR_INVALID, "HogExtractor: binSize must lie in [1, 1024]"};
  HogShape s;
  s.nx = static_cast<int>(std::floor(static_cast<double>(x_dim) / bin + 0.5));  // Scala math.round
  s.ny = static_cast<int>(std::floor(static_cast<double>(y_dim) / bin + 0.5));
  const int64_t vx = static_cast<int64_t>(s.nx) * bin, vy = static_cast<int64_t>(s.ny) * bin;
  // the reference reads c + x C + y C xDim unclamped; its largest read, channel 2 at (vx - 2, vy - 1), must stay inside the image
  if (vx >= 3 && vy >= 3 && 2 + (vx - 2) * 3 + (vy - 1) * 3 * static_cast<int64_t>(x_dim) >= 3 * static_cast<int64_t>(x_dim) * y_dim)
    throw KsError{KS_ERR_INVALID, "HogExtractor: binSize makes the pixel loop read past the end of the image"};
  s.rows = static_cast<int64_t>(std::max(s.nx - 2, 0)) * std::max(s.ny - 2, 0);
  return s;
}

std::unique_ptr<Matrix> hog_extract(Ctx& c, Matrix& im, int x_dim, int y_dim, int channels, int pixel_scale, int bin) {
  const HogShape s = hog_shape(x_dim, y_dim, channels, bin);
  if (im.cols != static_cast<int64_t>(x_dim) * y_dim * channels)
    throw KsError{KS_ERR_INVALID, "HogExtractor: image size does not match the matrix"};
  if (pixel_scale != 0 && pixel_scale != 1) throw KsError{KS_ERR_INVALID, "HogExtractor: pixel_scale must be 0 or 1"};
  check_finite(c, im, im.cols, "HogExtractor");
  auto out = zeroed_output(c, im.rows * s.rows, kHogFeatures);
  if (s.rows == 0 || im.rows == 0) return out;
  HogGeom g;
  g.x_dim = x_dim;
  g.nx = s.nx;
  g.ny = s.ny;
  g.vx = s.nx * bin;
  g.vy = s.ny * bin;
  g.bin = bin;
  g.scale = pixel_scale;
  const int64_t plane = static_cast<int64_t>(g.vx) * g.vy, cells = static_cast<int64_t>(g.nx) * g.ny;
  const int64_t per_img = plane * (sizeof(double) + 1) + cells * (kHogOri + 1) * sizeof(float);
  const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>({im.rows, kScratchBytes / per_img, 65535}));
  DevBuf scratch;
  scratch.alloc(static_cast<size_t>(chunk * per_img));
  double* mag = scratch.as<double>();
  float* hist = reinterpret_cast<float*>(mag + chunk * plane);
  float* norm = hist + chunk * kHogOri * cells;
  unsigned char* ori = reinterpret_cast<unsigned char*>(norm + chunk * cells);
  for (int64_t i0 = 0; i0 < im.rows; i0 += chunk) {
    const unsigned ni = static_cast<unsigned>(std::min(chunk, im.rows - i0));
    hog_gradient_kernel<<<dim3(grid_for((g.vx - 2) * static_cast<int64_t>(g.vy - 2), 256, c), ni), 256, 0, c.st>>>(im.d + i0 * im.ld, im.ld,
                                                                                                                   g, mag, ori);
    hog_hist_kernel<<<dim3(static_cast<unsigned>((cells + kCellWarps - 1) / kCellWarps), ni), 32 * kCellWarps, 0, c.st>>>(mag, ori, g, hist);
    hog_norm_kernel<<<dim3(grid_for(cells, 256, c), ni), 256, 0, c.st>>>(hist, cells, norm);
    hog_feature_kernel<<<dim3(grid_for(s.rows, 128, c), ni), 128, 0, c.st>>>(hist, norm, g, out->d + i0 * s.rows * out->ld, out->ld);
    c.launches += 4;
  }
  c.check_async("HogExtractor.apply");
  return out;
}

DaisyShape daisy_shape(int x_dim, int y_dim, int T, int Q, int R, int H, int border, int stride) {
  if (x_dim <= 0 || y_dim <= 0) throw KsError{KS_ERR_INVALID, "DaisyExtractor: image dimensions must be positive"};
  if (T < 1 || Q < 1 || R < 1 || H < 1 || stride < 1 || border < 0)
    throw KsError{KS_ERR_INVALID, "DaisyExtractor: daisyT, daisyQ, daisyR, daisyH and stride must be >= 1, pixelBorder >= 0"};
  if (T > 64 || Q > 16 || H > 64 || R > 4096 || stride > (1 << 16) || border > (1 << 16))
    throw KsError{KS_ERR_INVALID, "DaisyExtractor: daisyT, daisyH <= 64, daisyQ <= 16, daisyR <= 4096, stride and pixelBorder <= 65536"};
  DaisyShape s;
  // sigma_n^2 = (R n / 2Q)^2; layer q blurs by the difference D_q with radius ceil(sqrt(-2 D ln 1e-6 - D ln 2 pi D))
  std::vector<double> sq;
  for (int n = 0; n <= Q; ++n) {
    const double v = static_cast<double>(R) * n / (2 * Q);
    sq.push_back(v * v);
  }
  for (int q = 0; q < Q; ++q) {
    const double d = sq[static_cast<size_t>(q) + 1] - sq[static_cast<size_t>(q)];
    const double r = std::ceil(std::sqrt(-2 * d * std::log(1e-6) - d * std::log(2 * M_PI * d)));
    if (!(r <= 1024)) throw KsError{KS_ERR_INVALID, "DaisyExtractor: a blur radius exceeds 1024 (daisyR / daisyQ too large)"};
    const int t = static_cast<int>(r);
    std::vector<double> taps;
    for (int n = -t; n <= t; ++n) taps.push_back(std::exp(-(static_cast<double>(n) * n / (2 * d))) / std::sqrt(2 * M_PI * d));
    s.taps.push_back(taps);
  }
  s.nkx = x_dim - border - 1 >= border ? (x_dim - border - 1 - border) / stride + 1 : 0;
  s.nky = y_dim - border - 1 >= border ? (y_dim - border - 1 - border) / stride + 1 : 0;
  // ring sample (l, t): (round(r_l sin theta), round(r_l cos theta)), r_l = R (1 + l) / Q, theta = 2 pi (t - 1) / T, stored in
  // histogram order j = 1 + t Q + l after the centre (0, 0, layer 0)
  s.samples.assign(static_cast<size_t>(3 * (1 + T * Q)), 0);
  for (int t = 0; t < T; ++t)
    for (int l = 0; l < Q; ++l) {
      const double rad = R * (1 + static_cast<double>(l)) / Q, th = 2 * M_PI * (t - 1) / T;
      const int dx = static_cast<int>(std::floor(rad * std::sin(th) + 0.5)), dy = static_cast<int>(std::floor(rad * std::cos(th) + 0.5));
      const size_t j = static_cast<size_t>(1 + t * Q + l);
      s.samples[3 * j] = dx;
      s.samples[3 * j + 1] = dy;
      s.samples[3 * j + 2] = l;
      if (s.nkx > 0 && s.nky > 0 &&
          (border + dx < 0 || border + (s.nkx - 1) * static_cast<int64_t>(stride) + dx > x_dim - 1 || border + dy < 0 ||
           border + (s.nky - 1) * static_cast<int64_t>(stride) + dy > y_dim - 1))
        throw KsError{KS_ERR_INVALID, "DaisyExtractor: a ring sample of a keypoint leaves the image (raise pixelBorder or lower daisyR)"};
    }
  s.features = H * (T * Q + 1);
  return s;
}

std::unique_ptr<Matrix> daisy_extract(Ctx& c, Matrix& im, int x_dim, int y_dim, int T, int Q, int R, int H, int border, int stride) {
  const DaisyShape s = daisy_shape(x_dim, y_dim, T, Q, R, H, border, stride);
  const int X = x_dim, Y = y_dim;
  const int64_t npx = static_cast<int64_t>(X) * Y;
  if (im.cols != npx) throw KsError{KS_ERR_INVALID, "DaisyExtractor: the images must have one channel of x_dim * y_dim pixels"};
  check_finite(c, im, im.cols, "DaisyExtractor");
  const int64_t nkp = static_cast<int64_t>(s.nkx) * s.nky;
  auto out = zeroed_output(c, im.rows * nkp, s.features);
  if (nkp == 0 || im.rows == 0) return out;
  // filters: the gradient passes (x: [1 0 -1], [1 2 1]; y: [1 2 1], [1 0 -1]), then the Q blurs; the orientation cos / sin pairs
  std::vector<double> f = {1.0, 0.0, -1.0, 1.0, 2.0, 1.0, 1.0, 2.0, 1.0, 1.0, 0.0, -1.0};
  std::vector<size_t> tap0;
  for (const auto& t : s.taps) {
    tap0.push_back(f.size());
    f.insert(f.end(), t.begin(), t.end());
  }
  const size_t cs0 = f.size();
  for (int a = 0; a < H; ++a) {
    const double ang = 2 * M_PI * a / H;
    f.push_back(std::cos(ang));
    f.push_back(std::sin(ang));
  }
  DevBuf dconst;
  dconst.alloc(sizeof(double) * f.size() + sizeof(int) * s.samples.size());
  int* dsamp = reinterpret_cast<int*>(dconst.as<double>() + f.size());
  KS_CUDA(cudaMemcpyAsync(dconst.p, f.data(), sizeof(double) * f.size(), cudaMemcpyHostToDevice, c.st));
  KS_CUDA(cudaMemcpyAsync(dsamp, s.samples.data(), sizeof(int) * s.samples.size(), cudaMemcpyHostToDevice, c.st));
  const double* df = dconst.as<double>();
  // scratch per image: ix and iy, the pass-along-x buffer (max(2, H) planes) and the Q H layers
  const int64_t mid_planes = std::max(2, H), per_img = (2 + mid_planes + static_cast<int64_t>(Q) * H) * npx;
  const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>({im.rows, kScratchBytes / (8 * per_img), 65535 / mid_planes}));
  DevBuf scratch;
  scratch.alloc(sizeof(double) * static_cast<size_t>(chunk * per_img));
  double* G = scratch.as<double>();
  double* M = G + chunk * 2 * npx;
  double* L = M + chunk * mid_planes * npx;
  DaisyGeom g;
  g.X = X;
  g.Y = Y;
  g.H = H;
  g.Q = Q;
  g.n_hist = 1 + T * Q;
  g.kx0 = border;
  g.ky0 = border;
  g.nkx = s.nkx;
  g.nky = s.nky;
  g.stride = stride;
  g.layer_stride = chunk * H * npx;
  const unsigned gpx = grid_for(npx, 256, c);
  for (int64_t i0 = 0; i0 < im.rows; i0 += chunk) {
    const unsigned ni = static_cast<unsigned>(std::min(chunk, im.rows - i0));
    // ix = conv2D(gray, [1 0 -1], [1 2 1]), iy = conv2D(gray, [1 2 1], [1 0 -1]): planes 2i, 2i + 1
    conv_pass_kernel<float><<<dim3(gpx, 2 * ni), 256, 0, c.st>>>(im.d + i0 * im.ld, im.ld, 2, M, X, Y, df, 3, 2, 1);
    conv_pass_kernel<double><<<dim3(gpx, 2 * ni), 256, 0, c.st>>>(M, npx, 1, G, X, Y, df + 6, 3, 2, 0);
    for (int l = 0; l < Q; ++l) {
      const int len = static_cast<int>(s.taps[static_cast<size_t>(l)].size());
      const double* fl = df + tap0[static_cast<size_t>(l)];
      if (l == 0)
        orient_conv_x_kernel<<<dim3(gpx, ni * H), 256, 0, c.st>>>(G, H, df + cs0, M, X, Y, fl, len);
      else
        conv_pass_kernel<double><<<dim3(gpx, ni * H), 256, 0, c.st>>>(L + (l - 1) * g.layer_stride, npx, 1, M, X, Y, fl, len, 1, 1);
      conv_pass_kernel<double><<<dim3(gpx, ni * H), 256, 0, c.st>>>(M, npx, 1, L + l * g.layer_stride, X, Y, fl, len, 1, 0);
      c.launches += 2;
    }
    daisy_descriptor_kernel<<<dim3(static_cast<unsigned>((nkp + kKpWarps - 1) / kKpWarps), ni), 32 * kKpWarps, 0, c.st>>>(
        L, g, dsamp, out->d + i0 * nkp * out->ld, out->ld);
    c.launches += 3;
  }
  c.check_async("DaisyExtractor.apply");
  return out;
}

}  // namespace ks
