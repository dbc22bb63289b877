// Covariance-based transforms on the device: PCAEstimator / DistributedPCAEstimator, ZCAWhitenerEstimator and
// ApproximatePCAEstimator (K/nodes/learning/{PCA,DistributedPCA,ZCAWhitener,ApproximatePCA}.scala).  DESIGN.md section 15.
//
// Every product here runs in fp64 on the DMMA tensor core (mma.sync.m8n8k4.f64): the fits take no precision mode.
//   Gram     out = (A - 1 s^T)^T (B - 1 t^T), row-sharded A (N x m) and B (N x n), fp32 or fp64, the shifts applied in fp64 as the
//            operand is loaded; symmetric mode (B = A: upper tiles only, mirrored) or cross mode; split-K over rows with the
//            partial tiles summed in split order (no atomics), so one rank's result repeats bit for bit.
//   Skinny   Y = A B for a row-major A (N x d, fp32 or fp64) and a small fp64 B (d x l): one streaming pass over A (the column
//            tiles of one row panel are neighbouring CTAs, so A's second read of a panel hits L2).
// The eigen / singular-value problems and L^-1 run in cuSOLVER (fp64) and rank 0's results are broadcast, so models and Q factors
// are bit-identical across ranks.
#include "engine.h"

#include <math.h>

#include <algorithm>
#include <chrono>
#include <sstream>

namespace ks {

static constexpr int kPT = 64;           // output tile of both kernels (rows x columns)
static constexpr int kPK = 32;           // contraction depth per shared-memory stage
static constexpr int kPLd = kPT + 4;     // shared row stride in doubles: == 4 (mod 16), conflict-free fragment loads
static constexpr int kPThreads = 128;    // 4 warps, 32 x 32 outputs each
static constexpr int kPLoads = kPK * kPT / kPThreads;  // elements per thread per panel and stage

__device__ __forceinline__ void dmma_m8n8k4(double (&d)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(d[0]), "+d"(d[1])
               : "d"(a), "d"(b));
}

// acc += sum_k sA[k][m] sB[k][n] over one stage, for the warp's 32 x 32 sub-tile (wm, wn).  Fragments of m8n8k4.f64: A (8x4, row)
// lane -> (m = lane / 4, k = lane % 4); B (4x8, col) lane -> (k = lane % 4, n = lane / 4); C lane -> (m = lane / 4, n = 2 (lane % 4) + i).
__device__ __forceinline__ void dmma_stage(const double* sA, const double* sB, int wm, int wn, int lane, double (&acc)[4][4][2]) {
  const int kk = lane & 3, q = lane >> 2;
#pragma unroll
  for (int k = 0; k < kPK; k += 4) {
    double a[4], b[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = sA[(k + kk) * kPLd + wm * 32 + i * 8 + q];
#pragma unroll
    for (int j = 0; j < 4; ++j) b[j] = sB[(k + kk) * kPLd + wn * 32 + j * 8 + q];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) dmma_m8n8k4(acc[i][j], a[i], b[j]);
  }
}

// rows [r, r + kPK) x columns [c0, c0 + kPT) of a row-major operand, minus the column shift, as fp64 (zero outside the matrix)
template <class T>
__device__ __forceinline__ void load_row_panel(const T* __restrict__ A, int64_t lda, const double* __restrict__ shift, int cols, int c0,
                                               int64_t r, int64_t r_end, double (&v)[kPLoads]) {
  const int col = threadIdx.x & (kPT - 1), c = c0 + col;
  const double s = (shift && c < cols) ? shift[c] : 0.0;
#pragma unroll
  for (int u = 0; u < kPLoads; ++u) {
    const int64_t row = r + (threadIdx.x >> 6) + 2 * u;
    v[u] = (row < r_end && c < cols) ? static_cast<double>(A[row * lda + c]) - s : 0.0;
  }
}
__device__ __forceinline__ void store_row_panel(double* s, const double (&v)[kPLoads]) {
  const int col = threadIdx.x & (kPT - 1);
#pragma unroll
  for (int u = 0; u < kPLoads; ++u) s[((threadIdx.x >> 6) + 2 * u) * kPLd + col] = v[u];
}

// tile t of the upper triangle (bi <= bj) of an nt x nt tile grid, row by row
__device__ __forceinline__ void upper_tile(int64_t t, int nt, int* bi, int* bj) {
  int i = 0;
  while (t >= nt - i) {
    t -= nt - i;
    ++i;
  }
  *bi = i;
  *bj = i + static_cast<int>(t);
}

// One output tile over rows [blockIdx.y * rps, ...).  One split: written to out (symmetric mode: the element with row <= column and
// its mirror); several: to part[split][tile][64 x 64], summed by gram_reduce_kernel.
template <class TA, class TB>
__global__ void __launch_bounds__(kPThreads) gram_f64_kernel(const TA* __restrict__ A, int64_t lda, const double* __restrict__ sa, int m,
                                                             const TB* __restrict__ B, int64_t ldb, const double* __restrict__ sb, int n,
                                                             int64_t rows, int64_t rps, int sym, double* __restrict__ out, int64_t ldo,
                                                             double* __restrict__ part) {
  __shared__ double sA[kPK * kPLd], sB[kPK * kPLd];
  int bi, bj;
  if (sym) {
    upper_tile(blockIdx.x, (m + kPT - 1) / kPT, &bi, &bj);
  } else {
    const int ntn = (n + kPT - 1) / kPT;
    bi = blockIdx.x / ntn;
    bj = blockIdx.x % ntn;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wm = warp >> 1, wn = warp & 1;
  const int64_t r0 = blockIdx.y * rps, r1 = min(rows, r0 + rps);
  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
  double pa[kPLoads], pb[kPLoads];
  load_row_panel(A, lda, sa, m, bi * kPT, r0, r1, pa);
  load_row_panel(B, ldb, sb, n, bj * kPT, r0, r1, pb);
  for (int64_t r = r0; r < r1; r += kPK) {
    store_row_panel(sA, pa);
    store_row_panel(sB, pb);
    __syncthreads();
    if (r + kPK < r1) {  // the next stage's loads are in flight during this stage's MMAs
      load_row_panel(A, lda, sa, m, bi * kPT, r + kPK, r1, pa);
      load_row_panel(B, ldb, sb, n, bj * kPT, r + kPK, r1, pb);
    }
    dmma_stage(sA, sB, wm, wn, lane, acc);
    __syncthreads();
  }
  const bool direct = gridDim.y == 1;
  double* tile = part + (static_cast<int64_t>(blockIdx.y) * gridDim.x + blockIdx.x) * (kPT * kPT);
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int lm = wm * 32 + i * 8 + (lane >> 2), ln = wn * 32 + j * 8 + (lane & 3) * 2 + e;
        if (!direct) {
          tile[lm * kPT + ln] = acc[i][j][e];
          continue;
        }
        const int gi = bi * kPT + lm, gj = bj * kPT + ln;
        if (gi >= m || gj >= n) continue;
        if (sym) {
          if (gi > gj) continue;
          out[static_cast<int64_t>(gj) * ldo + gi] = acc[i][j][e];
        }
        out[static_cast<int64_t>(gi) * ldo + gj] = acc[i][j][e];
      }
}

// out element of tile t = sum over the splits of part[split][t], in split order
__global__ void gram_reduce_kernel(const double* __restrict__ part, int64_t tiles, int splits, int m, int n, int sym,
                                   double* __restrict__ out, int64_t ldo) {
  const int64_t total = tiles * kPT * kPT;
  const int ntn = (n + kPT - 1) / kPT, ntm = (m + kPT - 1) / kPT;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t t = i / (kPT * kPT);
    const int e = static_cast<int>(i - t * kPT * kPT);
    int bi, bj;
    if (sym) {
      upper_tile(t, ntm, &bi, &bj);
    } else {
      bi = static_cast<int>(t / ntn);
      bj = static_cast<int>(t % ntn);
    }
    const int gi = bi * kPT + e / kPT, gj = bj * kPT + e % kPT;
    if (gi >= m || gj >= n || (sym && gi > gj)) continue;
    double s = 0.0;
    for (int y = 0; y < splits; ++y) s += part[(static_cast<int64_t>(y) * tiles + t) * (kPT * kPT) + e];
    out[static_cast<int64_t>(gi) * ldo + gj] = s;
    if (sym) out[static_cast<int64_t>(gj) * ldo + gi] = s;
  }
}

// Y[rows x l] = A[rows x d] B[d x l]; CTA = 64 rows x 64 columns, blockIdx.x = row tile * column tiles + column tile
template <class TA>
__global__ void __launch_bounds__(kPThreads) skinny_f64_kernel(const TA* __restrict__ A, int64_t lda, int64_t rows, int d,
                                                               const double* __restrict__ B, int64_t ldb, int l, double* __restrict__ Y,
                                                               int64_t ldy) {
  __shared__ double sA[kPK * kPLd], sB[kPK * kPLd];
  const int nct = (l + kPT - 1) / kPT;
  const int64_t row0 = static_cast<int64_t>(blockIdx.x / nct) * kPT;
  const int col0 = (blockIdx.x % nct) * kPT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wm = warp >> 1, wn = warp & 1;
  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
  // A stage: 64 rows x 32 k, a warp reads 32 consecutive k of one row; stored transposed, sA[k][row]
  const int ak = threadIdx.x & (kPK - 1), arow = threadIdx.x >> 5;
  double pa[kPLoads], pb[kPLoads];
  auto load_a = [&](int k0) {
#pragma unroll
    for (int u = 0; u < kPLoads; ++u) {
      const int64_t r = row0 + arow + 4 * u;
      pa[u] = (r < rows && k0 + ak < d) ? static_cast<double>(A[r * lda + k0 + ak]) : 0.0;
    }
  };
  auto load_b = [&](int k0) {
    const int col = threadIdx.x & (kPT - 1);
#pragma unroll
    for (int u = 0; u < kPLoads; ++u) {
      const int k = k0 + (threadIdx.x >> 6) + 2 * u;
      pb[u] = (k < d && col0 + col < l) ? B[static_cast<int64_t>(k) * ldb + col0 + col] : 0.0;
    }
  };
  load_a(0);
  load_b(0);
  for (int k0 = 0; k0 < d; k0 += kPK) {
#pragma unroll
    for (int u = 0; u < kPLoads; ++u) sA[ak * kPLd + arow + 4 * u] = pa[u];
    store_row_panel(sB, pb);
    __syncthreads();
    if (k0 + kPK < d) {
      load_a(k0 + kPK);
      load_b(k0 + kPK);
    }
    dmma_stage(sA, sB, wm, wn, lane, acc);
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int64_t r = row0 + wm * 32 + i * 8 + (lane >> 2);
        const int cc = col0 + wn * 32 + j * 8 + (lane & 3) * 2 + e;
        if (r < rows && cc < l) Y[r * ldy + cc] = acc[i][j][e];
      }
}

// ------------------------------------------------------------------------------------ small fp64 helpers
// out[:, c] (d x ncols, column-major) = sign_c V[:, src_c] with src_c = d - 1 - c (reverse: eigenpairs ascending -> descending) or c;
// sign_c = +1 iff max(col) == max |col| (PCAEstimator.enforceMatlabPCASignConvention, PCA.scala:238-247: ties keep +)
__global__ void order_sign_kernel(const double* __restrict__ V, int64_t ldv, int d, int reverse, double* __restrict__ out) {
  __shared__ double smax[256], sabs[256];
  const int c = blockIdx.x, src = reverse ? d - 1 - c : c;
  const double* col = V + static_cast<int64_t>(src) * ldv;
  double mx = -INFINITY, ma = 0.0;
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    mx = fmax(mx, col[i]);
    ma = fmax(ma, fabs(col[i]));
  }
  smax[threadIdx.x] = mx;
  sabs[threadIdx.x] = ma;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      smax[threadIdx.x] = fmax(smax[threadIdx.x], smax[threadIdx.x + s]);
      sabs[threadIdx.x] = fmax(sabs[threadIdx.x], sabs[threadIdx.x + s]);
    }
    __syncthreads();
  }
  const double sg = smax[0] == sabs[0] ? 1.0 : -1.0;
  for (int i = threadIdx.x; i < d; i += blockDim.x) out[static_cast<int64_t>(c) * d + i] = sg * col[i];
}

// ZCA: M (d x d row-major) = diag(sqrt(w)) V^T with w_i = (max(lambda_i, 0) / (N - 1) + eps)^-1/2, so that M^T M = V diag(w) V^T.
// V column-major: row i of M is column i of V, scaled.
__global__ void zca_scale_kernel(const double* __restrict__ V, const double* __restrict__ lam, int d, double inv_nm1, double eps,
                                 double* __restrict__ M) {
  const int64_t total = static_cast<int64_t>(d) * d;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int e = static_cast<int>(i / d);
    const double w = 1.0 / sqrt(fmax(lam[e], 0.0) * inv_nm1 + eps);
    M[i] = sqrt(w) * V[i];
  }
}

__global__ void mean_from_sums_kernel(const double* __restrict__ sums, double inv_n, double* __restrict__ mean, int d) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < d) mean[i] = sums[i] * inv_n;
}

// H = G (+ c trace(G) I when c > 0): the shift of shifted CholeskyQR, sigma = 11 (N l + l (l + 1)) u |Y|_2^2 with |Y|_2^2 <= trace(G)
__global__ void shifted_copy_kernel(const double* __restrict__ G, double* __restrict__ H, int l, double c) {
  __shared__ double tr;
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < l; ++i) t += G[static_cast<int64_t>(i) * l + i];
    tr = t;
  }
  __syncthreads();
  const int64_t total = static_cast<int64_t>(l) * l;
  for (int64_t i = threadIdx.x; i < total; i += blockDim.x) {
    const int64_t r = i / l;
    H[i] = G[i] + ((c > 0.0 && r * l + r == i) ? c * tr : 0.0);
  }
}

// column-major L^-1 (lower) -> zero its strict upper part; the buffer is then L^-T row-major.  flag <- info (fp64, broadcast with it)
__global__ void lower_only_kernel(double* __restrict__ L, int l, const int* __restrict__ info, double* __restrict__ flag) {
  const int64_t total = static_cast<int64_t>(l) * l;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t col = i / l, row = i - col * l;
    if (row < col) L[i] = 0.0;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *flag = static_cast<double>(*info);
}
__global__ void info_to_flag_kernel(const int* __restrict__ info, double* __restrict__ flag) { *flag = static_cast<double>(*info); }

// ------------------------------------------------------------------------------------ launchers
template <class TA, class TB>
static void gram_launch(dim3 grid, const TA* A, const GramOperand& a, const TB* B, const GramOperand& b, int64_t rows, int64_t rps, int sym,
                        double* out, int64_t ldo, double* part, cudaStream_t st) {
  gram_f64_kernel<TA, TB><<<grid, kPThreads, 0, st>>>(A, a.ld, a.shift, a.cols, B, b.ld, b.shift, b.cols, rows, rps, sym, out, ldo, part);
}
void gram_f64(Ctx& c, const GramOperand& a, const GramOperand* b, int64_t rows, double* out, int64_t ldo, double* flops) {
  const bool sym = b == nullptr;
  const GramOperand& bb = sym ? a : *b;
  const int m = a.cols, n = bb.cols;
  const int ntm = (m + kPT - 1) / kPT, ntn = (n + kPT - 1) / kPT;
  const int64_t tiles = sym ? static_cast<int64_t>(ntm) * (ntm + 1) / 2 : static_cast<int64_t>(ntm) * ntn;
  if (m == 0 || n == 0) return;
  if (rows == 0) {  // a rank without rows contributes zeros to the all-reduce
    KS_CUDA(cudaMemset2DAsync(out, sizeof(double) * ldo, 0, sizeof(double) * n, m, c.st));
    return;
  }
  // split-K: about four CTAs per SM, at least 256 rows per split, at most 256 MB of partial tiles
  const int64_t want = (4LL * c.num_sms + tiles - 1) / tiles;
  const int64_t max_rows = (rows + 255) / 256;
  const int64_t max_mem = std::max<int64_t>(1, (int64_t(256) << 20) / (tiles * kPT * kPT * 8));
  int64_t splits = std::max<int64_t>(1, std::min({want, max_rows, max_mem, int64_t(65535)}));
  const int64_t rps = round_up((rows + splits - 1) / splits, kPK);
  splits = (rows + rps - 1) / rps;
  DevBuf part;
  if (splits > 1) part.alloc(sizeof(double) * static_cast<size_t>(splits * tiles) * kPT * kPT);
  const dim3 grid(static_cast<unsigned>(tiles), static_cast<unsigned>(splits));
  if (a.f32 && bb.f32) gram_launch(grid, a.f32, a, bb.f32, bb, rows, rps, sym, out, ldo, part.as<double>(), c.st);
  else if (a.f32) gram_launch(grid, a.f32, a, bb.f64, bb, rows, rps, sym, out, ldo, part.as<double>(), c.st);
  else if (bb.f32) gram_launch(grid, a.f64, a, bb.f32, bb, rows, rps, sym, out, ldo, part.as<double>(), c.st);
  else gram_launch(grid, a.f64, a, bb.f64, bb, rows, rps, sym, out, ldo, part.as<double>(), c.st);
  c.launches += 1;
  if (splits > 1) {
    const int64_t total = tiles * kPT * kPT;
    const unsigned g = static_cast<unsigned>(std::min<int64_t>((total + 255) / 256, 4 * c.num_sms));
    gram_reduce_kernel<<<g, 256, 0, c.st>>>(part.as<double>(), tiles, static_cast<int>(splits), m, n, sym ? 1 : 0, out, ldo);
    c.launches += 1;
  }
  if (flops) *flops += 2.0 * static_cast<double>(rows) * m * n * (sym ? 0.5 : 1.0);
}
void skinny_f64(Ctx& c, const GramOperand& a, int64_t rows, const double* B, int64_t ldb, int l, double* Y, int64_t ldy) {
  if (rows == 0 || l == 0) return;
  const int64_t nct = (l + kPT - 1) / kPT, nrt = (rows + kPT - 1) / kPT;
  if (nct * nrt > 0x7fffffffLL) throw KsError{KS_ERR_INVALID, "too many rows for the skinny product"};
  const unsigned g = static_cast<unsigned>(nct * nrt);
  if (a.f32) skinny_f64_kernel<float><<<g, kPThreads, 0, c.st>>>(a.f32, a.ld, rows, a.cols, B, ldb, l, Y, ldy);
  else skinny_f64_kernel<double><<<g, kPThreads, 0, c.st>>>(a.f64, a.ld, rows, a.cols, B, ldb, l, Y, ldy);
  c.launches += 1;
}

static void bcast_f64(Ctx& c, double* p, size_t n) {
  if (c.world <= 1 || n == 0) return;
  KS_NCCL(nccl_api().Broadcast(p, p, n, ncclFloat64, 0, c.comm, c.st));
}
static cusolverDnHandle_t solver_on_st(Ctx& c) {
  c.ensure_solver();
  if (c.solver_stream != c.st) {
    if (solver_api().SetStream(c.solver, c.st) != CUSOLVER_STATUS_SUCCESS) throw KsError{KS_ERR_SOLVER, "cusolverDnSetStream failed"};
    c.solver_stream = c.st;
  }
  return c.solver;
}

// per-phase device time of a fit: mean, gram, allreduce, eig (eigen / singular values), qr (CholeskyQR), other
struct PcaTimer {
  enum { MEAN = 0, GRAM, ALLREDUCE, EIG, QR, SKINNY, OTHER, COUNT };
  Ctx& c;
  std::vector<std::pair<int, std::pair<cudaEvent_t, cudaEvent_t>>> spans;
  explicit PcaTimer(Ctx& cc) : c(cc) {}
  void begin(int ph) {
    spans.push_back({ph, {c.get_event(), c.get_event()}});
    KS_CUDA(cudaEventRecord(spans.back().second.first, c.st));
  }
  void end() { KS_CUDA(cudaEventRecord(spans.back().second.second, c.st)); }
  void collect(double ms[COUNT]) {
    for (int i = 0; i < COUNT; ++i) ms[i] = 0.0;
    for (auto& s : spans) {
      float t = 0.f;
      cudaEventSynchronize(s.second.second);
      cudaEventElapsedTime(&t, s.second.first, s.second.second);
      ms[s.first] += t;
      c.event_pool.push_back(s.second.first);
      c.event_pool.push_back(s.second.second);
    }
    spans.clear();
  }
  ~PcaTimer() {
    for (auto& s : spans) {
      c.event_pool.push_back(s.second.first);
      c.event_pool.push_back(s.second.second);
    }
  }
};

static GramOperand operand_of(const Matrix& X, const double* shift = nullptr) {
  GramOperand o;
  o.f32 = X.d;
  o.ld = X.ld;
  o.cols = static_cast<int>(X.cols);
  o.shift = shift;
  return o;
}
static GramOperand operand_of(const double* p, int64_t ld, int cols) {
  GramOperand o;
  o.f64 = p;
  o.ld = ld;
  o.cols = cols;
  return o;
}

static double global_rows(Ctx& c, int64_t n_loc) {
  DevBuf t;
  t.alloc(sizeof(double));
  launch_set_f64(t.as<double>(), static_cast<double>(n_loc), c.st);
  c.launches += 1;
  c.allreduce_f64(t.as<double>(), 1);
  double n = 0;
  KS_CUDA(cudaMemcpyAsync(&n, t.p, sizeof(double), cudaMemcpyDeviceToHost, c.st));
  KS_CUDA(cudaStreamSynchronize(c.st));
  return n;
}

// exact fp64 column means of the row-sharded X (column sums, all-reduce, / N)
static void column_means(Ctx& c, Matrix& X, double n_total, DevBuf& mean, PcaTimer& tm) {
  const int d = static_cast<int>(X.cols);
  DevBuf sums;
  sums.alloc(sizeof(double) * d);
  mean.alloc(sizeof(double) * d);
  tm.begin(PcaTimer::MEAN);
  KS_CUDA(cudaMemsetAsync(sums.p, 0, sums.bytes, c.st));
  launch_colsum(X.d, nullptr, X.ld, X.rows, d, sums.as<double>(), c.st);
  c.launches += 1;
  tm.end();
  tm.begin(PcaTimer::ALLREDUCE);
  c.allreduce_f64(sums.as<double>(), d);
  tm.end();
  tm.begin(PcaTimer::MEAN);
  mean_from_sums_kernel<<<(d + 255) / 256, 256, 0, c.st>>>(sums.as<double>(), 1.0 / n_total, mean.as<double>(), d);
  c.launches += 1;
  tm.end();
}

// G = X_c^T X_c (d x d, fp64) over all ranks
static void centred_covariance(Ctx& c, Matrix& X, const double* mean, DevBuf& G, PcaTimer& tm, double* flops) {
  const int64_t d = X.cols;
  G.alloc(sizeof(double) * static_cast<size_t>(d * d));
  tm.begin(PcaTimer::GRAM);
  gram_f64(c, operand_of(X, mean), nullptr, X.rows, G.as<double>(), d, flops);
  tm.end();
  tm.begin(PcaTimer::ALLREDUCE);
  c.allreduce_f64(G.as<double>(), static_cast<size_t>(d * d));
  tm.end();
}

// Eigenpairs of the symmetric G (d x d): V (column-major, ascending eigenvalues) and lam, rank 0's broadcast
static void symmetric_eigen(Ctx& c, const DevBuf& G, int d, DevBuf& V, DevBuf& lam, PcaTimer& tm) {
  SolverApi& api = solver_api();
  cusolverDnHandle_t h = solver_on_st(c);
  const size_t dd = static_cast<size_t>(d) * d;
  V.alloc(sizeof(double) * (dd + d + 1));  // [V | lambda | info]
  DevBuf info;
  info.alloc(sizeof(int));
  tm.begin(PcaTimer::EIG);
  KS_CUDA(cudaMemcpyAsync(V.p, G.p, sizeof(double) * dd, cudaMemcpyDeviceToDevice, c.st));
  double* W = V.as<double>() + dd;
  int lwork = 0;
  if (api.DsyevdBufferSize(h, CUSOLVER_EIG_MODE_VECTOR, CUBLAS_FILL_MODE_LOWER, d, V.as<double>(), d, W, &lwork) != CUSOLVER_STATUS_SUCCESS)
    throw KsError{KS_ERR_SOLVER, "cusolverDnDsyevd_bufferSize failed"};
  DevBuf work;
  work.alloc(sizeof(double) * static_cast<size_t>(std::max(lwork, 1)));
  if (api.Dsyevd(h, CUSOLVER_EIG_MODE_VECTOR, CUBLAS_FILL_MODE_LOWER, d, V.as<double>(), d, W, work.as<double>(), lwork, info.as<int>()) !=
      CUSOLVER_STATUS_SUCCESS)
    throw KsError{KS_ERR_SOLVER, "cusolverDnDsyevd failed"};
  info_to_flag_kernel<<<1, 1, 0, c.st>>>(info.as<int>(), W + d);
  c.launches += 2;
  bcast_f64(c, V.as<double>(), dd + d + 1);
  tm.end();
  double flag = 0;
  KS_CUDA(cudaMemcpyAsync(&flag, W + d, sizeof(double), cudaMemcpyDeviceToHost, c.st));
  KS_CUDA(cudaStreamSynchronize(c.st));
  if (flag != 0) throw KsError{KS_ERR_SOLVER, "cusolverDnDsyevd did not converge (info " + std::to_string(static_cast<int64_t>(flag)) + ")"};
  lam.alloc(sizeof(double) * d);
  KS_CUDA(cudaMemcpyAsync(lam.p, W, sizeof(double) * d, cudaMemcpyDeviceToDevice, c.st));
}

// LinearMapper(P (d x k, column-major), None, mean): stored in feature blocks of up to 4096 rows like every fitted LinearMapper
static int64_t linear_model(Ctx& c, const double* P, int64_t d, int64_t k, const double* mean_or_null) {
  auto model = std::make_unique<Model>();
  const int bs = static_cast<int>(std::min<int64_t>(d, 4096));
  model->block_size = bs;
  model->k = k;
  model->has_mean = mean_or_null != nullptr;
  model->has_intercept = false;
  model->intercept.alloc(sizeof(double) * k);
  KS_CUDA(cudaMemsetAsync(model->intercept.p, 0, model->intercept.bytes, c.st));
  for (int64_t c0 = 0; c0 < d; c0 += bs) {
    const int64_t b = std::min<int64_t>(bs, d - c0);
    model->brows.push_back(b);
    auto Wj = std::make_unique<DevBuf>();
    Wj->alloc(sizeof(double) * static_cast<size_t>(b * k));
    KS_CUDA(cudaMemcpy2DAsync(Wj->p, sizeof(double) * b, P + c0, sizeof(double) * d, sizeof(double) * b, k, cudaMemcpyDeviceToDevice, c.st));
    model->W.push_back(std::move(Wj));
    if (mean_or_null) {
      auto mj = std::make_unique<DevBuf>();
      mj->alloc(sizeof(double) * b);
      KS_CUDA(cudaMemcpyAsync(mj->p, mean_or_null + c0, sizeof(double) * b, cudaMemcpyDeviceToDevice, c.st));
      model->mean.push_back(std::move(mj));
    }
  }
  if (c.host_mirror) {
    model_alloc_host(*model);
    for (size_t j = 0; j < model->brows.size(); ++j) model_block_to_host(*model, static_cast<int>(j), c.st);
  }
  return c.add(std::move(model));
}

static std::string json_list(const std::vector<double>& v) {
  std::ostringstream s;
  s.precision(17);
  s << "[";
  for (size_t i = 0; i < v.size(); ++i) s << (i ? "," : "") << v[i];
  s << "]";
  return s.str();
}
static void write_stats(Ctx& c, const char* solver, int64_t n_loc, double n_total, int64_t d, int dims, int l, int q, PcaTimer& tm,
                        cudaEvent_t e0, cudaEvent_t e1, double flops, const char* values_key, const std::vector<double>& values,
                        int64_t launches0, const std::chrono::steady_clock::time_point& host_t0, int shifted_passes = 0) {
  double ms[PcaTimer::COUNT];
  tm.collect(ms);
  float total = 0.f;
  cudaEventElapsedTime(&total, e0, e1);
  c.event_pool.push_back(e0);
  c.event_pool.push_back(e1);
  std::ostringstream js;
  js.precision(17);
  js << "{\"solver\":\"" << solver << "\",\"n_local\":" << n_loc << ",\"n_total\":" << static_cast<int64_t>(n_total) << ",\"d\":" << d
     << ",\"dims\":" << dims << ",\"l\":" << l << ",\"q\":" << q << ",\"world\":" << c.world << ",\"total_ms\":" << total
     << ",\"mean_ms\":" << ms[PcaTimer::MEAN] << ",\"gram_ms\":" << ms[PcaTimer::GRAM] << ",\"allreduce_ms\":" << ms[PcaTimer::ALLREDUCE]
     << ",\"eig_ms\":" << ms[PcaTimer::EIG] << ",\"qr_ms\":" << ms[PcaTimer::QR] << ",\"skinny_ms\":" << ms[PcaTimer::SKINNY]
     << ",\"other_ms\":" << ms[PcaTimer::OTHER] << ",\"local_flops\":" << flops << ",\"shifted_qr_passes\":" << shifted_passes
     << ",\"launches\":" << (c.launches - launches0) << ",\"mma\":\"dmma-f64\",\"" << values_key << "\":" << json_list(values)
     << ",\"host_ms\":" << std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count() << "}";
  c.stats_json = js.str();
}

// ------------------------------------------------------------------------------------ PCAEstimator / DistributedPCAEstimator
int64_t fit_pca(Ctx& c, Matrix& X, int dims) {
  const int64_t d = X.cols, n_loc = X.rows;
  if (d <= 0) throw KsError{KS_ERR_INVALID, "empty feature dimension"};
  if (dims < 1 || dims > d) throw KsError{KS_ERR_INVALID, "dims must be in [1, d]"};
  const auto host_t0 = std::chrono::steady_clock::now();
  const int64_t launches0 = c.launches;
  const double n_total = global_rows(c, n_loc);
  if (n_total < 1) throw KsError{KS_ERR_INVALID, "no rows"};
  PcaTimer tm(c);
  cudaEvent_t e0 = c.get_event(), e1 = c.get_event();
  KS_CUDA(cudaEventRecord(e0, c.st));
  double flops = 0;
  DevBuf mean, G, V, lam, P;
  column_means(c, X, n_total, mean, tm);
  centred_covariance(c, X, mean.as<double>(), G, tm, &flops);
  symmetric_eigen(c, G, static_cast<int>(d), V, lam, tm);
  P.alloc(sizeof(double) * static_cast<size_t>(d * dims));
  tm.begin(PcaTimer::OTHER);
  order_sign_kernel<<<dims, 256, 0, c.st>>>(V.as<double>(), d, static_cast<int>(d), 1, P.as<double>());
  c.launches += 1;
  tm.end();
  const int64_t id = linear_model(c, P.as<double>(), d, dims, nullptr);
  KS_CUDA(cudaEventRecord(e1, c.st));
  std::vector<double> ev(d);
  KS_CUDA(cudaMemcpyAsync(ev.data(), lam.p, sizeof(double) * d, cudaMemcpyDeviceToHost, c.st));
  c.check_async("PCAEstimator.fit");
  std::reverse(ev.begin(), ev.end());
  ev.resize(dims);
  write_stats(c, "pca", n_loc, n_total, d, dims, 0, 0, tm, e0, e1, flops, "eigenvalues", ev, launches0, host_t0);
  return id;
}

// ------------------------------------------------------------------------------------ ZCAWhitenerEstimator.fitSingle
int64_t fit_zca(Ctx& c, Matrix& X, double eps) {
  const int64_t d = X.cols, n_loc = X.rows;
  if (d <= 0) throw KsError{KS_ERR_INVALID, "empty feature dimension"};
  if (!(eps >= 0.0) || !std::isfinite(eps)) throw KsError{KS_ERR_INVALID, "eps must be finite and >= 0"};
  const auto host_t0 = std::chrono::steady_clock::now();
  const int64_t launches0 = c.launches;
  const double n_total = global_rows(c, n_loc);
  // ZCAWhitener.scala:50-63: sgesvd gives min(N, d) singular values, and v1.t * diag(...) * v1 needs d of them
  if (n_total < static_cast<double>(d) || n_total < 2) throw KsError{KS_ERR_INVALID, "ZCA whitening needs at least d rows (and 2)"};
  PcaTimer tm(c);
  cudaEvent_t e0 = c.get_event(), e1 = c.get_event();
  KS_CUDA(cudaEventRecord(e0, c.st));
  double flops = 0;
  DevBuf mean, G, V, lam, M, Wh;
  column_means(c, X, n_total, mean, tm);
  centred_covariance(c, X, mean.as<double>(), G, tm, &flops);
  symmetric_eigen(c, G, static_cast<int>(d), V, lam, tm);
  const size_t dd = static_cast<size_t>(d * d);
  M.alloc(sizeof(double) * dd);
  Wh.alloc(sizeof(double) * dd);
  tm.begin(PcaTimer::OTHER);
  zca_scale_kernel<<<static_cast<unsigned>(std::min<int64_t>((dd + 255) / 256, 4 * c.num_sms)), 256, 0, c.st>>>(
      V.as<double>(), lam.as<double>(), static_cast<int>(d), 1.0 / (n_total - 1.0), eps, M.as<double>());
  c.launches += 1;
  tm.end();
  tm.begin(PcaTimer::GRAM);  // whitener = M^T M = V diag(w) V^T: every rank holds the same M, no all-reduce
  gram_f64(c, operand_of(M.as<double>(), d, static_cast<int>(d)), nullptr, d, Wh.as<double>(), d, &flops);
  tm.end();
  const int64_t id = linear_model(c, Wh.as<double>(), d, d, mean.as<double>());
  KS_CUDA(cudaEventRecord(e1, c.st));
  std::vector<double> ev(d);
  KS_CUDA(cudaMemcpyAsync(ev.data(), lam.p, sizeof(double) * d, cudaMemcpyDeviceToHost, c.st));
  c.check_async("ZCAWhitenerEstimator.fit");
  std::reverse(ev.begin(), ev.end());
  write_stats(c, "zca", n_loc, n_total, d, static_cast<int>(d), 0, 0, tm, e0, e1, flops, "eigenvalues", ev, launches0, host_t0);
  return id;
}

// ------------------------------------------------------------------------------------ ApproximatePCAEstimator
// One CholeskyQR pass on Y (rows x l, row-major fp64, this rank's rows when distributed): G = Y^T Y [all-reduce], L L^T = G (+ shift),
// Y <- Y L^-T.  A plain pass whose factor shows cond(Y) > 1e5 (or fails) is repeated with the shift, so an exactly rank-deficient Y
// never breaks the factorisation.  Rank 0's L^-T is broadcast.  Returns whether the shift was used.
struct CholQrWork {
  DevBuf G, H, info, Ynew;
  DevBuf work;
  size_t work_bytes = 0;
  std::vector<uint8_t> host_work;
};
static bool cholqr_pass(Ctx& c, double* Y, int64_t rows, int l, double n_total, bool distributed, bool shift, CholQrWork& w, PcaTimer& tm,
                        double* flops) {
  SolverApi& api = solver_api();
  cusolverDnHandle_t h = solver_on_st(c);
  const size_t ll = static_cast<size_t>(l) * l;
  w.G.alloc(sizeof(double) * ll);
  w.H.alloc(sizeof(double) * (ll + 1));  // [L^-T | info]
  w.info.alloc(sizeof(int));
  w.Ynew.alloc(sizeof(double) * static_cast<size_t>(std::max<int64_t>(rows, 1)) * l);
  tm.begin(PcaTimer::QR);
  gram_f64(c, operand_of(Y, l, l), nullptr, rows, w.G.as<double>(), l, flops);
  tm.end();
  if (distributed) {
    tm.begin(PcaTimer::ALLREDUCE);
    c.allreduce_f64(w.G.as<double>(), ll);
    tm.end();
  }
  const double u = 1.1102230246251565e-16;
  const double shift_c = 11.0 * (n_total * l + static_cast<double>(l) * (l + 1)) * u;
  int lwork = 0;
  bool shifted = shift;
  for (int attempt = 0; attempt < 2; ++attempt) {
    tm.begin(PcaTimer::QR);
    shifted_copy_kernel<<<1, 256, 0, c.st>>>(w.G.as<double>(), w.H.as<double>(), l, shifted ? shift_c : 0.0);
    if (api.DpotrfBufferSize(h, CUBLAS_FILL_MODE_LOWER, l, w.H.as<double>(), l, &lwork) != CUSOLVER_STATUS_SUCCESS)
      throw KsError{KS_ERR_SOLVER, "cusolverDnDpotrf_bufferSize failed"};
    if (w.work_bytes < sizeof(double) * static_cast<size_t>(lwork)) {
      KS_CUDA(cudaStreamSynchronize(c.st));
      w.work.alloc(sizeof(double) * static_cast<size_t>(lwork));
      w.work_bytes = w.work.bytes;
    }
    if (api.Dpotrf(h, CUBLAS_FILL_MODE_LOWER, l, w.H.as<double>(), l, w.work.as<double>(), lwork, w.info.as<int>()) != CUSOLVER_STATUS_SUCCESS)
      throw KsError{KS_ERR_SOLVER, "cusolverDnDpotrf failed"};
    c.launches += 2;
    tm.end();
    if (shifted) break;
    // cond(Y) >= max L_ii / min L_ii: a plain pass is only accurate while cond(Y)^2 u is small
    std::vector<double> diag(l);
    int info = 0;
    KS_CUDA(cudaMemcpy2DAsync(diag.data(), sizeof(double), w.H.p, sizeof(double) * (l + 1), sizeof(double), l, cudaMemcpyDeviceToHost, c.st));
    KS_CUDA(cudaMemcpyAsync(&info, w.info.p, sizeof(int), cudaMemcpyDeviceToHost, c.st));
    KS_CUDA(cudaStreamSynchronize(c.st));
    double lo = INFINITY, hi = 0.0;
    for (double v : diag) {
      lo = std::min(lo, std::fabs(v));
      hi = std::max(hi, std::fabs(v));
    }
    if (info == 0 && lo > 0.0 && hi / lo <= 1e5 && std::isfinite(hi)) break;
    shifted = true;
  }
  tm.begin(PcaTimer::QR);
  size_t dev_bytes = 0, host_bytes = 0;
  if (api.XtrtriBufferSize(h, CUBLAS_FILL_MODE_LOWER, CUBLAS_DIAG_NON_UNIT, l, CUDA_R_64F, w.H.p, l, &dev_bytes, &host_bytes) !=
      CUSOLVER_STATUS_SUCCESS)
    throw KsError{KS_ERR_SOLVER, "cusolverDnXtrtri_bufferSize failed"};
  DevBuf info2;
  info2.alloc(sizeof(int));
  if (w.work_bytes < dev_bytes) {
    KS_CUDA(cudaStreamSynchronize(c.st));
    w.work.alloc(dev_bytes);
    w.work_bytes = w.work.bytes;
  }
  if (w.host_work.size() < host_bytes) w.host_work.resize(host_bytes);
  // a failed factorisation leaves info != 0: trtri still runs on the partial factor; the broadcast flag reports the failure
  if (api.Xtrtri(h, CUBLAS_FILL_MODE_LOWER, CUBLAS_DIAG_NON_UNIT, l, CUDA_R_64F, w.H.p, l, w.work.p, dev_bytes,
                 host_bytes ? w.host_work.data() : nullptr, host_bytes, info2.as<int>()) != CUSOLVER_STATUS_SUCCESS)
    throw KsError{KS_ERR_SOLVER, "cusolverDnXtrtri failed"};
  lower_only_kernel<<<static_cast<unsigned>(std::min<size_t>((ll + 255) / 256, 1024)), 256, 0, c.st>>>(w.H.as<double>(), l, w.info.as<int>(),
                                                                                                       w.H.as<double>() + ll);
  c.launches += 2;
  bcast_f64(c, w.H.as<double>(), ll + 1);
  tm.end();
  double flag = 0;
  KS_CUDA(cudaMemcpyAsync(&flag, w.H.as<double>() + ll, sizeof(double), cudaMemcpyDeviceToHost, c.st));
  KS_CUDA(cudaStreamSynchronize(c.st));
  if (flag != 0) throw KsError{KS_ERR_SOLVER, "CholeskyQR: the shifted Gram matrix is not positive definite (non-finite data?)"};
  tm.begin(PcaTimer::QR);
  skinny_f64(c, operand_of(Y, l, l), rows, w.H.as<double>(), l, l, w.Ynew.as<double>(), l);
  if (flops) *flops += 2.0 * static_cast<double>(rows) * l * l;
  if (rows > 0) KS_CUDA(cudaMemcpyAsync(Y, w.Ynew.p, sizeof(double) * static_cast<size_t>(rows) * l, cudaMemcpyDeviceToDevice, c.st));
  tm.end();
  return shifted;
}
// shifted CholeskyQR3: Y (rows x l) becomes the orthonormal Q of Y = Q R.  A shifted pass, then plain ones; when a later pass needs
// the shift too (an exactly rank-deficient Y: each shifted pass lifts its null directions by about 1 / sqrt(shift)), passes continue
// until one from the third on runs plain, at most 8.  Every rank takes the same decisions: they follow rank 0's broadcast factor.
static int cholqr3(Ctx& c, double* Y, int64_t rows, int l, double n_total, bool distributed, CholQrWork& w, PcaTimer& tm, double* flops) {
  int shifted = 0;
  for (int pass = 0; pass < 8; ++pass) {
    const bool sh = cholqr_pass(c, Y, rows, l, n_total, distributed, pass == 0, w, tm, flops);
    shifted += sh ? 1 : 0;
    if (pass >= 2 && !sh) break;
  }
  return shifted;
}

// ApproximatePCAEstimator.approximateQ (ApproximatePCA.scala:69-85, HMT Algorithm 4.4): Q (this rank's rows x l, fp64) of the
// global N x l basis, from the caller's omega (d x l column-major)
static void approximate_q(Ctx& c, Matrix& X, const double* omega_colmajor, int l, int q, double n_total, DevBuf& Q, PcaTimer& tm,
                          double* flops, int* shifted) {
  const int64_t d = X.cols, n_loc = X.rows;
  // omega as a row-major d x l operand of the skinny product
  std::vector<double> om(static_cast<size_t>(d) * l);
  for (int64_t i = 0; i < d; ++i)
    for (int j = 0; j < l; ++j) om[static_cast<size_t>(i) * l + j] = omega_colmajor[static_cast<size_t>(j) * d + i];
  DevBuf Om, Yh;
  Om.alloc(sizeof(double) * om.size());
  KS_CUDA(cudaMemcpyAsync(Om.p, om.data(), Om.bytes, cudaMemcpyHostToDevice, c.st));
  Q.alloc(sizeof(double) * static_cast<size_t>(std::max<int64_t>(n_loc, 1)) * l);
  Yh.alloc(sizeof(double) * static_cast<size_t>(d) * l);
  CholQrWork w, wh;
  const GramOperand xo = operand_of(X);
  tm.begin(PcaTimer::SKINNY);
  skinny_f64(c, xo, n_loc, Om.as<double>(), l, l, Q.as<double>(), l);  // Y = X omega
  *flops += 2.0 * static_cast<double>(n_loc) * d * l;
  tm.end();
  *shifted += cholqr3(c, Q.as<double>(), n_loc, l, n_total, true, w, tm, flops);
  for (int it = 0; it < q; ++it) {
    tm.begin(PcaTimer::GRAM);  // Yhat = X^T Q (d x l)
    const GramOperand qo = operand_of(Q.as<double>(), l, l);
    gram_f64(c, xo, &qo, n_loc, Yh.as<double>(), l, flops);
    tm.end();
    tm.begin(PcaTimer::ALLREDUCE);
    c.allreduce_f64(Yh.as<double>(), static_cast<size_t>(d) * l);
    tm.end();
    *shifted += cholqr3(c, Yh.as<double>(), d, l, static_cast<double>(d), false, wh, tm, flops);  // Q_h, the same on every rank
    tm.begin(PcaTimer::SKINNY);
    skinny_f64(c, xo, n_loc, Yh.as<double>(), l, l, Q.as<double>(), l);  // Y = X Q_h
    *flops += 2.0 * static_cast<double>(n_loc) * d * l;
    tm.end();
    *shifted += cholqr3(c, Q.as<double>(), n_loc, l, n_total, true, w, tm, flops);
  }
}

static void check_sketch_args(Ctx& c, Matrix& X, const double* omega, int l, int q, double n_total) {
  if (!omega) throw KsError{KS_ERR_INVALID, "null omega"};
  if (q < 0) throw KsError{KS_ERR_INVALID, "q must be >= 0"};
  if (l < 1 || static_cast<double>(l) > std::min(n_total, static_cast<double>(X.cols)))
    throw KsError{KS_ERR_INVALID, "the sketch size l = dims + p must be in [1, min(N, d)]"};
  (void)c;
}

int64_t approx_range(Ctx& c, Matrix& X, const double* omega_colmajor, int l, int q) {
  const int64_t launches0 = c.launches;
  const auto host_t0 = std::chrono::steady_clock::now();
  const double n_total = global_rows(c, X.rows);
  check_sketch_args(c, X, omega_colmajor, l, q, n_total);
  PcaTimer tm(c);
  cudaEvent_t e0 = c.get_event(), e1 = c.get_event();
  KS_CUDA(cudaEventRecord(e0, c.st));
  double flops = 0;
  int shifted = 0;
  DevBuf Q;
  approximate_q(c, X, omega_colmajor, l, q, n_total, Q, tm, &flops, &shifted);
  auto out = new_matrix(X.rows, l);
  KS_CUDA(cudaMemsetAsync(out->d, 0, out->buf.bytes, c.st));
  launch_f64_to_f32_rows(Q.as<double>(), l, out->d, out->ld, X.rows, l, c.st);
  c.launches += 1;
  KS_CUDA(cudaEventRecord(e1, c.st));
  c.check_async("ApproximatePCAEstimator.approximateQ");
  write_stats(c, "approximate_q", X.rows, n_total, X.cols, 0, l, q, tm, e0, e1, flops, "singular_values", {}, launches0, host_t0, shifted);
  return c.add(std::move(out));
}

int64_t fit_approx_pca(Ctx& c, Matrix& X, const double* omega_colmajor, int dims, int q, int p) {
  const int64_t d = X.cols, n_loc = X.rows;
  if (dims < 1 || dims > d) throw KsError{KS_ERR_INVALID, "dims must be in [1, d]"};
  if (p < 0) throw KsError{KS_ERR_INVALID, "p must be >= 0"};
  const int l = dims + p;
  const int64_t launches0 = c.launches;
  const auto host_t0 = std::chrono::steady_clock::now();
  const double n_total = global_rows(c, n_loc);
  check_sketch_args(c, X, omega_colmajor, l, q, n_total);
  PcaTimer tm(c);
  cudaEvent_t e0 = c.get_event(), e1 = c.get_event();
  KS_CUDA(cudaEventRecord(e0, c.st));
  double flops = 0;
  int shifted = 0;
  DevBuf Q, Cb, S, U, P, info;
  approximate_q(c, X, omega_colmajor, l, q, n_total, Q, tm, &flops, &shifted);
  // C = X^T Q (d x l, column-major) = (Q^T X) row-major: the cross Gram with the operands swapped
  Cb.alloc(sizeof(double) * static_cast<size_t>(d) * l);
  tm.begin(PcaTimer::GRAM);
  const GramOperand qo = operand_of(Q.as<double>(), l, l), xo = operand_of(X);
  gram_f64(c, qo, &xo, n_loc, Cb.as<double>(), d, &flops);
  tm.end();
  tm.begin(PcaTimer::ALLREDUCE);
  c.allreduce_f64(Cb.as<double>(), static_cast<size_t>(d) * l);
  tm.end();
  // the right singular vectors of B = Q^T X are the left singular vectors of C = B^T (d >= l)
  SolverApi& api = solver_api();
  cusolverDnHandle_t h = solver_on_st(c);
  U.alloc(sizeof(double) * (static_cast<size_t>(d) * l + l + 1));  // [U | S | info]
  double* Sv = U.as<double>() + static_cast<size_t>(d) * l;
  info.alloc(sizeof(int));
  tm.begin(PcaTimer::EIG);
  int lwork = 0;
  if (api.DgesvdBufferSize(h, static_cast<int>(d), l, &lwork) != CUSOLVER_STATUS_SUCCESS)
    throw KsError{KS_ERR_SOLVER, "cusolverDnDgesvd_bufferSize failed"};
  DevBuf work, rwork;
  work.alloc(sizeof(double) * static_cast<size_t>(std::max(lwork, 1)));
  rwork.alloc(sizeof(double) * static_cast<size_t>(l));
  if (api.Dgesvd(h, 'S', 'N', static_cast<int>(d), l, Cb.as<double>(), static_cast<int>(d), Sv, U.as<double>(), static_cast<int>(d), nullptr, 1,
                 work.as<double>(), lwork, rwork.as<double>(), info.as<int>()) != CUSOLVER_STATUS_SUCCESS)
    throw KsError{KS_ERR_SOLVER, "cusolverDnDgesvd failed"};
  info_to_flag_kernel<<<1, 1, 0, c.st>>>(info.as<int>(), Sv + l);
  c.launches += 2;
  bcast_f64(c, U.as<double>(), static_cast<size_t>(d) * l + l + 1);
  tm.end();
  double flag = 0;
  KS_CUDA(cudaMemcpyAsync(&flag, Sv + l, sizeof(double), cudaMemcpyDeviceToHost, c.st));
  KS_CUDA(cudaStreamSynchronize(c.st));
  if (flag != 0) throw KsError{KS_ERR_SOLVER, "cusolverDnDgesvd did not converge (info " + std::to_string(static_cast<int64_t>(flag)) + ")"};
  P.alloc(sizeof(double) * static_cast<size_t>(d) * dims);
  tm.begin(PcaTimer::OTHER);
  order_sign_kernel<<<dims, 256, 0, c.st>>>(U.as<double>(), d, static_cast<int>(d), 0, P.as<double>());
  c.launches += 1;
  tm.end();
  const int64_t id = linear_model(c, P.as<double>(), d, dims, nullptr);
  KS_CUDA(cudaEventRecord(e1, c.st));
  std::vector<double> sv(dims);
  KS_CUDA(cudaMemcpyAsync(sv.data(), Sv, sizeof(double) * dims, cudaMemcpyDeviceToHost, c.st));
  c.check_async("ApproximatePCAEstimator.fit");
  write_stats(c, "approximate_pca", n_loc, n_total, d, dims, l, q, tm, e0, e1, flops, "singular_values", sv, launches0, host_t0, shifted);
  return id;
}

// ------------------------------------------------------------------------------------ unit-test entry
void debug_gram_f64(Ctx& c, Matrix& A, Matrix* B, const double* shift_a, const double* shift_b, double* out, int64_t ld_out) {
  if (B && B->rows != A.rows) throw KsError{KS_ERR_INVALID, "row mismatch"};
  if (!out) throw KsError{KS_ERR_INVALID, "null out"};
  const int64_t m = A.cols, n = B ? B->cols : A.cols;
  if (ld_out < n) throw KsError{KS_ERR_INVALID, "ld_out < n"};
  DevBuf sa, sb, o;
  if (shift_a) {
    sa.alloc(sizeof(double) * m);
    KS_CUDA(cudaMemcpyAsync(sa.p, shift_a, sizeof(double) * m, cudaMemcpyHostToDevice, c.st));
  }
  if (B && shift_b) {
    sb.alloc(sizeof(double) * n);
    KS_CUDA(cudaMemcpyAsync(sb.p, shift_b, sizeof(double) * n, cudaMemcpyHostToDevice, c.st));
  }
  o.alloc(sizeof(double) * static_cast<size_t>(m * n));
  const GramOperand a = operand_of(A, shift_a ? sa.as<double>() : nullptr);
  GramOperand b;
  if (B) b = operand_of(*B, shift_b ? sb.as<double>() : nullptr);
  gram_f64(c, a, B ? &b : nullptr, A.rows, o.as<double>(), n);
  KS_CUDA(cudaMemcpy2DAsync(out, sizeof(double) * ld_out, o.p, sizeof(double) * n, sizeof(double) * n, m, cudaMemcpyDeviceToHost, c.st));
  c.check_async("debug_gram_f64");
}

}  // namespace ks
