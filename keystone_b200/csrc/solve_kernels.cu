// Multi-right-hand-side Cholesky solve  X = (L L^T)^{-1} B  in ONE kernel on the fp64 tensor cores (DMMA m8n8k4).
//
// Replaces cusolverDnDpotrs on the critical chain of the block solver (the reference's `\` on the driver,
// K/nodes/learning/BlockWeightedLeastSquares.scala:272, mlmatrix NormalEquations for BlockLS).  cuSOLVER runs the two
// triangular solves as ~230 small dependent kernels; when they share the GPU with the tensor-core kernels of the look-ahead,
// every one of those launches waits for SMs that Gram CTAs or the persistent projection kernel are holding -- on the critical
// path of the whole fit.  This kernel is built to run BESIDE them instead:
//   * one launch; a CTA owns NC right-hand sides and performs the complete forward and backward substitution for them, so
//     there is no inter-CTA dependency and no grid synchronisation;
//   * no shared-memory tiles in the bulk loops and 10 KB in total: it fits next to a ~196 KB Gram CTA on the same SM
//     (registers and thread slots are free there), so its CTAs become resident at once instead of queueing for an SM;
//   * all bulk arithmetic is DMMA (mma.sync.m8n8k4.f64) with operand fragments loaded straight from L2 in fully used
//     32 / 64 B sectors; the in-tile substitutions are products with the pre-inverted 64 x 64 diagonal tiles (tri_inv_tiles,
//     computed on the factor stream right after the Cholesky), i.e. DMMA as well -- no serial per-row dependency chains.
//
//   forward   for each 64-row tile I:  V = B_I - L[I, 0:i0] Y[0:i0]      Y_I = inv(L_II) V
//   backward  for each tile I (last to first): V = Y_I - L[i1:n, I]^T X[i1:n]      X_I = inv(L_II)^T V
//
// L: column-major n x n (ld = n), lower triangle valid (cusolverDnDpotrf, CUBLAS_FILL_MODE_LOWER).  B: column-major n x k.
// Dinv: ceil(n / 64) tiles of 64 x 64 doubles, column-major inside a tile, zero above the diagonal and beyond n.
#include "cluster.cuh"
#include "kernels.h"

namespace ks {

namespace {
constexpr int TS = 64;  // tile rows
constexpr int U = 16;   // k-steps (of 4) whose operand loads are in flight per warp (64 rows of the contraction)

__device__ __forceinline__ void dmma(double (&d)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(d[0]), "+d"(d[1])
               : "d"(a), "d"(b));
}

// acc[g] (8 rows x 8 columns per n-group g) += A[8 x K] * Bm[K x 8 NG] over K = [k0, k1) (multiples of 4 * U).
//   A(m, kk)  = TRANS ? Aptr[kk + m * lda] : Aptr[m + kk * lda]     m = lane / 4, kk = lane % 4 (+ 4 per step)
//   Bm(kk, c) = Bptr[kk + c * ldb]                                   kk = lane % 4, c = lane / 4 (+ 8 per n-group)
// Rows kk >= krow_limit of A / Bm and A rows m >= mrow_limit read as zero (ragged edges).
// A (the factor) streams from L2 and is prefetched one 64-row chunk ahead (its latency hides behind the 16 NG DMMAs of the
// current chunk); Bm (rows this CTA solved earlier) is read through L1, where the eight warps of the CTA share it.
template <int NG, bool TRANS>
__device__ __forceinline__ void bulk_dmma(double (&acc)[NG][2], const double* __restrict__ Aptr, size_t lda, int mrow_limit,
                                          const double* Bptr, size_t ldb, const bool (&col_ok)[NG], int k0, int k1, int krow_limit,
                                          int lane) {
  const int m = lane >> 2, kq = lane & 3;
  const bool m_ok = m < mrow_limit;
  if (k0 >= k1) return;
  double a[U], an[U];
  auto load_a = [&](double (&dst)[U], int kb) {
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int kk = kb + 4 * u + kq;
      dst[u] = (kk < krow_limit && m_ok) ? __ldg(TRANS ? Aptr + kk + static_cast<size_t>(m) * lda : Aptr + m + static_cast<size_t>(kk) * lda) : 0.0;
    }
  };
  load_a(a, k0);
  for (int kb = k0; kb < k1; kb += 4 * U) {
    const bool more = kb + 4 * U < k1;
    if (more) load_a(an, kb + 4 * U);
#pragma unroll
    for (int h = 0; h < 2; ++h) {   // two half-chunks: 8 steps of B operands in registers at a time
      double b[U / 2][NG];
#pragma unroll
      for (int u = 0; u < U / 2; ++u) {
        const int kk = kb + 4 * (h * (U / 2) + u) + kq;
#pragma unroll
        for (int g = 0; g < NG; ++g) b[u][g] = (kk < krow_limit && col_ok[g]) ? Bptr[kk + static_cast<size_t>(8 * g + m) * ldb] : 0.0;
      }
#pragma unroll
      for (int u = 0; u < U / 2; ++u)
#pragma unroll
        for (int g = 0; g < NG; ++g) dmma(acc[g], a[h * (U / 2) + u], b[u][g]);
    }
    if (more) {
#pragma unroll
      for (int u = 0; u < U; ++u) a[u] = an[u];
    }
  }
}
}  // namespace

// 8 warps: warp w owns rows 8 w .. 8 w + 8 of the current 64-row tile.  Shared memory: the 64 x NC tile right-hand side only
// (10 KB at NC = 16), registers ~130 x 256 threads: a CTA fits beside a Gram CTA (209 KB shared, 14 K registers) on one SM.
template <int NC>
__global__ void __maxnreg__(168)
chol_solve_kernel(const double* __restrict__ L, const double* __restrict__ Dinv, int n, double* B, int k) {
  constexpr int NG = NC / 8;
  constexpr int VP = NC + 4;                 // pitch of sV: conflict-free B-fragment reads (k * VP + c distinct mod 16)
  __shared__ double sV[TS * VP];             // tile right-hand side after the bulk update (B operand of the diagonal product)
  const int t = threadIdx.x, rg = t >> 5, lane = t & 31;
  const int c0 = blockIdx.x * NC;
  const size_t ld = static_cast<size_t>(n);
  const int ntiles = (n + TS - 1) / TS;
  const int npad = ntiles * TS;
  const int m = lane >> 2, cq = lane & 3;
  bool col_ok[NG];
#pragma unroll
  for (int g = 0; g < NG; ++g) col_ok[g] = c0 + 8 * g + m < k;       // B-fragment column of this lane
  double* Bc = B + static_cast<size_t>(c0) * ld;

  for (int pass = 0; pass < 2; ++pass) {
    for (int step = 0; step < ntiles; ++step) {
      const int it = pass == 0 ? step : ntiles - 1 - step;
      const int i0 = it * TS;
      const int r0 = i0 + 8 * rg;                                       // first row of this warp
      double acc[NG][2];
#pragma unroll
      for (int g = 0; g < NG; ++g) acc[g][0] = acc[g][1] = 0.0;
      // ---- bulk update over the already solved rows: [0, i0) forward, [i0 + TS, npad) backward
      if (pass == 0) bulk_dmma<NG, false>(acc, L + r0, ld, n - r0, Bc, ld, col_ok, 0, i0, n, lane);
      else bulk_dmma<NG, true>(acc, L + static_cast<size_t>(r0) * ld, ld, n - r0, Bc, ld, col_ok, i0 + TS, npad, n, lane);
      // ---- V = B_I - acc  (C fragment: row m, columns 2 cq, 2 cq + 1 of n-group g) -> shared
#pragma unroll
      for (int g = 0; g < NG; ++g)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int row = r0 + m, col = c0 + 8 * g + 2 * cq + e;
          const double bv = (row < n && col < k) ? B[row + static_cast<size_t>(col) * ld] : 0.0;
          sV[(8 * rg + m) * VP + 8 * g + 2 * cq + e] = bv - acc[g][e];
        }
      __syncthreads();
      // ---- in-tile solve as a product with the inverted diagonal tile (K = 64)
      double y[NG][2];
#pragma unroll
      for (int g = 0; g < NG; ++g) y[g][0] = y[g][1] = 0.0;
      {
        const double* Dt = Dinv + static_cast<size_t>(it) * TS * TS;
#pragma unroll
        for (int u = 0; u < TS / 4; ++u) {
          const int kk = 4 * u + cq;
          // forward: A(m, kk) = Dinv[8 rg + m][kk]; backward: A(m, kk) = Dinv[kk][8 rg + m]   (column-major tile)
          const double a = pass == 0 ? __ldg(Dt + (8 * rg + m) + kk * TS) : __ldg(Dt + kk + (8 * rg + m) * TS);
#pragma unroll
          for (int g = 0; g < NG; ++g) dmma(y[g], a, sV[kk * VP + 8 * g + m]);
        }
      }
#pragma unroll
      for (int g = 0; g < NG; ++g)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int row = r0 + m, col = c0 + 8 * g + 2 * cq + e;
          if (row < n && col < k) B[row + static_cast<size_t>(col) * ld] = y[g][e];
        }
      __syncthreads();  // the solved rows are visible to every warp of the CTA before the next tile reads them back
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Cluster variant for FEW right-hand sides (the column-sharded solve of the multi-GPU fit: k / world columns per rank).  A cluster
// of CL CTAs owns 8 right-hand sides; in every tile step each CTA accumulates its 1 / CL share of the contraction range, leaves the
// 64 x 8 partial sums in its own shared memory, the leader CTA reads them through distributed shared memory, finishes the tile
// (B_I - sum, product with the inverted diagonal tile) and publishes the solved rows; two cluster barriers per step.  The
// latency of the substitution (128 dependent tile steps) thus shrinks with CL: k = 125 -> 16 clusters of 8 CTAs.
__device__ __forceinline__ double ld_dsmem_f64(const double* local_ptr, uint32_t rank) {
  const uint32_t ra = cl_map_shared(static_cast<uint32_t>(__cvta_generic_to_shared(local_ptr)), rank);
  double v;
  asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(ra));
  return v;
}

// bulk update with the solved rows read through L2 (they were written by another CTA of the cluster)
template <bool TRANS>
__device__ __forceinline__ void bulk_dmma_cg(double (&acc)[2], const double* __restrict__ Aptr, size_t lda, int mrow_limit,
                                             const double* Bptr, size_t ldb, bool col_ok, int k0, int k1, int krow_limit, int lane) {
  const int m = lane >> 2, kq = lane & 3;
  const bool m_ok = m < mrow_limit;
  for (int kb = k0; kb < k1; kb += 4 * U) {
    double a[U], b[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int kk = kb + 4 * u + kq;
      const bool ok = kk < krow_limit;
      a[u] = (ok && m_ok) ? __ldg(TRANS ? Aptr + kk + static_cast<size_t>(m) * lda : Aptr + m + static_cast<size_t>(kk) * lda) : 0.0;
      b[u] = (ok && col_ok) ? __ldcg(Bptr + kk + static_cast<size_t>(m) * ldb) : 0.0;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) dmma(acc, a[u], b[u]);
  }
}

__global__ void __maxnreg__(168)
chol_solve_cluster_kernel(const double* __restrict__ L, const double* __restrict__ Dinv, int n, double* B, int k) {
  constexpr int NC = 8, VP = NC + 4;
  __shared__ double sV[TS * VP];      // leader: tile right-hand side after the bulk update
  __shared__ double sPart[TS * NC];   // every CTA: its partial sums of this tile step, read by the leader through DSMEM
  const int t = threadIdx.x, rg = t >> 5, lane = t & 31;
  const uint32_t cr = cl_ctarank(), cn = cl_nctarank();
  const int c0 = static_cast<int>(blockIdx.x / cn) * NC;
  const size_t ld = static_cast<size_t>(n);
  const int ntiles = (n + TS - 1) / TS;
  const int npad = ntiles * TS;
  const int m = lane >> 2, cq = lane & 3;
  const bool col_ok = c0 + m < k;
  double* Bc = B + static_cast<size_t>(c0) * ld;

  for (int pass = 0; pass < 2; ++pass) {
    for (int step = 0; step < ntiles; ++step) {
      const int it = pass == 0 ? step : ntiles - 1 - step;
      const int i0 = it * TS;
      const int r0 = i0 + 8 * rg;
      // this CTA's share of the contraction range, in whole 64-row chunks
      const int lo = pass == 0 ? 0 : i0 + TS;
      const int chunks = (pass == 0 ? i0 : npad - lo) / TS;
      const int kb0 = lo + TS * static_cast<int>(static_cast<int64_t>(chunks) * cr / cn);
      const int kb1 = lo + TS * static_cast<int>(static_cast<int64_t>(chunks) * (cr + 1) / cn);
      // the leader's operands that do not depend on this step's partial sums are fetched now, under the bulk update: the tile's
      // right-hand side and this warp's fragment of the inverted diagonal tile
      double bv[2] = {0.0, 0.0}, dfrag[TS / 4];
      if (cr == 0) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int row = r0 + m, col = c0 + 2 * cq + e;
          if (row < n && col < k) bv[e] = __ldcg(B + row + static_cast<size_t>(col) * ld);
        }
        const double* Dt = Dinv + static_cast<size_t>(it) * TS * TS;
#pragma unroll
        for (int u = 0; u < TS / 4; ++u) {
          const int kk = 4 * u + cq;
          dfrag[u] = pass == 0 ? __ldg(Dt + (8 * rg + m) + kk * TS) : __ldg(Dt + kk + (8 * rg + m) * TS);
        }
      }
      double acc[2] = {0.0, 0.0};
      if (pass == 0) bulk_dmma_cg<false>(acc, L + r0, ld, n - r0, Bc, ld, col_ok, kb0, kb1, n, lane);
      else bulk_dmma_cg<true>(acc, L + static_cast<size_t>(r0) * ld, ld, n - r0, Bc, ld, col_ok, kb0, kb1, n, lane);
      sPart[(8 * rg + m) * NC + 2 * cq + 0] = acc[0];
      sPart[(8 * rg + m) * NC + 2 * cq + 1] = acc[1];
      cl_sync();   // every CTA's partial sums are in its shared memory
      if (cr == 0) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          double part[8];
#pragma unroll
          for (int r = 0; r < 8; ++r)   // all loads in flight together; summed in a fixed order: deterministic
            part[r] = static_cast<uint32_t>(r) < cn ? ld_dsmem_f64(&sPart[(8 * rg + m) * NC + 2 * cq + e], static_cast<uint32_t>(r)) : 0.0;
          double s = 0.0;
#pragma unroll
          for (int r = 0; r < 8; ++r) s += part[r];
          sV[(8 * rg + m) * VP + 2 * cq + e] = bv[e] - s;
        }
        __syncthreads();
        double y[2] = {0.0, 0.0};
#pragma unroll
        for (int u = 0; u < TS / 4; ++u) dmma(y, dfrag[u], sV[(4 * u + cq) * VP + m]);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int row = r0 + m, col = c0 + 2 * cq + e;
          if (row < n && col < k) B[row + static_cast<size_t>(col) * ld] = y[e];
        }
        __threadfence();   // the solved rows are visible to the other CTAs of the cluster after the barrier
      }
      cl_sync();   // also: the partial-sum buffers may be overwritten again
    }
  }
}

// Inverse of every 64 x 64 diagonal tile of the Cholesky factor (lower triangular): one CTA per tile, thread j builds column j
// of the inverse by forward substitution.  Output tile it: Dinv[it][r + 64 c], zero above the diagonal and for rows / columns >= n.
__global__ void __launch_bounds__(TS)
tri_inv_tiles_kernel(const double* __restrict__ L, int n, double* __restrict__ Dinv) {
  __shared__ double sL[TS][TS + 1];
  const int it = blockIdx.x, j = threadIdx.x, i0 = it * TS;
  const size_t ld = static_cast<size_t>(n);
  for (int c = 0; c < TS; ++c) {
    const int r = j;
    sL[r][c] = (i0 + r < n && i0 + c < n && r >= c) ? L[(i0 + r) + (i0 + c) * ld] : (r == c ? 1.0 : 0.0);
  }
  __syncthreads();
  double x[TS];
#pragma unroll
  for (int r = 0; r < TS; ++r) x[r] = 0.0;
  const bool live = i0 + j < n;
#pragma unroll
  for (int r = 0; r < TS; ++r) {
    if (r >= j) {
      double s = (r == j) ? 1.0 : 0.0;
#pragma unroll
      for (int q = 0; q < TS; ++q)
        if (q < r && q >= j) s -= sL[r][q] * x[q];
      x[r] = s / sL[r][r];
    }
  }
  double* out = Dinv + static_cast<size_t>(it) * TS * TS + static_cast<size_t>(j) * TS;
#pragma unroll
  for (int r = 0; r < TS; ++r) out[r] = (live && r >= j && i0 + r < n) ? x[r] : 0.0;
}

size_t chol_solve_dinv_doubles(int n) { return static_cast<size_t>((n + TS - 1) / TS) * TS * TS; }

cudaError_t launch_tri_inv_tiles(const double* L, int n, double* Dinv, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  tri_inv_tiles_kernel<<<(n + TS - 1) / TS, TS, 0, st>>>(L, n, Dinv);
  return cudaGetLastError();
}

cudaError_t launch_chol_solve(const double* L, const double* Dinv, int n, double* B, int k, cudaStream_t st) {
  if (n <= 0 || k <= 0) return cudaSuccess;
  // 16 right-hand sides per CTA halve the L2 traffic for L (every CTA streams the whole factor twice); with few columns (the
  // column-sharded multi-GPU solve) 8 per CTA keep more SMs busy
  // few right-hand sides: clusters of CTAs share one group of 8 columns, so that up to one CTA per SM (132) works whatever k is
  const int groups = (k + 7) / 8;
  const int cl = groups <= 16 ? 8 : groups <= 33 ? 4 : groups <= 66 ? 2 : 1;
  if (cl > 1) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(static_cast<unsigned>(groups * cl));
    cfg.blockDim = dim3(256);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = static_cast<unsigned>(cl);
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, chol_solve_cluster_kernel, L, Dinv, n, B, k);
  }
  if (k > 8 * 132) chol_solve_kernel<16><<<(k + 15) / 16, 256, 0, st>>>(L, Dinv, n, B, k);
  else chol_solve_kernel<8><<<(k + 7) / 8, 256, 0, st>>>(L, Dinv, n, B, k);
  return cudaGetLastError();
}

}  // namespace ks
