// Row-sharded sparse matrices on the device: upload with a CSC copy, the two gather products of sparse L-BFGS (Q = A P over
// CSR, C = A^T R over CSC), Densify and SparseLinearMapper.apply.  DESIGN.md section 20.
//
// Both products are fp64 on CUDA cores and bound by memory and gathers.  Load is balanced by entries: every row / column is cut
// into chunks of at most kSpChunk entries (the work tables, built once at upload), one warp per chunk.  A chunk that covers its
// whole line writes the line; the chunks of a longer line write partials, and a second pass adds them in chunk order.  Within a
// chunk the sum order is fixed too (lanes in a fixed stride, then a fixed butterfly), and no floating-point sum uses atomics, so
// a product repeats bit for bit.
#include "engine.h"

#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cmath>
#include <limits>
#include <vector>

namespace ks {

static constexpr int kSpWarps = 8;  // warps per CTA of the chunk kernels

// ------------------------------------------------------------------------------------ upload
// flag |= 1: a column index outside [0, n_cols); |= 2: a value that is not finite
__global__ void sp_validate_kernel(const int32_t* __restrict__ idx, const double* __restrict__ val, int64_t nnz, int64_t n_cols,
                                   unsigned* flag) {
  unsigned f = 0;
  for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < nnz; e += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    if (idx[e] < 0 || idx[e] >= n_cols) f |= 1u;
    if (!isfinite(val[e])) f |= 2u;
  }
  if (f) atomicOr(flag, f);
}
__global__ void sp_iota_kernel(int64_t* __restrict__ p, int64_t n) {
  for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < n; e += static_cast<int64_t>(gridDim.x) * blockDim.x)
    p[e] = e;
}
// the row holding entry e: the last r with indptr[r] <= e
__device__ __forceinline__ int32_t sp_row_of(const int64_t* __restrict__ indptr, int64_t rows, int64_t e) {
  int64_t lo = 0, hi = rows;  // indptr[lo] <= e < indptr[hi]
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (indptr[mid] <= e) lo = mid;
    else hi = mid;
  }
  return static_cast<int32_t>(lo);
}
// CSC entry q = CSR entry perm[q] (columns sorted stably: rows ascend within a column, repeated entries keep their order)
__global__ void sp_gather_csc_kernel(const int64_t* __restrict__ perm, const int64_t* __restrict__ indptr, int64_t rows,
                                     const double* __restrict__ val, int32_t* __restrict__ rowidx, double* __restrict__ cval, int64_t nnz) {
  for (int64_t q = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; q < nnz; q += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t e = perm[q];
    rowidx[q] = sp_row_of(indptr, rows, e);
    cval[q] = val[e];
  }
}
// colptr[c] = the first sorted entry with column >= c, c in [0, n_cols]
__global__ void sp_colptr_kernel(const int32_t* __restrict__ keys, int64_t nnz, int64_t n_cols, int64_t* __restrict__ colptr) {
  const int64_t c = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (c > n_cols) return;
  int64_t lo = 0, hi = nnz;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (keys[mid] < c) lo = mid + 1;
    else hi = mid;
  }
  colptr[c] = lo;
}

static unsigned sp_grid(int64_t n, int threads = 256) {
  return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((n + threads - 1) / threads, 132 * 16)));
}

// the work table of lines [0, lines) with entry offsets ptr[0 .. lines]
static void build_table(const std::vector<int64_t>& ptr, int64_t lines, SpTable& t, cudaStream_t st) {
  std::vector<SpChunk> ch;
  std::vector<SpSplit> sp;
  ch.reserve(static_cast<size_t>(lines));
  int64_t parts = 0;
  for (int64_t l = 0; l < lines; ++l) {
    const int64_t b = ptr[l], e = ptr[l + 1];
    const int64_t n = std::max<int64_t>(1, (e - b + kSpChunk - 1) / kSpChunk);
    if (n == 1) {
      ch.push_back(SpChunk{b, e, -1, static_cast<int32_t>(l), 0});
      continue;
    }
    sp.push_back(SpSplit{parts, static_cast<int32_t>(l), static_cast<int32_t>(n)});
    for (int64_t q = 0; q < n; ++q) ch.push_back(SpChunk{b + q * kSpChunk, std::min(e, b + (q + 1) * kSpChunk), parts++, static_cast<int32_t>(l), 0});
  }
  t.n_chunks = static_cast<int64_t>(ch.size());
  t.n_splits = static_cast<int64_t>(sp.size());
  t.n_parts = parts;
  t.chunks.alloc(sizeof(SpChunk) * ch.size());
  t.splits.alloc(sizeof(SpSplit) * sp.size());
  if (!ch.empty()) KS_CUDA(cudaMemcpyAsync(t.chunks.p, ch.data(), sizeof(SpChunk) * ch.size(), cudaMemcpyHostToDevice, st));
  if (!sp.empty()) KS_CUDA(cudaMemcpyAsync(t.splits.p, sp.data(), sizeof(SpSplit) * sp.size(), cudaMemcpyHostToDevice, st));
  KS_CUDA(cudaStreamSynchronize(st));  // the host vectors go out of scope
}

std::unique_ptr<SparseMat> sparse_from_host_csr(Ctx& c, const int64_t* indptr, const int32_t* indices, const double* values, int64_t n_rows,
                                                int64_t n_cols) {
  if (!indptr) throw KsError{KS_ERR_INVALID, "null indptr"};
  if (n_rows < 0 || n_rows > std::numeric_limits<int32_t>::max()) throw KsError{KS_ERR_INVALID, "n_rows must lie in [0, 2^31)"};
  if (n_cols < 1 || n_cols > std::numeric_limits<int32_t>::max()) throw KsError{KS_ERR_INVALID, "n_cols must lie in [1, 2^31)"};
  if (indptr[0] != 0) throw KsError{KS_ERR_INVALID, "indptr[0] must be 0"};
  for (int64_t r = 0; r < n_rows; ++r)
    if (indptr[r + 1] < indptr[r]) throw KsError{KS_ERR_INVALID, "indptr decreases at row " + std::to_string(r)};
  const int64_t nnz = indptr[n_rows];
  if (nnz > 0 && (!indices || !values)) throw KsError{KS_ERR_INVALID, "null indices or values"};
  cudaStream_t st = c.st;
  auto s = std::make_unique<SparseMat>();
  s->rows = n_rows;
  s->cols = n_cols;
  s->nnz = nnz;
  s->indptr.alloc(sizeof(int64_t) * (n_rows + 1));
  s->indices.alloc(sizeof(int32_t) * nnz);
  s->values.alloc(sizeof(double) * nnz);
  KS_CUDA(cudaMemcpyAsync(s->indptr.p, indptr, sizeof(int64_t) * (n_rows + 1), cudaMemcpyHostToDevice, st));
  if (nnz > 0) {
    KS_CUDA(cudaMemcpyAsync(s->indices.p, indices, sizeof(int32_t) * nnz, cudaMemcpyHostToDevice, st));
    KS_CUDA(cudaMemcpyAsync(s->values.p, values, sizeof(double) * nnz, cudaMemcpyHostToDevice, st));
  }
  return sparse_from_device_csr(c, std::move(s), indptr);
}

std::unique_ptr<SparseMat> sparse_from_device_csr(Ctx& c, std::unique_ptr<SparseMat> s, const int64_t* host_indptr_or_null) {
  cudaStream_t st = c.st;
  const int64_t n_rows = s->rows, n_cols = s->cols, nnz = s->nnz;
  DevBuf flag;
  flag.alloc(sizeof(unsigned));
  KS_CUDA(cudaMemsetAsync(flag.p, 0, sizeof(unsigned), st));
  if (nnz > 0) {
    sp_validate_kernel<<<sp_grid(nnz), 256, 0, st>>>(s->indices.as<int32_t>(), s->values.as<double>(), nnz, n_cols, flag.as<unsigned>());
    c.launches += 1;
  }
  unsigned bad = 0;
  KS_CUDA(cudaMemcpyAsync(&bad, flag.p, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
  c.check_async("sparse upload");
  if (bad & 1u) throw KsError{KS_ERR_INVALID, "a column index lies outside [0, n_cols)"};
  if (bad & 2u) throw KsError{KS_ERR_INVALID, "a value is not finite"};

  // ---- CSC: a stable radix sort of (column, entry) pairs, then the rows and values gathered in that order
  s->colptr.alloc(sizeof(int64_t) * (n_cols + 1));
  s->rowidx.alloc(sizeof(int32_t) * nnz);
  s->cvalues.alloc(sizeof(double) * nnz);
  if (nnz > 0) {
    DevBuf keys, pos_in, pos_out, temp;
    keys.alloc(sizeof(int32_t) * nnz);
    pos_in.alloc(sizeof(int64_t) * nnz);
    pos_out.alloc(sizeof(int64_t) * nnz);
    sp_iota_kernel<<<sp_grid(nnz), 256, 0, st>>>(pos_in.as<int64_t>(), nnz);
    int end_bit = 1;
    while (end_bit < 31 && (int64_t(1) << end_bit) < n_cols) ++end_bit;
    size_t tb = 0;
    KS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, s->indices.as<int32_t>(), keys.as<int32_t>(), pos_in.as<int64_t>(),
                                            pos_out.as<int64_t>(), nnz, 0, end_bit, st));
    temp.alloc(tb);
    KS_CUDA(cub::DeviceRadixSort::SortPairs(temp.p, tb, s->indices.as<int32_t>(), keys.as<int32_t>(), pos_in.as<int64_t>(),
                                            pos_out.as<int64_t>(), nnz, 0, end_bit, st));
    sp_gather_csc_kernel<<<sp_grid(nnz), 256, 0, st>>>(pos_out.as<int64_t>(), s->indptr.as<int64_t>(), n_rows, s->values.as<double>(),
                                                       s->rowidx.as<int32_t>(), s->cvalues.as<double>(), nnz);
    sp_colptr_kernel<<<static_cast<unsigned>((n_cols + 256) / 256), 256, 0, st>>>(keys.as<int32_t>(), nnz, n_cols, s->colptr.as<int64_t>());
    c.launches += 4;
    KS_CUDA(cudaStreamSynchronize(st));
  } else {
    KS_CUDA(cudaMemsetAsync(s->colptr.p, 0, s->colptr.bytes, st));
  }
  std::vector<int64_t> colptr(static_cast<size_t>(n_cols + 1));
  KS_CUDA(cudaMemcpyAsync(colptr.data(), s->colptr.p, sizeof(int64_t) * (n_cols + 1), cudaMemcpyDeviceToHost, st));
  KS_CUDA(cudaStreamSynchronize(st));
  std::vector<int64_t> indptr(static_cast<size_t>(n_rows + 1));
  if (host_indptr_or_null) {
    std::copy(host_indptr_or_null, host_indptr_or_null + n_rows + 1, indptr.begin());
  } else {
    KS_CUDA(cudaMemcpyAsync(indptr.data(), s->indptr.p, sizeof(int64_t) * (n_rows + 1), cudaMemcpyDeviceToHost, st));
    KS_CUDA(cudaStreamSynchronize(st));
  }
  build_table(indptr, n_rows, s->rowt, st);
  build_table(colptr, n_cols, s->colt, st);
  c.check_async("sparse upload (CSC)");
  return s;
}

// ------------------------------------------------------------------------------------ the products
// One warp per chunk.  K > 0 (k == K <= 4): the lanes split the chunk's entries (lane l takes entries l, l + 32, ...), each with
// K accumulators, then a butterfly; lane 0's sum is the chunk's.  K == 0: the lanes take the k columns (c, c + 32, ...) and each
// runs over the chunk's entries in order.
template <int K>
__global__ void __launch_bounds__(32 * kSpWarps) sp_chunk_kernel(const SpChunk* __restrict__ chunks, int64_t n_chunks,
                                                                 const int32_t* __restrict__ idx, const double* __restrict__ val,
                                                                 const double* __restrict__ X, int k, const double* __restrict__ bias,
                                                                 double* __restrict__ out, double* __restrict__ partials) {
  const int lane = threadIdx.x & 31;
  const int64_t w = blockIdx.x * static_cast<int64_t>(kSpWarps) + (threadIdx.x >> 5);
  if (w >= n_chunks) return;
  const SpChunk ch = chunks[w];
  double* dst = ch.part < 0 ? out + static_cast<int64_t>(ch.line) * k : partials + ch.part * k;
  const bool add_bias = bias && ch.part < 0;
  if constexpr (K > 0) {
    double acc[K];
#pragma unroll
    for (int c = 0; c < K; ++c) acc[c] = 0.0;
    for (int64_t e = ch.begin + lane; e < ch.end; e += 32) {
      const double v = val[e];
      const double* x = X + static_cast<int64_t>(idx[e]) * K;
#pragma unroll
      for (int c = 0; c < K; ++c) acc[c] = fma(v, x[c], acc[c]);
    }
#pragma unroll
    for (int c = 0; c < K; ++c)
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], off);
    if (lane == 0) {
#pragma unroll
      for (int c = 0; c < K; ++c) dst[c] = add_bias ? acc[c] + bias[c] : acc[c];
    }
  } else {
    for (int c = lane; c < k; c += 32) {
      double a = 0.0;
#pragma unroll 4
      for (int64_t e = ch.begin; e < ch.end; ++e) a = fma(val[e], X[static_cast<int64_t>(idx[e]) * k + c], a);
      dst[c] = add_bias ? a + bias[c] : a;
    }
  }
}
// One CTA per split line: the line's partials added in a fixed order, plus the bias.  k >= 32: the threads take the columns, each
// summing its column's partials in chunk order; k < 32: thread t sums partials t, t + 256, ... in order, then a fixed tree.  (The
// head of a Zipf column distribution is split into tens of thousands of chunks: a single warp would walk them serially.)
__global__ void __launch_bounds__(256) sp_split_kernel(const SpSplit* __restrict__ splits, const double* __restrict__ partials, int k,
                                                       const double* __restrict__ bias, double* __restrict__ out) {
  __shared__ double red[256];
  const SpSplit sp = splits[blockIdx.x];
  double* dst = out + static_cast<int64_t>(sp.line) * k;
  const double* p = partials + sp.first * k;
  if (k >= 32) {
    for (int c = threadIdx.x; c < k; c += blockDim.x) {
      double a = p[c];
      for (int q = 1; q < sp.count; ++q) a += p[static_cast<int64_t>(q) * k + c];
      dst[c] = bias ? a + bias[c] : a;
    }
    return;
  }
  for (int c = 0; c < k; ++c) {
    double a = 0.0;
    for (int q = threadIdx.x; q < sp.count; q += blockDim.x) a += p[static_cast<int64_t>(q) * k + c];
    red[threadIdx.x] = a;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
      if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
      __syncthreads();
    }
    if (threadIdx.x == 0) dst[c] = bias ? red[0] + bias[c] : red[0];
    __syncthreads();
  }
}

void sparse_product(Ctx& c, const SparseMat& s, bool transpose, const double* X, int k, const double* bias, double* out, cudaStream_t st) {
  const SpTable& t = transpose ? s.colt : s.rowt;
  const int32_t* idx = transpose ? s.rowidx.as<int32_t>() : s.indices.as<int32_t>();
  const double* val = transpose ? s.cvalues.as<double>() : s.values.as<double>();
  if (t.n_chunks == 0) return;
  DevBuf partials;
  partials.alloc(sizeof(double) * static_cast<size_t>(t.n_parts) * k);
  const unsigned grid = static_cast<unsigned>((t.n_chunks + kSpWarps - 1) / kSpWarps);
  const SpChunk* ch = t.chunks.as<SpChunk>();
  switch (k) {
    case 1: sp_chunk_kernel<1><<<grid, 32 * kSpWarps, 0, st>>>(ch, t.n_chunks, idx, val, X, k, bias, out, partials.as<double>()); break;
    case 2: sp_chunk_kernel<2><<<grid, 32 * kSpWarps, 0, st>>>(ch, t.n_chunks, idx, val, X, k, bias, out, partials.as<double>()); break;
    case 3: sp_chunk_kernel<3><<<grid, 32 * kSpWarps, 0, st>>>(ch, t.n_chunks, idx, val, X, k, bias, out, partials.as<double>()); break;
    case 4: sp_chunk_kernel<4><<<grid, 32 * kSpWarps, 0, st>>>(ch, t.n_chunks, idx, val, X, k, bias, out, partials.as<double>()); break;
    default: sp_chunk_kernel<0><<<grid, 32 * kSpWarps, 0, st>>>(ch, t.n_chunks, idx, val, X, k, bias, out, partials.as<double>()); break;
  }
  c.launches += 1;
  if (t.n_splits > 0) {
    sp_split_kernel<<<static_cast<unsigned>(t.n_splits), 256, 0, st>>>(t.splits.as<SpSplit>(), partials.as<double>(), k, bias, out);
    c.launches += 1;
  }
}

// ------------------------------------------------------------------------------------ Densify and apply
// One thread per CSC chunk: each run of entries at the same (row, column) -- adjacent in the CSC, in upload order -- is summed in
// fp64 from 0 and rounded once.  A run that crosses a chunk boundary belongs to the chunk where it starts.
__global__ void sp_densify_kernel(const SpChunk* __restrict__ chunks, int64_t n_chunks, const int64_t* __restrict__ colptr,
                                  const int32_t* __restrict__ rowidx, const double* __restrict__ val, float* __restrict__ out, int64_t ld) {
  const int64_t w = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (w >= n_chunks) return;
  const SpChunk ch = chunks[w];
  const int64_t col_begin = colptr[ch.line], col_end = colptr[ch.line + 1];
  int64_t e = ch.begin;
  if (e > col_begin)
    while (e < ch.end && rowidx[e] == rowidx[ch.begin - 1]) ++e;
  while (e < ch.end) {
    const int32_t r = rowidx[e];
    double a = 0.0;
    for (; e < col_end && rowidx[e] == r; ++e) a += val[e];
    out[static_cast<int64_t>(r) * ld + ch.line] = static_cast<float>(a);
  }
}
std::unique_ptr<Matrix> sparse_densify(Ctx& c, const SparseMat& s) {
  auto m = new_matrix(s.rows, s.cols);
  KS_CUDA(cudaMemsetAsync(m->buf.p, 0, m->buf.bytes, c.st));
  if (s.colt.n_chunks > 0) {
    sp_densify_kernel<<<static_cast<unsigned>((s.colt.n_chunks + 255) / 256), 256, 0, c.st>>>(
        s.colt.chunks.as<SpChunk>(), s.colt.n_chunks, s.colptr.as<int64_t>(), s.rowidx.as<int32_t>(), s.cvalues.as<double>(), m->d, m->ld);
    c.launches += 1;
  }
  c.check_async("Densify");
  return m;
}

// Xr[(c0 + r) k + c] = W_j[c b + r]: model block j (column-major b x k) into the row-major operand of the CSR product
__global__ void sp_rows_from_block_kernel(const double* __restrict__ Wj, int64_t b, int k, int64_t c0, double* __restrict__ Xr) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= b * k) return;
  const int64_t r = i / k, cc = i - r * k;
  Xr[(c0 + r) * k + cc] = Wj[cc * b + r];
}
void launch_rows_from_block(Ctx& c, const double* Wj, int64_t b, int k, int64_t c0, double* Xr, cudaStream_t st) {
  sp_rows_from_block_kernel<<<static_cast<unsigned>((b * k + 255) / 256), 256, 0, st>>>(Wj, b, k, c0, Xr);
  c.launches += 1;
}
__global__ void sp_to_f32_kernel(const double* __restrict__ in, int64_t rows, int k, float* __restrict__ out, int64_t ld) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= rows * k) return;
  const int64_t r = i / k;
  out[r * ld + (i - r * k)] = static_cast<float>(in[i]);
}
std::unique_ptr<Matrix> sparse_model_apply(Ctx& c, Model& m, const SparseMat& s) {
  if (m.kernel) throw KsError{KS_ERR_INVALID, "a kernel model (KernelBlockLinearMapper) is not applied to sparse rows"};
  if (m.has_mean) throw KsError{KS_ERR_INVALID, "SparseLinearMapper has no feature means: the model carries feature scalers"};
  int64_t d = 0;
  for (auto r : m.brows) d += r;
  if (d != s.cols) throw KsError{KS_ERR_INVALID, "the model has " + std::to_string(d) + " feature rows, the data " + std::to_string(s.cols) + " columns"};
  const int k = static_cast<int>(m.k);
  cudaStream_t st = c.st;
  DevBuf Xr, out64;
  Xr.alloc(sizeof(double) * static_cast<size_t>(d) * k);
  out64.alloc(sizeof(double) * static_cast<size_t>(std::max<int64_t>(s.rows, 1)) * k);
  int64_t c0 = 0;
  for (size_t j = 0; j < m.brows.size(); ++j) {
    launch_rows_from_block(c, m.W[j]->as<double>(), m.brows[j], k, c0, Xr.as<double>(), st);
    c0 += m.brows[j];
  }
  sparse_product(c, s, false, Xr.as<double>(), k, m.has_intercept ? m.intercept.as<double>() : nullptr, out64.as<double>(), st);
  auto y = new_matrix(s.rows, k);
  KS_CUDA(cudaMemsetAsync(y->buf.p, 0, y->buf.bytes, st));
  if (s.rows > 0) {
    sp_to_f32_kernel<<<static_cast<unsigned>((s.rows * k + 255) / 256), 256, 0, st>>>(out64.as<double>(), s.rows, k, y->d, y->ld);
    c.launches += 1;
  }
  c.check_async("SparseLinearMapper.apply");
  return y;
}

}  // namespace ks
