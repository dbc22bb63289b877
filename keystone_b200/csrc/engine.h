// Host-side engine state shared by engine.cu (C ABI, BlockLS, apply) and bwls.cu (weighted solver).
#pragma once
#include <cuda_runtime.h>
#include <cusolverDn.h>
#include <nccl.h>
#include <stdint.h>

#include <functional>
#include <map>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/keystone_b200.h"
#include "kernels.h"

namespace ks {

struct KsError {
  int code;
  std::string msg;
};

#define KS_CUDA(call)                                                                                   \
  do {                                                                                                  \
    cudaError_t e__ = (call);                                                                           \
    if (e__ != cudaSuccess)                                                                             \
      throw ::ks::KsError{KS_ERR_CUDA, std::string(#call) + " failed: " + cudaGetErrorString(e__)};    \
  } while (0)

inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

// Device memory comes from a per-process caching pool (engine.cu): a fit needs ~35 GB of workspace (slab, residuals,
// operand copies) and cudaMalloc/cudaFree of that much costs ~0.25 s per call -- more than the featurize phase.
void* pool_alloc(size_t bytes);
void pool_free(void* p, size_t bytes);
void pool_release_all();

struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  void release() {
    if (p) pool_free(p, bytes);
    p = nullptr;
    bytes = 0;
  }
  void alloc(size_t n) {
    release();
    if (n == 0) n = 16;
    p = pool_alloc(n);
    bytes = n;
  }
  template <class T>
  T* as() const { return static_cast<T*>(p); }
};

// pinned host memory from a per-process caching pool (cudaHostAlloc of 0.5 GB costs ~0.2 s)
void* host_pool_alloc(size_t bytes);
void host_pool_free(void* p, size_t bytes);
struct HostBuf {
  void* p = nullptr;
  size_t bytes = 0;
  HostBuf() = default;
  HostBuf(const HostBuf&) = delete;
  HostBuf& operator=(const HostBuf&) = delete;
  ~HostBuf() { release(); }
  void release() {
    if (p) host_pool_free(p, bytes);
    p = nullptr;
    bytes = 0;
  }
  void alloc(size_t n) {
    release();
    p = host_pool_alloc(n ? n : 16);
    bytes = n ? n : 16;
  }
};

struct Matrix {  // fp32 row-major, ld % 32 == 0, padding columns are zero
  DevBuf buf;
  float* d = nullptr;
  int64_t rows = 0, cols = 0, ld = 0;
};

struct CosRF {
  DevBuf wbuf, wfbuf, bbuf;
  float* W = nullptr;     // [n_out][ld] tf32-rounded, K-major GEMM operand
  float* Wfull = nullptr; // [n_out][ld] fp32(W) unrounded: source of the fp16 / split operands (rounding once, not twice)
  float* bias = nullptr;  // [n_out]
  int64_t n_out = 0, n_in = 0, ld = 0;
  // kind 0: cos(x W^T + bias) (CosineRandomFeatures); kind 1: max(rect_floor, x W^T - bias) -- a dense linear node followed by
  // LinearRectifier (K/nodes/stats/LinearRectifier.scala:12-17; bias holds alpha per column, rect_floor = -inf: no rectifier)
  int kind = 0;
  float rect_floor = 0.f;
};

// Convolver [+ SymmetricRectifier + sum Pooler + ImageVectorizer] (K/nodes/images/{Convolver,SymmetricRectifier,Pooler}.scala),
// the featurizer of K/pipelines/images/cifar/RandomPatchCifar.scala:59-63
struct ConvPool {
  int x_dim = 0, y_dim = 0, ch = 0, conv = 0, n_filters = 0, normalize = 1;
  float var_constant = 10.f;
  int pd = 0;                 // patch dimension conv * conv * ch
  int64_t ld1 = 0, ld3 = 0;   // leading dimensions (fp16 elements) of the plain and of the K-concatenated operands
  DevBuf w16, w3, wscale, wmeans, fzero;  // filters as fp16 [n_filters][ld1] and [w_hi | w_hi | w_lo] [n_filters][ld3], times 2^e
  bool has_means = false;
};

// GaussianKernelGenerator.fit (K/nodes/learning/KernelGenerator.scala:121-176): the whole training X, replicated on every rank,
// shifted by its exact column mean m (distances are shift-invariant; the shift removes the cancellation in
// |x|^2 + |y|^2 - 2 x.y for uncentred data), with its split-operand copies and squared norms.  krr.cu, DESIGN.md section 13.
struct GaussKernel {
  double gamma = 0;
  int64_t n = 0, d = 0, ld = 0, ld3 = 0;
  int64_t row_off = 0, n_loc = 0;  // this rank's training rows [row_off, row_off + n_loc) in the global order
  DevBuf xs;     // fp32 [n][ld]: x - m
  DevBuf mean;   // fp64 [d]: m
  DevBuf xb3;    // fp16 [n][ld3]: [hi | hi | lo] of 2^e (x - m), the column-side operand of the generation GEMM
  DevBuf norms;  // fp32 [n]: sum of ((hi + lo) 2^-e)^2, the squared norm of exactly the values the pair represents
  DevBuf scale;  // fp32 [2]: 2^e, 2^-e
};

// GaussianMixtureModel(means, variances, weights, weightThreshold) (K/nodes/learning/GaussianMixtureModel.scala): fp64 parameters on
// the device for the posteriors and the Fisher vectors (fisher.cu, DESIGN.md section 16)
struct Gmm {
  int64_t dim = 0, k = 0;
  double thr = 1e-4;
  DevBuf buf;  // [mu | var | 0.5 / var] each dim x k row-major ([d][k]), then ck[k] = log w - 1/2 sum_d log var - dim/2 log 2 pi, w[k]
  const double* mu() const { return buf.as<double>(); }
  const double* var() const { return mu() + dim * k; }
  const double* hiv() const { return mu() + 2 * dim * k; }
  const double* ck() const { return mu() + 3 * dim * k; }
  const double* w() const { return ck() + k; }
};

struct Model {  // BlockLinearMapper state (K/nodes/learning/BlockLinearMapper.scala:22-33)
  std::shared_ptr<GaussKernel> kernel;  // KernelBlockLinearMapper (K/nodes/learning/KernelBlockLinearMapper.scala): the training rows
  int block_size = 0;
  int64_t k = 0;
  std::vector<int64_t> brows;
  std::vector<std::unique_ptr<DevBuf>> W;     // column-major (rows_j x k) fp64
  std::vector<std::unique_ptr<DevBuf>> mean;  // rows_j fp64 (if has_mean)
  DevBuf intercept;                           // k fp64
  bool has_mean = false, has_intercept = false;
  // Pinned host mirror written by async D2H copies while the fit is still running (block j's W_j / mean_j are final as soon
  // as its last update is packed): "all W_j, intercept on host" (SURVEY 8d) costs no extra time after the fit.
  HostBuf host;                               // [W_0 | mean_0 | W_1 | mean_1 | ... | intercept]
  std::vector<size_t> host_w_off, host_mean_off;
  size_t host_b_off = 0;
  bool host_valid = false;
};

// A rank's rows of a sparse matrix (sparse.cu, DESIGN.md section 20): CSR as uploaded and a CSC copy of the same entries (columns
// in order, rows ascending within a column, repeated entries in upload order), each with a work table that cuts its rows / columns
// into chunks of at most kSpChunk entries.  A line (row or column) of one chunk is written by that chunk; a longer line's chunks write
// partials that a second pass adds in chunk order.
static constexpr int64_t kSpChunk = 256;
struct SpChunk {
  int64_t begin, end;  // entry range
  int64_t part;        // -1: the chunk writes its line; otherwise its partial slot
  int32_t line, pad;
};
struct SpSplit {
  int64_t first;  // partial slots [first, first + count) of the line, in chunk order
  int32_t line, count;
};
struct SpTable {
  int64_t n_chunks = 0, n_splits = 0;
  DevBuf chunks, splits;  // SpChunk[n_chunks], SpSplit[n_splits]
  int64_t n_parts = 0;
};
struct SparseMat {
  int64_t rows = 0, cols = 0, nnz = 0;
  DevBuf indptr, indices, values;   // CSR: int64[rows + 1], int32[nnz], fp64[nnz]
  DevBuf colptr, rowidx, cvalues;   // CSC: int64[cols + 1], int32[nnz], fp64[nnz]
  SpTable rowt, colt;
};

struct TextObj;  // text batches, token batches, term frequencies and fitted feature spaces (text.cu, DESIGN.md section 23)

struct SolverApi {
  void* lib = nullptr;
  cusolverStatus_t (*Create)(cusolverDnHandle_t*) = nullptr;
  cusolverStatus_t (*Destroy)(cusolverDnHandle_t) = nullptr;
  cusolverStatus_t (*SetStream)(cusolverDnHandle_t, cudaStream_t) = nullptr;
  cusolverStatus_t (*DpotrfBufferSize)(cusolverDnHandle_t, cublasFillMode_t, int, double*, int, int*) = nullptr;
  cusolverStatus_t (*Dpotrf)(cusolverDnHandle_t, cublasFillMode_t, int, double*, int, double*, int, int*) = nullptr;
  cusolverStatus_t (*Dpotrs)(cusolverDnHandle_t, cublasFillMode_t, int, int, const double*, int, double*, int, int*) = nullptr;
  // PCA / ZCA / ApproximatePCA (pca.cu)
  cusolverStatus_t (*DsyevdBufferSize)(cusolverDnHandle_t, cusolverEigMode_t, cublasFillMode_t, int, const double*, int, const double*,
                                       int*) = nullptr;
  cusolverStatus_t (*Dsyevd)(cusolverDnHandle_t, cusolverEigMode_t, cublasFillMode_t, int, double*, int, double*, double*, int, int*) = nullptr;
  cusolverStatus_t (*DgesvdBufferSize)(cusolverDnHandle_t, int, int, int*) = nullptr;
  cusolverStatus_t (*Dgesvd)(cusolverDnHandle_t, signed char, signed char, int, int, double*, int, double*, double*, int, double*, int,
                             double*, int, double*, int*) = nullptr;
  cusolverStatus_t (*XtrtriBufferSize)(cusolverDnHandle_t, cublasFillMode_t, cublasDiagType_t, int64_t, cudaDataType, void*, int64_t,
                                       size_t*, size_t*) = nullptr;
  cusolverStatus_t (*Xtrtri)(cusolverDnHandle_t, cublasFillMode_t, cublasDiagType_t, int64_t, cudaDataType, void*, int64_t, void*, size_t,
                             void*, size_t, int*) = nullptr;
};
struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*CommSplit)(ncclComm_t, int, int, ncclComm_t*, ncclConfig_t*) = nullptr;  // optional (NCCL >= 2.18)
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
SolverApi& solver_api();  // throws KsError if libcusolver cannot be loaded
NcclApi& nccl_api();      // throws KsError if libnccl cannot be loaded
#define KS_NCCL(call)                                                                                      \
  do {                                                                                                     \
    ncclResult_t r__ = (call);                                                                             \
    if (r__ != ncclSuccess)                                                                                \
      throw ::ks::KsError{KS_ERR_NCCL, std::string(#call) + " failed: " + ::ks::nccl_api().GetErrorString(r__)}; \
  } while (0)

enum Phase { PH_FEATURIZE = 0, PH_GRAM, PH_ALLREDUCE, PH_SOLVE, PH_UPDATE, PH_OTHER, PH_COUNT };

struct Ctx {
  int device = 0, rank = 0, world = 1;
  int num_sms = 132;
  // Stream roles of the pipelined fit (engine.cu::fit_blockls), LA = look-ahead in blocks:
  //   st  (highest priority) solve chain: all-reduce of C, rhs assembly, triangular solves, operand packing
  //   st2 (lowest priority)  ALL tensor-core kernels in one order: C(t), G(t+LA), update(t), proj(t+LA+1) -- never two at once
  //   st3 (mid)              factor chain: fp64 system assembly + Cholesky of the blocks ahead
  //   st4 (mid)              all-reduce of G
  //   st5 (mid)              D2H copies of finished model blocks into the pinned host mirror
  cudaStream_t st = nullptr, st2 = nullptr, st3 = nullptr, st4 = nullptr, st5 = nullptr;
  ncclComm_t comm = nullptr;   // collectives issued on st
  ncclComm_t comm2 = nullptr;  // collectives issued on st2 (split of comm; falls back to comm)
  ncclComm_t comm3 = nullptr;  // collectives issued on st4 (all-reduce of G)
  int lookahead = 0;    // blocks the projection / G-Gram / factorisation run ahead of the residual chain; 0 = 1 on one GPU, 2 on several
  int host_mirror = 1;  // fits mirror the model into pinned host memory while they run
  int shard_solve = 1;  // world > 1: every rank runs the triangular solves for its k / world right-hand sides only and the
                        // columns of dW are gathered (grouped ncclBroadcast, 32 MB at b = 4096, k = 1000) -- the solve is the
                        // serial term of the strong-scaling curve and its cost is proportional to the number of columns
  cusolverDnHandle_t solver = nullptr;   // triangular solves (main stream)
  cudaStream_t solver_stream = nullptr, solver2_stream = nullptr;  // streams the handles are currently bound to
  cusolverDnHandle_t solver2 = nullptr;  // factorizations (factor stream): a handle's internal cuBLAS workspace is per stream
  DevBuf solver_work;
  int solver_lwork = 0;
  // independent small factorisations (the per-class systems of the weighted solver) run on several lanes at once
  struct SolveLane {
    cudaStream_t s = nullptr;
    cusolverDnHandle_t h = nullptr;
    DevBuf work;
    int lwork = 0;
  };
  std::vector<std::unique_ptr<SolveLane>> lanes;
  int solve_lanes = 4;
  // ks_debug_bwls_capture: the next weighted fit copies the assembled fp64 system (H, rhs) of class bwls_cap_cls in block
  // bwls_cap_block at sweep 0 to these host buffers, then disarms
  int bwls_cap_block = -1, bwls_cap_cls = -1;
  double* bwls_cap_H = nullptr;
  double* bwls_cap_rhs = nullptr;
  // ks_debug_blockls_capture: steps of the next block least-squares fit whose state is copied to host buffers (KS_BLS_CAP_*)
  struct BlsCapture {
    int sweep, block;
    double* out[KS_BLS_CAP_COUNT];
  };
  std::vector<BlsCapture> bls_cap;
  void ensure_lanes(int n);
  // Cholesky factorisation of H (n x n, lower) + solve of nrhs right-hand sides in place, on lane q; status -> dev_info[slot]
  void lane_potrf_potrs(int q, double* H, int n, double* B, int nrhs, int info_slot);
  // *flag (device, fp64) = number of non-zero entries among dev_info[0, used); the slots are cleared
  void infos_to_flag(int used, double* flag, cudaStream_t s);
  DevBuf dev_info;  // int[kMaxInfo]
  std::string err;
  std::string stats_json;
  int64_t launches = 0;
  int64_t gram_chunk_rows = 0;  // rows of the contraction per Gram CTA; 0 = chosen from the local row count (engine.cu)
  int64_t split_chunk_rows = 4096;  // the same in the parity mode: short accumulation chains (the tensor core chops products at the accumulator granularity)
  int proj_f16 = 1;   // fp16 mode: the projection GEMM X W^T runs with fp16 operands too (0: tf32 operands, fp16 slab)
  int precision = KS_PRECISION_F16X2;  // what KS_PRECISION_DEFAULT resolves to: the split-operand parity mode
  int reserve_sms = 8; // SMs the persistent look-ahead kernel leaves to the critical chain
  int custom_solve = -1; // triangular solves of the critical chain: 0 = cusolverDnDpotrs, 1 = the library's DMMA kernel
                         // (solve_kernels.cu: one launch, co-resident with the look-ahead Gram CTAs), -1 = automatic: the DMMA
                         // kernel when the rank solves <= 512 right-hand sides (the column-sharded multi-GPU solve, where its
                         // CTA clusters cut the latency of the substitution), potrs otherwise.
  int64_t sample_rows = 16384;
  int64_t next_id = 1;
  std::unordered_map<int64_t, std::unique_ptr<Matrix>> matrices;
  std::unordered_map<int64_t, std::unique_ptr<CosRF>> rfs;
  std::unordered_map<int64_t, std::unique_ptr<Model>> models;
  std::unordered_map<int64_t, std::unique_ptr<ConvPool>> convs;
  std::unordered_map<int64_t, std::shared_ptr<GaussKernel>> kernels;
  std::unordered_map<int64_t, std::unique_ptr<Gmm>> gmms;
  std::unordered_map<int64_t, std::unique_ptr<SparseMat>> sparses;
  std::unordered_map<int64_t, std::shared_ptr<TextObj>> texts;
  int text_hash_bits = 64;  // bits kept of the 64-bit content hashes of text.cu (a test lowers it to force collisions)
  std::map<std::vector<int>, std::unique_ptr<DevBuf>> tile_cache;
  // phase timing of the current fit
  struct Span { int phase; cudaEvent_t a, b; int stream; };
  cudaEvent_t timeline_origin = nullptr;  // when set, collect_spans also renders (phase, stream, start, end) per span
  std::string timeline_json;
  std::vector<Span> spans;
  std::vector<cudaEvent_t> event_pool;

  Matrix& matrix(int64_t h);
  CosRF& rf(int64_t h);
  Model& model(int64_t h);
  SparseMat& sparse(int64_t h);
  int64_t add(std::unique_ptr<Matrix> m);
  int64_t add(std::unique_ptr<Model> m);
  cudaEvent_t get_event();
  void span_begin(int phase, cudaStream_t s = nullptr);
  void span_end(cudaStream_t s = nullptr);
  void collect_spans(double out_ms[PH_COUNT]);
  void allreduce_f32(float* p, size_t n, bool prep = false);
  void allreduce_f64(double* p, size_t n, bool prep = false);
  void allreduce_on(void* p, size_t n, bool f64, ncclComm_t cm, cudaStream_t s);
  DevBuf tile_counters;  // ring of zero-initialised tile counters for the persistent projection kernel (one per launch in flight)
  int tile_counter_next = 0;
  int dyn_tiles = 1;     // the projection kernel draws its tiles from a counter (0: static striding)
  int* next_tile_counter(cudaStream_t s);
  std::vector<cudaEvent_t> fit_events;  // events of the fit in flight (returned to event_pool when it ends, also on error)
  void allreduce_max_u32(unsigned* p, size_t n);
  void ensure_solver();
  void potrf(double* H, int n, int info_slot, cudaStream_t s);
  void potrs(const double* H, int n, double* B, int nrhs, int info_slot, cudaStream_t s);
  void check_infos(int used_slots);
  void check_async(const char* what);
};

// The feature map of a generated source, independent of its rows: the concatenated parameters (owned by the source they
// were gathered for) and the map kind.  Sources over other rows of the same map copy this part whole (derive_feat_src).
struct FeatMap {
  float* Wall = nullptr;
  float* Wfull = nullptr;  // unrounded fp32 weights (same layout as Wall)
  int kind = 0;            // feature-map kind of every gathered map (CosRF::kind; mixing kinds in one gather is rejected)
  float rect_floor = 0.f;
  float* ball = nullptr;
  int64_t ldw = 0, d_in = 0;
  int64_t D = 0;
};
// Feature source: a materialised matrix or raw input + concatenated CosineRandomFeatures parameters.
struct FeatSrc : FeatMap {
  Matrix* F = nullptr;
  Matrix* X = nullptr;
  DevBuf xop;   // tf32-rounded copy of X (GEMM operand)
  // fp16 operand mode: X and the projection weights as fp16, each multiplied by a device-chosen power of two;
  // pscale[0] = 1 / (x scale * w scale) is applied to the accumulator before the cosine
  DevBuf xop16, w16, pscale;
  bool proj16 = false;
  // split-operand mode (KS_PRECISION_F16X2): K-concatenated fp16 operands [x_hi | x_lo | x_hi] and [w_hi | w_hi | w_lo], so one
  // GEMM of depth 3 d_in accumulates x_hi w_hi + x_lo w_hi + x_hi w_lo
  DevBuf x3, w3;
  int64_t ldx3 = 0, ldw3 = 0;
  bool proj_x2 = false;
  DevBuf wcat, wcat_full, bcat;
  int64_t n_rows = 0;
  DevBuf zeros;  // max(D-block, d_in) zero floats
};
void make_feat_src(Ctx& c, int64_t features, int64_t x_in, const int64_t* rfs, int32_t n_rfs, FeatSrc& out,
                   int precision = 0);  // KS_PRECISION_*: which operand copies of X / W to prepare
void prepare_generated_operands(Ctx& c, FeatSrc& out, int precision);
// out: the generated source `src` (which must outlive it) applied to the rows of X instead of its own
void derive_feat_src(Ctx& c, const FeatSrc& src, Matrix* X, FeatSrc& out, int precision);
// slab[rows x lds] = round_tf32(features[row_begin : row_begin+rows, c0 : c0+cols] - shift)   (shift may be the zero vector)
// colsum (optional, fp32[cols], must be zeroed): receives the column sums of the stored slab
// out16: the slab is fp16 (lds in fp16 elements), generated features only
void produce_slab(Ctx& c, FeatSrc& src, int64_t c0, int64_t cols, const float* shift, void* slab, int64_t lds,
                  int64_t row_begin, int64_t rows, bool round_out = true, float* colsum = nullptr, cudaStream_t st = nullptr,
                  bool out16 = false, bool x2 = false,  // x2: unrounded slab from the K-concatenated split operands: fp32, or
                  void* slab_lo = nullptr,              // (slab_lo given) the fp16 pair hi -> slab, lo -> slab_lo written by the epilogue
                  double* colsumsq = nullptr);          // fp16 pair with colsum only (fp64[cols], zeroed): += sum of (hi + lo)^2
// split: the CTA-pair list of the split Gram (two entries per pair, see GramTile)
const GramTile* gram_tiles(Ctx& c, int b, int kcols, bool with_g, bool with_c, bool split, int* num_tiles);
// f16: slab and R are fp16 matrices (leading dimensions in elements); G / C stay fp32
void launch_gram_block(Ctx& c, const void* slab, int64_t lds, int64_t rows, int b, const void* R, int64_t ldr, int kcols,
                       float* G, int ldg, float* C, int ldc, bool with_g, bool with_c, cudaStream_t st = nullptr,
                       bool f16 = false, int64_t chunk_rows = 0,  // chunk_rows 0: the context's choice
                       const void* slab_lo = nullptr, const void* R_lo = nullptr);  // fp16 pairs: hi^T hi + lo^T hi + hi^T lo, one pass
// out[rows x k] (+)= (epi == EPI_UPDATE ? -1 : +1) * slab[rows x b] * bop[k x b]^T + cbias   (reduce: add into out)
// f16: slab and bop are fp16; the product is multiplied by *acc_scale_ptr (device scalar, may be null) before the epilogue
void launch_update(Ctx& c, const void* slab, int64_t lds, int64_t rows, int b, const void* bop, int64_t ldb, int k,
                   float* out, int64_t ldo, const float* cbias, int epi, bool reduce, cudaStream_t st = nullptr,
                   bool f16 = false, const float* acc_scale_ptr = nullptr,
                   const void* slab_lo = nullptr, const void* bop_lo = nullptr);  // fp16 pairs: all three products in one pass

int64_t fit_bwls(Ctx& c, FeatSrc& src, Matrix& Y, int bs, int num_iter, double lam, double w, int64_t nf_opt,
                 int precision = KS_PRECISION_TF32);
// small device helpers (engine.cu): *p = v;  dst (fp32) / dst64 (fp64) [i] = src[i] * scale, either output may be null
void launch_set_f64(double* p, double v, cudaStream_t st);
void launch_scale_f64(const double* src, double scale, float* dst, double* dst64, int n, cudaStream_t st);
// dense L-BFGS least squares (lbfgs.cu); collective
int64_t fit_lbfgs(Ctx& c, FeatSrc& src, Matrix& Y, bool fit_intercept, int num_corrections, double convergence_tol, int num_iterations,
                  double reg_param, int precision);
// allocates the pinned mirror of a model whose brows / k / has_mean are set; enqueue_block_to_host copies block j (async, stream s)
void model_alloc_host(Model& m);
void model_block_to_host(Model& m, int j, cudaStream_t s);
void model_intercept_to_host(Model& m, cudaStream_t s);

// Gaussian-kernel ridge regression (krr.cu)
std::unique_ptr<Matrix> new_matrix(int64_t rows, int64_t cols);
int64_t gaussian_kernel_create(Ctx& c, Matrix& X, double gamma);  // collective
std::unique_ptr<Matrix> gaussian_kernel_block(Ctx& c, const GaussKernel& K, Matrix& x, int64_t col0, int64_t cols);
int64_t fit_krr(Ctx& c, const std::shared_ptr<GaussKernel>& K, Matrix& Y, double lam, int bs, int epochs,
                const int32_t* order_or_null);  // collective
std::unique_ptr<Matrix> kernel_model_apply(Ctx& c, Model& md, Matrix& x);
int64_t kernel_model_from_host(Ctx& c, const std::shared_ptr<GaussKernel>& K, const double* const* xs, const int64_t* block_rows,
                               int32_t n_blocks, int64_t k, int32_t block_size);

// PCA, ZCA whitening and approximate PCA on the fp64 DMMA kernels (pca.cu); all collective
int64_t fit_pca(Ctx& c, Matrix& X, int dims);
int64_t fit_zca(Ctx& c, Matrix& X, double eps);
int64_t approx_range(Ctx& c, Matrix& X, const double* omega_colmajor, int l, int q);  // returns a matrix handle
int64_t fit_approx_pca(Ctx& c, Matrix& X, const double* omega_colmajor, int dims, int q, int p);
// out (m x n, row-major fp64, host) = (A - 1 s^T)^T (B - 1 t^T); B null: symmetric mode.  Not collective.
void debug_gram_f64(Ctx& c, Matrix& A, Matrix* B, const double* shift_a, const double* shift_b, double* out, int64_t ld_out);
// The fp64 DMMA products of pca.cu, on c.st.  An operand is row-major with exactly one of f32 (fp32 device matrix) / f64 set; its
// column shift (may be null) is subtracted in fp64 as it is loaded.
struct GramOperand {
  const float* f32 = nullptr;
  const double* f64 = nullptr;
  int64_t ld = 0;
  int cols = 0;
  const double* shift = nullptr;
};
// out (a.cols x b.cols, row-major, ld ldo) = (A - 1 s^T)^T (B - 1 t^T) over `rows` rows; b null: symmetric mode (B = A).  Split-K over
// rows with the partials summed in split order: deterministic.  rows = 0 writes zeros.  flops (may be null) += the product's flops.
void gram_f64(Ctx& c, const GramOperand& a, const GramOperand* b, int64_t rows, double* out, int64_t ldo, double* flops = nullptr);
// Y (rows x l, row-major, ld ldy) = A B for A = a (rows x a.cols, no shift) and a row-major fp64 B (a.cols x l, ld ldb)
void skinny_f64(Ctx& c, const GramOperand& a, int64_t rows, const double* B, int64_t ldb, int l, double* Y, int64_t ldy);

// LCS descriptors, GMM posteriors, Fisher vectors and row normalisation (fisher.cu); none is collective
std::unique_ptr<Matrix> lcs_extract(Ctx& c, Matrix& images, int x_dim, int y_dim, int channels, int stride, int stride_start,
                                    int sub_patch_size);
int64_t gmm_create(Ctx& c, const double* means_colmajor, const double* vars_colmajor, const double* weights, int64_t dim, int64_t k,
                   double weight_threshold);
std::unique_ptr<Matrix> gmm_posteriors(Ctx& c, const Gmm& g, Matrix& X);
std::unique_ptr<Matrix> fisher_vector_apply(Ctx& c, const Gmm& g, Matrix& X, const int64_t* item_offsets, int64_t n_items);
std::unique_ptr<Matrix> normalize_rows(Ctx& c, Matrix& in);
void launch_signed_sqrt(Ctx& c, const float* in, float* out, int64_t n);
// building blocks of the mixture fit (fisher.cu): the posterior kernel with epilogue epi (1: posteriors and the per-row Xerox
// log-sum-exp into row_out, 2: one-hot hard assignment and the best distance into row_out; Q: rows x g.k, row_out indexed from row 0
// of X), fv_stats_kernel over n_items row ranges d_offs (device, absolute rows of X; Q row 0 is row q_row0), its tiles per item, and
// the rows of one posterior chunk (256 MB of fp64 Q)
void launch_gmm_estep(Ctx& c, const Gmm& g, const Matrix& X, int64_t row0, int64_t rows, double* Q, float* out, int64_t ldo, int epi,
                      double* row_out);
void launch_fv_stats(Ctx& c, const Matrix& X, const double* Q, int64_t ldq, int64_t q_row0, const int64_t* d_offs, int64_t n_items, int D,
                     int K, double* S);
int64_t fv_stats_tiles(int D, int K);
int64_t posterior_chunk_rows(const Gmm& g);

// Gaussian-mixture EM and k-means++ (gmm_fit.cu); not collective.  uniforms: the draw rule of include/keystone_b200.h.
struct KmeansResult {
  std::vector<double> means;  // K x D row-major
  std::vector<int64_t> seeds;
  int iterations = 0;
};
KmeansResult kmeans_fit(Ctx& c, Matrix& X, int64_t k, int max_iter, double tol, const double* uniforms);
std::unique_ptr<Matrix> kmeans_assign(Ctx& c, Matrix& X, const double* means_rowmajor, int64_t k, int64_t dim);
struct GmmFitArgs {
  int64_t k = 0;
  int max_iter = 100, init = 0;
  double min_cluster = 40, tol = 1e-4, thr = 1e-4, small_var = 1e-2, abs_var = 1e-9;
  const double* uniforms = nullptr;
};
// returns the model handle (weightThreshold 1e-4); means / vars D x K column-major, weights K
int64_t gmm_fit(Ctx& c, Matrix& X, const GmmFitArgs& a, double* means_colmajor, double* vars_colmajor, double* weights, int* iterations);
std::unique_ptr<Matrix> gather_rows(Ctx& c, Matrix& X, const int64_t* rows, int64_t n);

// PixelScaler, GrayScaler and dense multi-scale SIFT (sift.cu); none is collective
struct SiftScale {
  int b = 0, st = 0, lo = 0;  // bin size, step and first frame coordinate of the scale
  int nfx = 0, nfy = 0;       // frames along x (vlfeat's x, the Image's rows) and y
};
// validates the parameters (throws KS_ERR_INVALID) and returns the per-scale geometry; host only
std::vector<SiftScale> sift_geometry(int x_dim, int y_dim, int step, int bin, int scales, int scale_step);
std::unique_ptr<Matrix> image_pixel_scale(Ctx& c, Matrix& images);
std::unique_ptr<Matrix> image_grayscale(Ctx& c, Matrix& images, int x_dim, int y_dim, int channels, int pixel_scale);
std::unique_ptr<Matrix> sift_extract(Ctx& c, Matrix& gray_images, int x_dim, int y_dim, int step, int bin, int scales, int scale_step);
// throws KS_ERR_INVALID naming `who` when any of the first `cols` values of a row of m is not finite (sift.cu)
void check_finite(Ctx& c, const Matrix& m, int64_t cols, const char* who);

// HOG and DAISY descriptors (hog_daisy.cu); neither is collective
struct HogShape {
  int nx = 0, ny = 0;  // cells along x (the Image's rows) and y: Scala's round(dim / bin)
  int64_t rows = 0;    // feature rows per image, (nx - 2)(ny - 2) or 0
};
// validates the shape and bin (throws KS_ERR_INVALID), including the reference's out-of-image read; host only
HogShape hog_shape(int x_dim, int y_dim, int channels, int bin);
std::unique_ptr<Matrix> hog_extract(Ctx& c, Matrix& images, int x_dim, int y_dim, int channels, int pixel_scale, int bin);
struct DaisyShape {
  int nkx = 0, nky = 0, features = 0;     // keypoints along x and y; H (T Q + 1)
  std::vector<std::vector<double>> taps;  // the Gaussian taps of each blur layer
  std::vector<int> samples;               // (dx, dy, layer) of each histogram, the centre first, then ring sample (t, l) at 1 + t Q + l
};
// validates the parameters (throws KS_ERR_INVALID), including ring samples that leave the image; host only
DaisyShape daisy_shape(int x_dim, int y_dim, int T, int Q, int R, int H, int border, int stride);
std::unique_ptr<Matrix> daisy_extract(Ctx& c, Matrix& gray_images, int x_dim, int y_dim, int T, int Q, int R, int H, int border, int stride);

// Image views, Stats.normalizeRows, StandardScaler and the grouped confusion matrix (augment.cu).  Only the scaler fit is collective.
// views: n x 4 int32 (src_row, x0, y0, flip); throws KS_ERR_INVALID for a view ImageUtils.crop would reject or a flip outside {0, 1}
void check_views(const int32_t* views, int64_t n_views, int64_t n_images, int x_dim, int y_dim, int out_x, int out_y);
// rows [0, n) of out (ld ldo) = the views d_views[0, n) (device, checked) of images, each out_x * out_y * ch values, padding zeroed
void launch_image_views(Ctx& c, const Matrix& images, int x_dim, int ch, const int32_t* d_views, int64_t n, int out_x, int out_y,
                        float* out, int64_t ldo);
std::unique_ptr<Matrix> image_views(Ctx& c, Matrix& images, int x_dim, int y_dim, int ch, const int32_t* views, int64_t n_views, int out_x,
                                    int out_y);
std::unique_ptr<Matrix> stats_normalize_rows(Ctx& c, Matrix& in, double alpha);
void standard_scaler_fit(Ctx& c, Matrix& X, int normalize_std, double eps, double* mean_out, double* std_out);
std::unique_ptr<Matrix> standard_scaler_apply(Ctx& c, Matrix& X, const double* mean, const double* std_or_null);
void grouped_confusion_matrix(Ctx& c, Matrix& scores, const int64_t* rows, const int64_t* group_offsets, int64_t n_groups,
                              const int32_t* labels, int64_t k, int policy, double* out);

// Sparse matrices (sparse.cu); none of these is collective
std::unique_ptr<SparseMat> sparse_from_host_csr(Ctx& c, const int64_t* indptr, const int32_t* indices, const double* values, int64_t n_rows,
                                                int64_t n_cols);
// the rest of an upload for a CSR already on the device (s: rows, cols, nnz, indptr, indices, values set): the checks of
// sparse_from_host_csr on the entries, the CSC copy and the work tables.  host_indptr_or_null: a host copy of indptr, if there is one.
std::unique_ptr<SparseMat> sparse_from_device_csr(Ctx& c, std::unique_ptr<SparseMat> s, const int64_t* host_indptr_or_null);
// out (lines x k, row-major fp64) = A X (transpose = false: lines = rows, X is cols x k) or A^T X (transpose = true: lines = cols,
// X is rows x k), X row-major with ld k; bias_or_null (k values) is added to every line.  Fixed summation order.
void sparse_product(Ctx& c, const SparseMat& s, bool transpose, const double* X, int k, const double* bias_or_null, double* out,
                    cudaStream_t st);
// Xr[(c0 + r) k + c] = Wj[c b + r]: a column-major b x k block of a model (or of the fit's blocked W / P) into rows [c0, c0 + b) of a
// row-major operand of the CSR product
void launch_rows_from_block(Ctx& c, const double* Wj, int64_t b, int k, int64_t c0, double* Xr, cudaStream_t st);
std::unique_ptr<Matrix> sparse_densify(Ctx& c, const SparseMat& s);
std::unique_ptr<Matrix> sparse_model_apply(Ctx& c, Model& m, const SparseMat& s);
// SparseLBFGSwithL2 (lbfgs.cu); collective
int64_t fit_sparse_lbfgs(Ctx& c, const SparseMat& s, Matrix& Y, bool fit_intercept, int num_corrections, double convergence_tol,
                         int num_iterations, double reg_param);
// LogisticRegressionEstimator and NaiveBayesEstimator (logistic.cu); collective.  Exactly one of features / sparse is a handle, the
// other 0; labels: the rank's n_labels class ids (host).
int64_t fit_logistic(Ctx& c, int64_t features, int64_t sparse, const int32_t* labels, int64_t n_labels, int num_classes, double reg_param,
                     int num_iterations, double convergence_tol);
int64_t fit_naive_bayes(Ctx& c, int64_t features, int64_t sparse, const int32_t* labels, int64_t n_labels, int num_classes, double lambda);

// runs fn on the context ctx as every C ABI entry does: KS_ERR_HANDLE for an unknown context, a thrown KsError becomes its code and
// ks_last_error's message (engine.cu)
int32_t guarded(int64_t ctx, const std::function<void(Ctx&)>& fn);

}  // namespace ks
