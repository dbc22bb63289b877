// Host-side engine state shared by engine.cu (C ABI, BlockLS, apply) and bwls.cu (weighted solver).
#pragma once
#include <cuda_runtime.h>
#include <cusolverDn.h>
#include <nccl.h>
#include <stdint.h>

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

struct SolverApi {
  void* lib = nullptr;
  cusolverStatus_t (*Create)(cusolverDnHandle_t*) = nullptr;
  cusolverStatus_t (*Destroy)(cusolverDnHandle_t) = nullptr;
  cusolverStatus_t (*SetStream)(cusolverDnHandle_t, cudaStream_t) = nullptr;
  cusolverStatus_t (*DpotrfBufferSize)(cusolverDnHandle_t, cublasFillMode_t, int, double*, int, int*) = nullptr;
  cusolverStatus_t (*Dpotrf)(cusolverDnHandle_t, cublasFillMode_t, int, double*, int, double*, int, int*) = nullptr;
  cusolverStatus_t (*Dpotrs)(cusolverDnHandle_t, cublasFillMode_t, int, int, const double*, int, double*, int, int*) = nullptr;
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
  // Stream roles of the pipelined fit (engine.cu::fit_blockls), pipeline = 1 (default):
  //   st  (highest priority) solve chain: all-reduce of C, rhs assembly, triangular solves, operand packing
  //   st2 (lowest priority)  ALL tensor-core kernels in one order: C(j), G(j+1), proj(j+2), update(j) -- never two at once
  //   st3 (mid)              factor chain: fp64 system assembly + Cholesky of the block ahead
  //   st4 (mid)              all-reduce of G
  //   st5 (mid)              D2H copies of finished model blocks into the pinned host mirror
  // pipeline = 0 is the round-1 arrangement (residual chain incl. its tensor kernels on st, look-ahead tensor kernels on st2).
  cudaStream_t st = nullptr, st2 = nullptr, st3 = nullptr, st4 = nullptr, st5 = nullptr;
  ncclComm_t comm = nullptr;   // collectives issued on st
  ncclComm_t comm2 = nullptr;  // collectives issued on st2 (split of comm; falls back to comm)
  ncclComm_t comm3 = nullptr;  // collectives issued on st4 (pipeline 1: all-reduce of G)
  int pipeline = 1;
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
  std::map<std::vector<int>, std::unique_ptr<DevBuf>> tile_cache;
  // phase timing of the current fit
  struct Span { int phase; cudaEvent_t a, b; int stream; };
  cudaEvent_t timeline_origin = nullptr;  // when set, collect_spans also renders (phase, stream, start, end) per span
  std::string timeline_json;
  std::vector<Span> spans;
  std::vector<cudaEvent_t> event_pool;
  bool timing = true;

  Matrix& matrix(int64_t h);
  CosRF& rf(int64_t h);
  Model& model(int64_t h);
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

// Feature source: a materialised matrix or raw input + concatenated CosineRandomFeatures parameters.
struct FeatSrc {
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
  float* Wall = nullptr;
  float* Wfull = nullptr;  // unrounded fp32 weights (same layout as Wall)
  int kind = 0;            // feature-map kind of every gathered map (CosRF::kind; mixing kinds in one gather is rejected)
  float rect_floor = 0.f;
  float* ball = nullptr;
  int64_t ldw = 0, d_in = 0;
  int64_t D = 0, n_rows = 0;
  DevBuf zeros;  // max(D-block, d_in) zero floats
};
void make_feat_src(Ctx& c, int64_t features, int64_t x_in, const int64_t* rfs, int32_t n_rfs, FeatSrc& out,
                   int precision = 0);  // KS_PRECISION_*: which operand copies of X / W to prepare
void prepare_generated_operands(Ctx& c, FeatSrc& out, int precision);
// slab[rows x lds] = round_tf32(features[row_begin : row_begin+rows, c0 : c0+cols] - shift)   (shift may be the zero vector)
// colsum (optional, fp32[cols], must be zeroed): receives the column sums of the stored slab
// out16: the slab is fp16 (lds in fp16 elements), generated features only
void produce_slab(Ctx& c, FeatSrc& src, int64_t c0, int64_t cols, const float* shift, void* slab, int64_t lds,
                  int64_t row_begin, int64_t rows, bool round_out = true, float* colsum = nullptr, cudaStream_t st = nullptr,
                  bool out16 = false, bool x2 = false,  // x2: unrounded slab from the K-concatenated split operands: fp32, or
                  void* slab_lo = nullptr);             // (slab_lo given) the fp16 pair hi -> slab, lo -> slab_lo written by the epilogue
const GramTile* gram_tiles(Ctx& c, int b, int kcols, bool with_g, bool with_c, int* num_tiles);
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

}  // namespace ks
