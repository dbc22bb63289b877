// Host engine + C ABI of libkeystone_b200: contexts, row-sharded device matrices, the
// BlockLeastSquaresEstimator solver loop (K/nodes/learning/BlockLinearMapper.scala:212-243 and the
// mlmatrix BlockCoordinateDescent it delegates to), BlockLinearMapper apply (:40-87) and computeCost
// (:142-187).  All arithmetic of the hot path runs in the CUDA kernels of tc_kernels.cu /
// aux_kernels.cu and in cuSOLVER (dense Cholesky of the reduced b x b system); there is no CPU path.
#include "engine.h"

#include <cuda_fp16.h>
#include <dlfcn.h>
#include <stdlib.h>
#include <math.h>
#include <string.h>

#include <chrono>
#include <mutex>
#include <sstream>

namespace ks {

// ------------------------------------------------------------------------------------ dynamic libraries
template <class F>
static void load_sym(void* lib, const char* name, F& out, const char* libname) {
  void* s = dlsym(lib, name);
  if (!s) throw KsError{KS_ERR_SOLVER, std::string("symbol ") + name + " missing from " + libname};
  out = reinterpret_cast<F>(s);
}
static void* open_first(const std::vector<const char*>& names) {
  for (const char* n : names) {
    void* h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (h) return h;
  }
  return nullptr;
}
SolverApi& solver_api() {
  static SolverApi api;
  static std::once_flag once;
  static std::string fail;
  std::call_once(once, [] {
    try {
      api.lib = open_first({"libcusolver.so.11", "libcusolver.so", "/usr/local/cuda/lib64/libcusolver.so.11"});
      if (!api.lib) throw KsError{KS_ERR_SOLVER, std::string("cannot load libcusolver: ") + dlerror()};
      load_sym(api.lib, "cusolverDnCreate", api.Create, "libcusolver");
      load_sym(api.lib, "cusolverDnDestroy", api.Destroy, "libcusolver");
      load_sym(api.lib, "cusolverDnSetStream", api.SetStream, "libcusolver");
      load_sym(api.lib, "cusolverDnDpotrf_bufferSize", api.DpotrfBufferSize, "libcusolver");
      load_sym(api.lib, "cusolverDnDpotrf", api.Dpotrf, "libcusolver");
      load_sym(api.lib, "cusolverDnDpotrs", api.Dpotrs, "libcusolver");
    } catch (const KsError& e) {
      fail = e.msg;
    }
  });
  if (!fail.empty()) throw KsError{KS_ERR_SOLVER, fail};
  return api;
}
NcclApi& nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  static std::string fail;
  std::call_once(once, [] {
    try {
      api.lib = open_first({"libnccl.so.2", "libnccl.so"});
      if (!api.lib) throw KsError{KS_ERR_NCCL, std::string("cannot load libnccl: ") + dlerror()};
      load_sym(api.lib, "ncclGetUniqueId", api.GetUniqueId, "libnccl");
      load_sym(api.lib, "ncclCommInitRank", api.CommInitRank, "libnccl");
      load_sym(api.lib, "ncclCommDestroy", api.CommDestroy, "libnccl");
      load_sym(api.lib, "ncclAllReduce", api.AllReduce, "libnccl");
      load_sym(api.lib, "ncclBroadcast", api.Broadcast, "libnccl");
      load_sym(api.lib, "ncclGroupStart", api.GroupStart, "libnccl");
      load_sym(api.lib, "ncclGroupEnd", api.GroupEnd, "libnccl");
      load_sym(api.lib, "ncclGetErrorString", api.GetErrorString, "libnccl");
      api.CommSplit = reinterpret_cast<decltype(api.CommSplit)>(dlsym(api.lib, "ncclCommSplit"));
    } catch (const KsError& e) {
      fail = e.msg;
    }
  });
  if (!fail.empty()) throw KsError{KS_ERR_NCCL, fail};
  return api;
}
// ------------------------------------------------------------------------------------ caching device-memory pool
// Blocks are keyed by (device, size rounded up to 2 MiB); freed blocks are kept for reuse and released when the last
// context is destroyed.  Buffers freed here may still be in use by work queued on the context's stream: every path that
// frees workspace synchronises the stream first (check_async at the end of each entry point), as with cudaFree.
static std::mutex g_pool_mu;
static std::multimap<std::pair<int, size_t>, void*> g_pool_free;
static size_t pool_round(size_t n) { return (n + (size_t(2) << 20) - 1) & ~((size_t(2) << 20) - 1); }
void* pool_alloc(size_t bytes) {
  int dev = 0;
  cudaGetDevice(&dev);
  const size_t key = pool_round(bytes);
  {
    std::lock_guard<std::mutex> lk(g_pool_mu);
    auto it = g_pool_free.find({dev, key});
    if (it != g_pool_free.end()) {
      void* p = it->second;
      g_pool_free.erase(it);
      return p;
    }
  }
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, key);
  if (e != cudaSuccess) {  // give cached blocks back to the driver and retry once
    cudaGetLastError();
    pool_release_all();
    e = cudaMalloc(&p, key);
  }
  if (e != cudaSuccess) {
    cudaGetLastError();
    throw KsError{KS_ERR_CUDA, "cudaMalloc(" + std::to_string(key) + " bytes) failed: " + cudaGetErrorString(e)};
  }
  return p;
}
void pool_free(void* p, size_t bytes) {
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lk(g_pool_mu);
  g_pool_free.insert({{dev, pool_round(bytes)}, p});
}
void pool_release_all() {
  std::lock_guard<std::mutex> lk(g_pool_mu);
  int cur = 0;
  cudaGetDevice(&cur);
  for (auto& kv : g_pool_free) {
    cudaSetDevice(kv.first.first);
    cudaFree(kv.second);
  }
  g_pool_free.clear();
  cudaSetDevice(cur);
}

// pinned host blocks (model mirrors, upload staging): same caching scheme, keyed by size only
static std::multimap<size_t, void*> g_host_free;
void* host_pool_alloc(size_t bytes) {
  const size_t key = pool_round(bytes);
  {
    std::lock_guard<std::mutex> lk(g_pool_mu);
    auto it = g_host_free.find(key);
    if (it != g_host_free.end()) {
      void* p = it->second;
      g_host_free.erase(it);
      return p;
    }
  }
  void* p = nullptr;
  cudaError_t e = cudaHostAlloc(&p, key, cudaHostAllocPortable);
  if (e != cudaSuccess) {
    cudaGetLastError();
    throw KsError{KS_ERR_CUDA, "cudaHostAlloc(" + std::to_string(key) + " bytes) failed: " + cudaGetErrorString(e)};
  }
  return p;
}
void host_pool_free(void* p, size_t bytes) {
  std::lock_guard<std::mutex> lk(g_pool_mu);
  g_host_free.insert({pool_round(bytes), p});
}
static void host_pool_release_all() {
  std::lock_guard<std::mutex> lk(g_pool_mu);
  for (auto& kv : g_host_free) cudaFreeHost(kv.second);
  g_host_free.clear();
}

void model_alloc_host(Model& m) {
  size_t off = 0;
  m.host_w_off.clear();
  m.host_mean_off.clear();
  for (size_t j = 0; j < m.brows.size(); ++j) {
    m.host_w_off.push_back(off);
    off += sizeof(double) * static_cast<size_t>(m.brows[j]) * m.k;
    m.host_mean_off.push_back(off);
    off += sizeof(double) * static_cast<size_t>(m.brows[j]);
  }
  m.host_b_off = off;
  off += sizeof(double) * static_cast<size_t>(m.k);
  m.host.alloc(off);
  m.host_valid = true;
}
void model_block_to_host(Model& m, int j, cudaStream_t s) {
  if (!m.host_valid) return;
  uint8_t* h = static_cast<uint8_t*>(m.host.p);
  KS_CUDA(cudaMemcpyAsync(h + m.host_w_off[j], m.W[j]->p, sizeof(double) * static_cast<size_t>(m.brows[j]) * m.k,
                          cudaMemcpyDeviceToHost, s));
  if (m.has_mean)
    KS_CUDA(cudaMemcpyAsync(h + m.host_mean_off[j], m.mean[j]->p, sizeof(double) * static_cast<size_t>(m.brows[j]),
                            cudaMemcpyDeviceToHost, s));
}
void model_intercept_to_host(Model& m, cudaStream_t s) {
  if (!m.host_valid || !m.has_intercept) return;
  KS_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(m.host.p) + m.host_b_off, m.intercept.p, sizeof(double) * static_cast<size_t>(m.k),
                          cudaMemcpyDeviceToHost, s));
}

// ------------------------------------------------------------------------------------ Ctx
static constexpr int kMaxInfo = 4096;

Matrix& Ctx::matrix(int64_t h) {
  auto it = matrices.find(h);
  if (it == matrices.end()) throw KsError{KS_ERR_HANDLE, "unknown matrix handle " + std::to_string(h)};
  return *it->second;
}
CosRF& Ctx::rf(int64_t h) {
  auto it = rfs.find(h);
  if (it == rfs.end()) throw KsError{KS_ERR_HANDLE, "unknown CosineRandomFeatures handle " + std::to_string(h)};
  return *it->second;
}
Model& Ctx::model(int64_t h) {
  auto it = models.find(h);
  if (it == models.end()) throw KsError{KS_ERR_HANDLE, "unknown model handle " + std::to_string(h)};
  return *it->second;
}
int64_t Ctx::add(std::unique_ptr<Matrix> m) {
  const int64_t id = next_id++;
  matrices[id] = std::move(m);
  return id;
}
int64_t Ctx::add(std::unique_ptr<Model> m) {
  const int64_t id = next_id++;
  models[id] = std::move(m);
  return id;
}
cudaEvent_t Ctx::get_event() {
  cudaEvent_t e;
  if (!event_pool.empty()) {
    e = event_pool.back();
    event_pool.pop_back();
    return e;
  }
  KS_CUDA(cudaEventCreate(&e));
  return e;
}
void Ctx::span_begin(int phase, cudaStream_t s) {
  if (!timing) return;
  Span sp{phase, get_event(), get_event(), s == st2 ? 2 : s == st3 ? 3 : s == st4 ? 4 : s == st5 ? 5 : 1};
  KS_CUDA(cudaEventRecord(sp.a, s ? s : st));
  spans.push_back(sp);
}
void Ctx::span_end(cudaStream_t s) {
  if (!timing) return;
  KS_CUDA(cudaEventRecord(spans.back().b, s ? s : st));
}
void Ctx::collect_spans(double out_ms[PH_COUNT]) {
  for (int i = 0; i < PH_COUNT; ++i) out_ms[i] = 0;
  std::ostringstream tl;
  tl << "[";
  bool first = true;
  for (auto& s : spans) {
    float ms = 0;
    cudaEventSynchronize(s.b);
    cudaEventElapsedTime(&ms, s.a, s.b);
    out_ms[s.phase] += ms;
    if (timeline_origin) {
      float t0 = 0;
      cudaEventElapsedTime(&t0, timeline_origin, s.a);
      tl << (first ? "" : ",") << "[" << s.phase << "," << s.stream << "," << t0 << "," << (t0 + ms) << "]";
      first = false;
    }
    event_pool.push_back(s.a);
    event_pool.push_back(s.b);
  }
  tl << "]";
  timeline_json = timeline_origin ? tl.str() : "[]";
  spans.clear();
}
void Ctx::allreduce_f32(float* p, size_t n, bool prep) {
  if (world <= 1 || n == 0) return;
  KS_NCCL(nccl_api().AllReduce(p, p, n, ncclFloat32, ncclSum, prep ? comm2 : comm, prep ? st2 : st));
}
void Ctx::allreduce_f64(double* p, size_t n, bool prep) {
  if (world <= 1 || n == 0) return;
  KS_NCCL(nccl_api().AllReduce(p, p, n, ncclFloat64, ncclSum, prep ? comm2 : comm, prep ? st2 : st));
}
int* Ctx::next_tile_counter(cudaStream_t s) {
  constexpr int kCounters = 256;
  if (!tile_counters.p) tile_counters.alloc(sizeof(int) * kCounters);
  int* p = tile_counters.as<int>() + (tile_counter_next++ % kCounters);
  KS_CUDA(cudaMemsetAsync(p, 0, sizeof(int), s));
  return p;
}
void Ctx::allreduce_on(void* p, size_t n, bool f64, ncclComm_t cm, cudaStream_t s) {
  if (world <= 1 || n == 0) return;
  KS_NCCL(nccl_api().AllReduce(p, p, n, f64 ? ncclFloat64 : ncclFloat32, ncclSum, cm, s));
}
void Ctx::allreduce_max_u32(unsigned* p, size_t n) {
  if (world <= 1 || n == 0) return;
  KS_NCCL(nccl_api().AllReduce(p, p, n, ncclUint32, ncclMax, comm, st));
}
void Ctx::ensure_solver() {
  if (solver) return;
  SolverApi& api = solver_api();
  if (api.Create(&solver) != CUSOLVER_STATUS_SUCCESS) throw KsError{KS_ERR_SOLVER, "cusolverDnCreate failed"};
  if (api.Create(&solver2) != CUSOLVER_STATUS_SUCCESS) throw KsError{KS_ERR_SOLVER, "cusolverDnCreate failed"};
  if (api.SetStream(solver, st) != CUSOLVER_STATUS_SUCCESS) throw KsError{KS_ERR_SOLVER, "cusolverDnSetStream failed"};
  solver_stream = st;
  dev_info.alloc(sizeof(int) * (kMaxInfo + 64));
  KS_CUDA(cudaMemsetAsync(dev_info.p, 0, sizeof(int) * (kMaxInfo + 64), st));
}
void Ctx::potrf(double* H, int n, int info_slot, cudaStream_t s) {
  ensure_solver();
  SolverApi& api = solver_api();
  if (s != solver2_stream) {
    if (api.SetStream(solver2, s) != CUSOLVER_STATUS_SUCCESS) throw KsError{KS_ERR_SOLVER, "cusolverDnSetStream failed"};
    solver2_stream = s;
  }
  int lwork = 0;
  if (api.DpotrfBufferSize(solver2, CUBLAS_FILL_MODE_LOWER, n, H, n, &lwork) != CUSOLVER_STATUS_SUCCESS)
    throw KsError{KS_ERR_SOLVER, "cusolverDnDpotrf_bufferSize failed"};
  if (lwork > solver_lwork) {
    KS_CUDA(cudaStreamSynchronize(st));
    KS_CUDA(cudaStreamSynchronize(st2));
    KS_CUDA(cudaStreamSynchronize(st3));
    solver_work.alloc(sizeof(double) * static_cast<size_t>(lwork));
    solver_lwork = lwork;
  }
  if (api.Dpotrf(solver2, CUBLAS_FILL_MODE_LOWER, n, H, n, solver_work.as<double>(), solver_lwork,
                 dev_info.as<int>() + (info_slot % kMaxInfo)) != CUSOLVER_STATUS_SUCCESS)
    throw KsError{KS_ERR_SOLVER, "cusolverDnDpotrf failed"};
  launches += 1;
}
void Ctx::potrs(const double* H, int n, double* B, int nrhs, int info_slot, cudaStream_t s) {
  ensure_solver();
  if (nrhs == 0 || n == 0) return;
  if (s != solver_stream) {
    if (solver_api().SetStream(solver, s) != CUSOLVER_STATUS_SUCCESS) throw KsError{KS_ERR_SOLVER, "cusolverDnSetStream failed"};
    solver_stream = s;
  }
  if (solver_api().Dpotrs(solver, CUBLAS_FILL_MODE_LOWER, n, nrhs, H, n, B, n, dev_info.as<int>() + (info_slot % kMaxInfo)) !=
      CUSOLVER_STATUS_SUCCESS)
    throw KsError{KS_ERR_SOLVER, "cusolverDnDpotrs failed"};
  launches += 1;
}
void Ctx::ensure_lanes(int n) {
  ensure_solver();
  SolverApi& api = solver_api();
  int prio_least = 0, prio_greatest = 0;
  KS_CUDA(cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest));
  while (static_cast<int>(lanes.size()) < n) {
    auto ln = std::make_unique<SolveLane>();
    KS_CUDA(cudaStreamCreateWithPriority(&ln->s, cudaStreamNonBlocking, prio_greatest));
    if (api.Create(&ln->h) != CUSOLVER_STATUS_SUCCESS) throw KsError{KS_ERR_SOLVER, "cusolverDnCreate failed"};
    if (api.SetStream(ln->h, ln->s) != CUSOLVER_STATUS_SUCCESS) throw KsError{KS_ERR_SOLVER, "cusolverDnSetStream failed"};
    lanes.push_back(std::move(ln));
  }
}
void Ctx::lane_potrf_potrs(int q, double* H, int n, double* B, int nrhs, int info_slot) {
  SolverApi& api = solver_api();
  SolveLane& ln = *lanes[q];
  int lwork = 0;
  if (api.DpotrfBufferSize(ln.h, CUBLAS_FILL_MODE_LOWER, n, H, n, &lwork) != CUSOLVER_STATUS_SUCCESS)
    throw KsError{KS_ERR_SOLVER, "cusolverDnDpotrf_bufferSize failed"};
  if (lwork > ln.lwork) {
    KS_CUDA(cudaStreamSynchronize(ln.s));
    ln.work.alloc(sizeof(double) * static_cast<size_t>(lwork));
    ln.lwork = lwork;
  }
  int* info = dev_info.as<int>() + (info_slot % kMaxInfo);
  if (api.Dpotrf(ln.h, CUBLAS_FILL_MODE_LOWER, n, H, n, ln.work.as<double>(), ln.lwork, info) != CUSOLVER_STATUS_SUCCESS)
    throw KsError{KS_ERR_SOLVER, "cusolverDnDpotrf failed"};
  // potrs reports only argument errors: it shares a scratch slot past the factorisation statuses
  if (api.Dpotrs(ln.h, CUBLAS_FILL_MODE_LOWER, n, nrhs, H, n, B, n, dev_info.as<int>() + kMaxInfo + q) != CUSOLVER_STATUS_SUCCESS)
    throw KsError{KS_ERR_SOLVER, "cusolverDnDpotrs failed"};
  launches += 2;
}
__global__ void infos_to_flag_kernel(int* info, int used, double* flag) {
  int bad = 0;
  for (int i = 0; i < used; ++i) {
    if (info[i] != 0) ++bad;
    info[i] = 0;
  }
  *flag = static_cast<double>(bad);
}
void Ctx::infos_to_flag(int used, double* flag, cudaStream_t s) {
  ensure_solver();
  infos_to_flag_kernel<<<1, 1, 0, s>>>(dev_info.as<int>(), used, flag);
  launches += 1;
}
void Ctx::check_infos(int used_slots) {
  if (!solver || used_slots <= 0) return;
  if (used_slots > kMaxInfo) used_slots = kMaxInfo;
  std::vector<int> h(used_slots);
  KS_CUDA(cudaMemcpyAsync(h.data(), dev_info.p, sizeof(int) * used_slots, cudaMemcpyDeviceToHost, st));
  KS_CUDA(cudaStreamSynchronize(st));
  KS_CUDA(cudaMemsetAsync(dev_info.p, 0, sizeof(int) * used_slots, st));
  for (int i = 0; i < used_slots; ++i)
    if (h[i] != 0)
      throw KsError{KS_ERR_NOT_SPD, "Cholesky failed (slot " + std::to_string(i) + ", info " + std::to_string(h[i]) +
                                        "): the regularised Gram matrix is not positive definite (lambda too small?)"};
}
void Ctx::check_async(const char* what) {
  cudaError_t e = cudaStreamSynchronize(st);
  if (e == cudaSuccess && st2) e = cudaStreamSynchronize(st2);
  if (e == cudaSuccess && st3) e = cudaStreamSynchronize(st3);
  if (e == cudaSuccess && st4) e = cudaStreamSynchronize(st4);
  if (e == cudaSuccess && st5) e = cudaStreamSynchronize(st5);
  if (e != cudaSuccess) {
    std::string extra;
    if (e == cudaErrorLaunchFailure || e == cudaErrorIllegalInstruction) extra = " (kernel trapped: barrier wait budget exceeded or illegal instruction)";
    throw KsError{KS_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e) + extra};
  }
}

// ------------------------------------------------------------------------------------ feature source
__global__ void combine_scales_kernel(const float* a, const float* b, float* out) { out[0] = a[1] * b[1]; }

// operand copies of X / W for the projection GEMM of generated (cosine) features: tf32-rounded X always; fp16 copies
// (KS_PRECISION_F16) or K-concatenated fp16 hi / lo copies (KS_PRECISION_F16X2) on request.  out.X, out.Wall, out.Wfull,
// out.ldw, out.d_in, out.D, out.n_rows must be set.
void prepare_generated_operands(Ctx& c, FeatSrc& out, int precision) {
  const bool want_f16 = precision == KS_PRECISION_F16, want_x2 = precision == KS_PRECISION_F16X2;
  const int64_t total = out.D;
  out.zeros.alloc(sizeof(float) * static_cast<size_t>(round_up(std::max(out.D, out.d_in), 32) + 32));
  KS_CUDA(cudaMemsetAsync(out.zeros.p, 0, out.zeros.bytes, c.st));
  // GEMM operand copy of X rounded to tf32 (round-to-nearest instead of the MMA's truncation)
  out.xop.alloc(sizeof(float) * static_cast<size_t>(std::max<int64_t>(out.n_rows, 1) * out.X->ld));
  launch_center_round(out.X->d, out.X->ld, 0, out.zeros.as<float>(), out.xop.as<float>(), nullptr, out.X->ld, out.n_rows,
                      static_cast<int>(out.X->cols), c.st);
  c.launches += 1;
  if ((want_f16 && c.proj_f16) || want_x2) {
    // fp16 copies of X and W for the fp16 projection.  Each carries its own power-of-two scale (largest magnitude
    // mapped into [2048, 4096]), so the input units do not matter; the product of the two inverse scales is applied to the
    // fp32 accumulator in the epilogue.  Same 10-bit mantissa as the tf32 operands above.
    out.pscale.alloc(sizeof(float) * 8);  // [0] 1/(sx*sw)  [1] maxbits x  [2] maxbits w  [4,5] x {s, 1/s}  [6,7] w {s, 1/s}
    KS_CUDA(cudaMemsetAsync(out.pscale.p, 0, out.pscale.bytes, c.st));
    float* ps = out.pscale.as<float>();
    unsigned* mb = out.pscale.as<unsigned>();
    launch_max_abs_f32(out.X->d, out.X->ld, out.n_rows, static_cast<int>(out.X->cols), mb + 1, c.st);
    launch_max_abs_f32(out.Wfull, out.ldw, total, static_cast<int>(out.d_in), mb + 2, c.st);
    launch_pow2_scale(mb + 1, 4096.f, ps + 4, c.st);
    launch_pow2_scale(mb + 2, 4096.f, ps + 6, c.st);
    combine_scales_kernel<<<1, 1, 0, c.st>>>(ps + 4, ps + 6, ps);
    if (want_x2) {
      out.ldx3 = out.ldw3 = round_up(3 * out.d_in, 64);
      out.x3.alloc(2 * static_cast<size_t>(std::max<int64_t>(out.n_rows, 1) * out.ldx3));
      out.w3.alloc(2 * static_cast<size_t>(total * out.ldw3));
      launch_split_concat3(out.X->d, out.X->ld, out.n_rows, static_cast<int>(out.d_in), ps + 4, out.x3.p, out.ldx3, 0, c.st);
      launch_split_concat3(out.Wfull, out.ldw, total, static_cast<int>(out.d_in), ps + 6, out.w3.p, out.ldw3, 1, c.st);
      out.proj_x2 = true;
    } else {
      out.xop16.alloc(2 * static_cast<size_t>(std::max<int64_t>(out.n_rows, 1) * out.X->ld));
      out.w16.alloc(2 * static_cast<size_t>(total * out.ldw));
      launch_f32_to_f16_rows(out.X->d, out.X->ld, out.xop16.p, out.X->ld, out.n_rows, out.X->cols, c.st, ps + 4);
      launch_f32_to_f16_rows(out.Wfull, out.ldw, out.w16.p, out.ldw, total, out.d_in, c.st, ps + 6);
      out.proj16 = true;
    }
    c.launches += 7;
  }
}

void make_feat_src(Ctx& c, int64_t features, int64_t x_in, const int64_t* rfs, int32_t n_rfs, FeatSrc& out, int precision) {
  const bool want_f16 = precision == KS_PRECISION_F16, want_x2 = precision == KS_PRECISION_F16X2;
  if (features != 0) {
    if (x_in != 0 || n_rfs != 0) throw KsError{KS_ERR_INVALID, "pass either features or (x_in, rfs), not both"};
    out.F = &c.matrix(features);
    out.D = out.F->cols;
    out.n_rows = out.F->rows;
    out.zeros.alloc(sizeof(float) * static_cast<size_t>(round_up(out.D, 32) + 32));
    KS_CUDA(cudaMemsetAsync(out.zeros.p, 0, out.zeros.bytes, c.st));
    return;
  }
  if (x_in == 0 || n_rfs <= 0 || rfs == nullptr) throw KsError{KS_ERR_INVALID, "no feature source given"};
  out.X = &c.matrix(x_in);
  out.n_rows = out.X->rows;
  out.d_in = out.X->cols;
  int64_t total = 0;
  for (int i = 0; i < n_rfs; ++i) {
    CosRF& r = c.rf(rfs[i]);
    if (r.n_in != out.d_in) throw KsError{KS_ERR_INVALID, "feature map input dimension does not match x_in"};
    if (r.kind != c.rf(rfs[0]).kind || r.rect_floor != c.rf(rfs[0]).rect_floor)
      throw KsError{KS_ERR_INVALID, "gathered feature maps must be of one kind (all cosine, or all rectified with the same maxVal)"};
    total += r.n_out;
  }
  out.kind = c.rf(rfs[0]).kind;
  out.rect_floor = c.rf(rfs[0]).rect_floor;
  out.D = total;
  CosRF& r0 = c.rf(rfs[0]);
  out.ldw = r0.ld;
  const bool need_full = (want_f16 && c.proj_f16) || want_x2;
  if (n_rfs == 1) {
    out.Wall = r0.W;
    out.Wfull = r0.Wfull;
    out.ball = r0.bias;
  } else {  // VectorCombiner: concatenate the gathered feature maps
    out.wcat.alloc(sizeof(float) * static_cast<size_t>(total * out.ldw));
    if (need_full) out.wcat_full.alloc(out.wcat.bytes);
    out.bcat.alloc(sizeof(float) * static_cast<size_t>(total));
    int64_t off = 0;
    for (int i = 0; i < n_rfs; ++i) {
      CosRF& r = c.rf(rfs[i]);
      KS_CUDA(cudaMemcpyAsync(out.wcat.as<float>() + off * out.ldw, r.W, sizeof(float) * r.n_out * r.ld,
                              cudaMemcpyDeviceToDevice, c.st));
      if (need_full)
        KS_CUDA(cudaMemcpyAsync(out.wcat_full.as<float>() + off * out.ldw, r.Wfull, sizeof(float) * r.n_out * r.ld,
                                cudaMemcpyDeviceToDevice, c.st));
      KS_CUDA(cudaMemcpyAsync(out.bcat.as<float>() + off, r.bias, sizeof(float) * r.n_out, cudaMemcpyDeviceToDevice, c.st));
      off += r.n_out;
    }
    out.Wall = out.wcat.as<float>();
    out.Wfull = need_full ? out.wcat_full.as<float>() : nullptr;
    out.ball = out.bcat.as<float>();
  }
  prepare_generated_operands(c, out, precision);
}

static void tmap16_or_throw(CUtensorMap* m, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_cols, int box_rows,
                            int swizzle) {
  const int r = make_tmap_any(m, base, rows, cols, ld, box_cols, box_rows, 2, swizzle);
  if (r != 0)
    throw KsError{KS_ERR_CUDA, "cuTensorMapEncodeTiled (fp16) failed (" + std::to_string(r) + ") rows=" + std::to_string(rows) +
                                   " cols=" + std::to_string(cols) + " ld=" + std::to_string(ld)};
}

static void tmap_or_throw(CUtensorMap* m, const float* base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  const int r = make_tmap_2d(m, base, rows, cols, ld, box_rows);
  if (r != 0)
    throw KsError{KS_ERR_CUDA, "cuTensorMapEncodeTiled failed (" + std::to_string(r) + ") rows=" + std::to_string(rows) +
                                   " cols=" + std::to_string(cols) + " ld=" + std::to_string(ld)};
}

void produce_slab(Ctx& c, FeatSrc& src, int64_t c0, int64_t cols, const float* shift, void* slab_v, int64_t lds,
                  int64_t row_begin, int64_t rows, bool round_out, float* colsum, cudaStream_t st, bool out16, bool x2, void* slab_lo) {
  if (rows <= 0 || cols <= 0) return;
  if (!st) st = c.st;
  float* slab = static_cast<float*>(slab_v);
  if (src.F) {
    if (!round_out || out16 || x2) throw KsError{KS_ERR_INVALID, "unrounded / fp16 slabs only for generated features"};
    launch_center_round(src.F->d + row_begin * src.F->ld, src.F->ld, static_cast<int>(c0), shift, slab, colsum, lds, rows,
                        static_cast<int>(cols), st);
    c.launches += 1;
    return;
  }
  KmLaunch k;
  int64_t kdepth = src.d_in;
  if (x2) {  // split operands concatenated along K: depth 3 d_in, fp32 output, no rounding
    if (!src.proj_x2 || out16 || round_out) throw KsError{KS_ERR_INVALID, "split-operand slab requested without split operands"};
    kdepth = 3 * src.d_in;
    tmap16_or_throw(&k.tmA, static_cast<const uint16_t*>(src.x3.p) + row_begin * src.ldx3, rows, kdepth, src.ldx3, 64, 128, TMAP_SW128);
    tmap16_or_throw(&k.tmB, static_cast<const uint16_t*>(src.w3.p) + c0 * src.ldw3, cols, kdepth, src.ldw3, 64, 128, TMAP_SW128);
    k.f16 = 1;
    k.p.acc_scale_ptr = src.pscale.as<float>();
  } else if (out16 && src.proj16) {  // fp16 operands: 64 K-elements (128 B) per box row
    tmap16_or_throw(&k.tmA, static_cast<const uint16_t*>(src.xop16.p) + row_begin * src.X->ld, rows, src.d_in, src.X->ld, 64, 128,
                    TMAP_SW128);
    tmap16_or_throw(&k.tmB, static_cast<const uint16_t*>(src.w16.p) + c0 * src.ldw, cols, src.d_in, src.ldw, 64, 128, TMAP_SW128);
    k.f16 = 1;
    k.p.acc_scale_ptr = src.pscale.as<float>();
  } else {
    tmap_or_throw(&k.tmA, src.xop.as<float>() + row_begin * src.X->ld, rows, src.d_in, src.X->ld, 128);
    tmap_or_throw(&k.tmB, src.Wall + c0 * src.ldw, cols, src.d_in, src.ldw, 128);
  }
  if (slab_lo && !x2) throw KsError{KS_ERR_INVALID, "a lo plane needs the split operands"};
  if (slab_lo) {  // the epilogue splits the unrounded value into the fp16 pair itself: no fp32 copy of the block, no second pass
    tmap16_or_throw(&k.tmOut, slab_v, rows, cols, lds, 32, 32, TMAP_NONE);
    tmap16_or_throw(&k.tmOut2, slab_lo, rows, cols, lds, 32, 32, TMAP_NONE);
    k.out16 = 2;
  } else {
    if (out16) tmap16_or_throw(&k.tmOut, slab_v, rows, cols, lds, 32, 32, TMAP_NONE);
    else tmap_or_throw(&k.tmOut, slab, rows, cols, lds, 32);
    k.out16 = out16 ? 1 : 0;
  }
  k.p.vec0 = src.ball + c0;
  k.p.vec1 = shift;
  k.p.colsum = colsum;
  k.p.M = static_cast<int>(rows);
  k.p.N = static_cast<int>(cols);
  k.p.K = static_cast<int>(kdepth);
  k.p.flags = (round_out ? 0 : KM_FLAG_NO_ROUND) | (src.kind == 1 ? KM_FLAG_RECT : 0);
  k.p.rect_floor = src.rect_floor;
  k.epi = EPI_COS;
  // the projection kernel is persistent (one CTA per SM for its whole duration); on the look-ahead stream leave a few SMs
  // free so that the critical chain's small kernels (NCCL all-reduce, triangular solves) can always be scheduled
  k.num_sms = (st == c.st2) ? std::max(1, c.num_sms - c.reserve_sms) : c.num_sms;
  if (c.dyn_tiles) k.p.tile_counter = c.next_tile_counter(st);
  KS_CUDA(launch_kmajor(k, st));
  c.launches += 1;
}

const GramTile* gram_tiles(Ctx& c, int b, int kcols, bool with_g, bool with_c, int* num_tiles) {
  std::vector<int> key = {b, kcols, with_g ? 1 : 0, with_c ? 1 : 0};
  auto it = c.tile_cache.find(key);
  std::vector<GramTile> t;
  const int tm = 128, tn = 128;
  const int mb = (b + tm - 1) / tm;
  if (with_g) {
    const int nbk = (b + tn - 1) / tn;
    for (int i = 0; i < mb; ++i)
      for (int j = 0; j < nbk; ++j)
        if ((j + 1) * tn - 1 >= i * tm) t.push_back(GramTile{i, j, 0, 0});  // tile touches the upper triangle
  }
  if (with_c) {
    const int nck = (kcols + tn - 1) / tn;
    for (int i = 0; i < mb; ++i)
      for (int j = 0; j < nck; ++j) t.push_back(GramTile{i, j, 1, 0});
  }
  *num_tiles = static_cast<int>(t.size());
  if (it != c.tile_cache.end()) return it->second->as<GramTile>();
  auto buf = std::make_unique<DevBuf>();
  buf->alloc(sizeof(GramTile) * std::max<size_t>(t.size(), 1));
  KS_CUDA(cudaMemcpyAsync(buf->p, t.data(), sizeof(GramTile) * t.size(), cudaMemcpyHostToDevice, c.st));
  KS_CUDA(cudaStreamSynchronize(c.st));  // t is a stack temporary
  const GramTile* p = buf->as<GramTile>();
  c.tile_cache[key] = std::move(buf);
  return p;
}

void launch_gram_block(Ctx& c, const void* slab, int64_t lds, int64_t rows, int b, const void* R, int64_t ldr, int kcols,
                       float* G, int ldg, float* C, int ldc, bool with_g, bool with_c, cudaStream_t st, bool f16,
                       int64_t chunk_rows, const void* slab_lo, const void* R_lo) {
  if (rows <= 0 || b <= 0 || (!with_g && !with_c)) return;
  if (!st) st = c.st;
  const bool split = slab_lo != nullptr;
  if (split && (!f16 || (with_c && !R_lo))) throw KsError{KS_ERR_INVALID, "split Gram operands must be fp16 pairs"};
  GramLaunch g;
  int nt = 0;
  g.f16 = f16 ? 1 : 0;
  g.split = split ? 1 : 0;
  g.tiles = gram_tiles(c, b, kcols, with_g, with_c, &nt);
  g.num_tiles = nt;
  const int stage_rows = split ? 32 : f16 ? 64 : kGramStageRows;
  if (f16) {  // MN-major fp16 operands: 64-column (128 B) x 64-row boxes (pairs: 32-row), plain 128 B swizzle
    tmap16_or_throw(&g.tmA, slab, rows, b, lds, 64, stage_rows, TMAP_SW128);
    g.tmB0 = g.tmA;
    if (with_c) tmap16_or_throw(&g.tmB1, R, rows, kcols, ldr, 64, stage_rows, TMAP_SW128);
    else g.tmB1 = g.tmA;
    if (split) {  // the G tiles are A^T A: B0 is A again, lo plane included
      tmap16_or_throw(&g.tmAlo, slab_lo, rows, b, lds, 64, stage_rows, TMAP_SW128);
      g.tmB0lo = g.tmAlo;
      if (with_c) tmap16_or_throw(&g.tmB1lo, R_lo, rows, kcols, ldr, 64, stage_rows, TMAP_SW128);
      else g.tmB1lo = g.tmAlo;
    }
  } else {
    tmap_or_throw(&g.tmA, static_cast<const float*>(slab), rows, b, lds, kGramStageRows);
    g.tmB0 = g.tmA;
    if (with_c) tmap_or_throw(&g.tmB1, static_cast<const float*>(R), rows, kcols, ldr, kGramStageRows);
    else g.tmB1 = g.tmA;
  }
  g.rows = static_cast<int>(rows);
  // Rows of the contraction per CTA.  Every chunk ends in a reduce-add of its 128 x 128 partial tile, so long chunks mean
  // less reduce traffic and fewer, longer CTAs next to the critical chain's kernels; short chunks keep enough CTAs per
  // launch to balance the SMs when the rows are sharded (tools/ab_fit.py compares settings).
  int64_t chunk = chunk_rows > 0 ? chunk_rows : c.gram_chunk_rows;
  if (chunk <= 0) chunk = !f16 ? 4096 : rows >= 400000 ? 16384 : rows >= 200000 ? 8192 : 4096;
  chunk = std::max<int64_t>(stage_rows, chunk / stage_rows * stage_rows);
  g.chunk_rows = static_cast<int>(chunk);
  if (with_g) tmap_or_throw(&g.tmOut0, G, b, b, ldg, 32);
  if (with_c) tmap_or_throw(&g.tmOut1, C, b, kcols, ldc, 32);
  if (!with_g) g.tmOut0 = g.tmOut1;
  if (!with_c) g.tmOut1 = g.tmOut0;
  g.n_valid0 = b;
  g.n_valid1 = kcols;
  KS_CUDA(launch_gram(g, st));
  c.launches += 1;
}

void launch_update(Ctx& c, const void* slab, int64_t lds, int64_t rows, int b, const void* bop, int64_t ldb, int k,
                   float* out, int64_t ldo, const float* cbias, int epi, bool reduce, cudaStream_t st, bool f16,
                   const float* acc_scale_ptr, const void* slab_lo, const void* bop_lo) {
  if (rows <= 0 || k <= 0 || b <= 0) return;
  if (!st) st = c.st;
  const bool split = slab_lo != nullptr;
  if (split && (!f16 || !bop_lo || epi != EPI_UPDATE)) throw KsError{KS_ERR_INVALID, "split update operands must be fp16 pairs"};
  KmLaunch u;
  u.f16 = f16 ? 1 : 0;
  u.split = split ? 1 : 0;
  u.p.acc_scale_ptr = acc_scale_ptr;
  if (split) {  // four K-major fp16 planes per stage: 32 K-elements (64 B) x 128 rows per box, 64 B swizzle
    tmap16_or_throw(&u.tmA, slab, rows, b, lds, 32, 128, TMAP_SW64);
    tmap16_or_throw(&u.tmAlo, slab_lo, rows, b, lds, 32, 128, TMAP_SW64);
    tmap16_or_throw(&u.tmB, bop, k, b, ldb, 32, 128, TMAP_SW64);
    tmap16_or_throw(&u.tmBlo, bop_lo, k, b, ldb, 32, 128, TMAP_SW64);
  } else if (f16) {  // K-major fp16 operands: 64 K-elements (128 B) x 128 rows per box
    tmap16_or_throw(&u.tmA, slab, rows, b, lds, 64, 128, TMAP_SW128);
    tmap16_or_throw(&u.tmB, bop, k, b, ldb, 64, 128, TMAP_SW128);
  } else {
    tmap_or_throw(&u.tmA, static_cast<const float*>(slab), rows, b, lds, 128);
    tmap_or_throw(&u.tmB, static_cast<const float*>(bop), k, b, ldb, 128);
  }
  tmap_or_throw(&u.tmOut, out, rows, k, ldo, 32);  // k valid columns: the store never touches columns >= k
  u.p.vec0 = cbias;
  u.p.vec1 = nullptr;
  u.p.colsum = nullptr;
  u.p.M = static_cast<int>(rows);
  u.p.N = k;
  u.p.K = b;
  u.p.flags = reduce ? KM_FLAG_REDUCE : 0;
  u.epi = epi;
  u.num_sms = c.num_sms;
  KS_CUDA(launch_kmajor(u, st));
  c.launches += 1;
}

// ------------------------------------------------------------------------------------ small device helpers
__global__ void scale_f64_to_f32_kernel(const double* src, double scale, float* dst, double* dst64, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const double v = src[i] * scale;
    if (dst) dst[i] = static_cast<float>(v);
    if (dst64) dst64[i] = v;
  }
}
__global__ void set_f64_kernel(double* p, double v) { *p = v; }
void launch_set_f64(double* p, double v, cudaStream_t st) { set_f64_kernel<<<1, 1, 0, st>>>(p, v); }
void launch_scale_f64(const double* src, double scale, float* dst, double* dst64, int n, cudaStream_t st) {
  if (n > 0) scale_f64_to_f32_kernel<<<(n + 255) / 256, 256, 0, st>>>(src, scale, dst, dst64, n);
}
__global__ void sumsq_f64_kernel(const double* p, int64_t n, double* out) {
  double acc = 0;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    acc += p[i] * p[i];
  __shared__ double red[256];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) atomicAdd(out, red[0]);
}

// ------------------------------------------------------------------------------------ BlockLS fit
// Per block j the work splits into a part that does NOT depend on the residual
//   proj(j)   slab S_j = round(features_j - m_j)                       tensor (projection GEMM) or HBM (materialised F)
//   G(j)      G_j = S_j^T S_j, all-reduce                              tensor
//   factor(j) H_j = G_j - N d d^T + lambda I, Cholesky                 fp64, ~100 small latency-bound kernels
// and the residual-dependent chain
//   C(j)      Rr = round(R), C_j = S_j^T Rr, all-reduce                tensor
//   solve(j)  rhs, triangular solves, W_j += dW, pack dW               fp64, ~230 small kernels
//   update(j) R -= S_j dW                                              tensor
//
// pipeline 1 (default): ONE stream carries every tensor-core kernel in the order C(j), G(j+1), proj(j+2), update(j); the
// solve and factor chains run on their own higher-priority streams and hide under G(j+1) + proj(j+2).  Two tensor
// kernels never share the SMs: each is written to own an SM (one CTA, ~200 KB of shared memory), so running two at once
// only splits the machine, thrashes L2 and stretches both.
// pipeline 0: the round-1 arrangement (residual chain on st, look-ahead tensor kernels on st2), kept for A/B runs.
// Slabs, G and H are triple-buffered; cross-stream dependencies are CUDA events; no host synchronisation inside the loop.
static int64_t fit_blockls(Ctx& c, FeatSrc& src, Matrix& Y, int bs, int num_iter, double lam, int64_t nf_opt,
                           int precision = KS_PRECISION_TF32) {
  if (bs <= 0 || num_iter < 1) throw KsError{KS_ERR_INVALID, "blockSize must be > 0 and numIter >= 1"};
  if (Y.rows != src.n_rows) throw KsError{KS_ERR_INVALID, "features and labels have different row counts"};
  const int64_t n_loc = Y.rows;
  const int k = static_cast<int>(Y.cols);
  const int64_t D = nf_opt > 0 ? nf_opt : src.D;
  if (D > src.D) throw KsError{KS_ERR_INVALID, "numFeaturesOpt exceeds the feature dimension"};
  if (D <= 0 || k <= 0) throw KsError{KS_ERR_INVALID, "empty problem"};
  const int nb = static_cast<int>((D + bs - 1) / bs);
  const int bmax = static_cast<int>(std::min<int64_t>(bs, D));
  const int64_t lds = round_up(bmax, 32);
  const int64_t kpad = round_up(k, 32);
  const bool serial = c.pipeline != 0;
  // stream roles (see the Ctx comment)
  cudaStream_t S1 = c.st, S2 = c.st2, S3 = c.st3, S4 = c.st4, S5 = c.st5;
  cudaStream_t ST = S2;                       // projection + G-Gram (both pipelines)
  cudaStream_t SR = serial ? S2 : S1;         // C-Gram and update: the residual chain's tensor kernels
  cudaStream_t SS = S1;                       // solve chain
  cudaStream_t SF = S3;                       // factor chain
  cudaStream_t SG = serial ? S4 : S2;         // all-reduce of G
  ncclComm_t commG = serial ? c.comm3 : c.comm2;
  const auto host_t0 = std::chrono::steady_clock::now();
  c.spans.clear();
  const int64_t launches0 = c.launches;
  auto new_event = [&]() {
    cudaEvent_t e = c.get_event();
    c.fit_events.push_back(e);
    return e;
  };
  cudaEvent_t ev0 = new_event(), ev1 = new_event(), ev_init = new_event();
  KS_CUDA(cudaStreamSynchronize(S2));
  KS_CUDA(cudaStreamSynchronize(S3));
  KS_CUDA(cudaStreamSynchronize(S4));
  KS_CUDA(cudaStreamSynchronize(S5));
  KS_CUDA(cudaEventRecord(ev0, S1));

  // ---- label mean (StandardScaler on labels, BlockLinearMapper.scala:215) + global row count
  DevBuf ysum;  // [k] sums, [k] = local row count
  ysum.alloc(sizeof(double) * (k + 1));
  KS_CUDA(cudaMemsetAsync(ysum.p, 0, ysum.bytes, S1));
  c.span_begin(PH_OTHER);
  launch_colsum(Y.d, nullptr, Y.ld, n_loc, k, ysum.as<double>(), S1);
  c.launches += 1;
  {
    const double nl = static_cast<double>(n_loc);
    KS_CUDA(cudaMemcpyAsync(ysum.as<double>() + k, &nl, sizeof(double), cudaMemcpyHostToDevice, S1));
    KS_CUDA(cudaStreamSynchronize(S1));
  }
  c.allreduce_f64(ysum.as<double>(), k + 1);
  double n_total_d = 0;
  KS_CUDA(cudaMemcpyAsync(&n_total_d, ysum.as<double>() + k, sizeof(double), cudaMemcpyDeviceToHost, S1));
  KS_CUDA(cudaStreamSynchronize(S1));
  if (n_total_d < 1) throw KsError{KS_ERR_INVALID, "no training rows"};
  auto model = std::make_unique<Model>();
  model->block_size = bs;
  model->k = k;
  model->has_mean = true;
  model->has_intercept = true;
  model->intercept.alloc(sizeof(double) * k);
  scale_f64_to_f32_kernel<<<(k + 255) / 256, 256, 0, S1>>>(ysum.as<double>(), 1.0 / n_total_d, nullptr,
                                                          model->intercept.as<double>(), k);
  c.launches += 1;
  auto block_cols = [&](int j, int64_t* c0) {
    *c0 = static_cast<int64_t>(j) * bs;
    return static_cast<int>(std::min<int64_t>(D, *c0 + bs) - *c0);
  };
  for (int j = 0; j < nb; ++j) {
    int64_t c0;
    const int b = block_cols(j, &c0);
    model->brows.push_back(b);
    auto W = std::make_unique<DevBuf>();
    W->alloc(sizeof(double) * static_cast<size_t>(b) * k);
    auto mean = std::make_unique<DevBuf>();
    mean->alloc(sizeof(double) * b);
    model->W.push_back(std::move(W));
    model->mean.push_back(std::move(mean));
  }
  if (c.host_mirror) model_alloc_host(*model);

  // ---- operand modes
  // KS_PRECISION_F16: the slab, the residual operand and the increment operand are fp16 and the three big GEMMs run as
  //   fp16 MMA -- same 10-bit mantissa as tf32 at twice the MMA rate and half the slab bytes.  Only for generated cosine
  //   features (|value| <= 2: no range problem); the residual and the increments are scaled by device-chosen powers of two.
  //   Materialised feature matrices have arbitrary scale and keep the tf32 path.
  // KS_PRECISION_F16X2 (the parity mode): every MMA operand v is carried as hi + lo (hi = round(v), lo = round(v - hi): 21+
  //   significant bits) and every product keeps hi*hi + hi*lo + lo*hi (the projection once, on operands concatenated along
  //   K).  Generated features: fp16 pairs (fp16 MMA); G, C and the update are each one pass of the split kernels, which load
  //   the four planes once and reduce-add once.  Materialised features: tf32 pairs (tf32 MMA, no range limits), three passes
  //   of the single-product kernels, and G keeps the cross Gram S_hi^T S_lo in a second buffer.
  // fp16 slabs only for cosine features (|value| <= 2); rectified linear features have the scale of their input
  const bool x2 = precision == KS_PRECISION_F16X2 && (src.F || src.proj_x2);
  const bool f16 = !src.F && src.kind == 0 && (precision == KS_PRECISION_F16 || x2);
  const size_t es = f16 ? 2 : 4;  // bytes per slab / operand element
  const int64_t x2_chunk = c.split_chunk_rows;  // short accumulation chains: the tensor core's fp32 accumulate truncates
  // fp16 pairs: every product is one pass of the split kernels (G upper tiles only).  tf32 pairs: three passes, and G keeps the
  // full S_hi^T S_lo beside its upper S_hi^T S_hi tiles for launch_build_system.
  const bool g_cross = x2 && !f16;
  // look-ahead of the residual-independent work (projection, G-Gram, factorisation) over the residual chain, in blocks.  With the
  // rows sharded over GPUs the Cholesky of block t+1 (slower next to tensor kernels than alone) sits in a dependency cycle
  // G(t+1) -> factor(t+1) -> solve(t+1) -> update(t+1) -> ... -> G(t+1+LA): a deeper look-ahead spreads it over more blocks.
  const int LA = (serial && (c.pipeline == 1 || c.pipeline == 4)) ? (c.lookahead > 0 ? c.lookahead : (c.world > 1 ? 2 : 1)) : 1;
  const int NBUF = LA + 2;
  // which kernel performs the triangular solves of the critical chain (Ctx::custom_solve)
  const bool custom_solve = c.custom_solve == 1 || (c.custom_solve < 0 && c.world > 1 && c.shard_solve && k >= c.world &&
                                                    (k + c.world - 1) / c.world <= 512);
  DevBuf r_f32, r_op, cm, rhs, rsum, bop, cbias, samp, fsum, scales, sf32, r_lo, bop_lo;
  std::unique_ptr<DevBuf[]> slab_lo;
  std::unique_ptr<DevBuf[]> slab(new DevBuf[NBUF]), gbuf(new DevBuf[NBUF]), Hbuf(new DevBuf[NBUF]), ssum(new DevBuf[NBUF]);
  std::unique_ptr<DevBuf[]> Dbuf(new DevBuf[NBUF]);  // inverted diagonal tiles of the factors (operand of the library's own solve)
  std::unique_ptr<DevBuf[]> dsq(new DevBuf[NBUF]);   // parity mode: exact diagonal of S^T S (fp64), see launch_colsumsq_pair
  r_f32.alloc(sizeof(float) * static_cast<size_t>(std::max<int64_t>(n_loc, 1) * kpad));
  r_op.alloc(f16 ? r_f32.bytes / 2 : r_f32.bytes);
  if (x2) r_lo.alloc(r_op.bytes);
  launch_init_residual(Y.d, Y.ld, model->intercept.as<double>(), r_f32.as<float>(), kpad, n_loc, k, S1);
  c.launches += 1;
  // scales: [0] max|R0| bits, [1] max|dW| bits (per block), then float pairs {2^e, 2^-e}: [2,3] residual, [4,5] increment
  scales.alloc(sizeof(float) * 8);
  unsigned* maxbits = scales.as<unsigned>();
  const float* rscale = scales.as<float>() + 2;
  float* dwscale = scales.as<float>() + 4;
  if (f16) {
    KS_CUDA(cudaMemsetAsync(scales.p, 0, scales.bytes, S1));
    launch_max_abs_f32(r_f32.as<float>(), kpad, n_loc, k, maxbits, S1);
    c.allreduce_max_u32(maxbits, 1);  // every rank must scale its rows of R alike: C is summed over the ranks
    launch_pow2_scale(maxbits, 4096.f, scales.as<float>() + 2, S1);  // 16x headroom below fp16's 65504 for later residuals
    c.launches += 2;
  }
  c.span_end();

  const int ldg = static_cast<int>(lds), ldc = static_cast<int>(kpad);
  const size_t g_elems = static_cast<size_t>(bmax) * ldg, c_elems = static_cast<size_t>(bmax) * ldc;
  const bool cache_factors = num_iter > 1;
  for (int i = 0; i < NBUF; ++i) {
    slab[i].alloc(es * static_cast<size_t>(std::max<int64_t>(n_loc, 1) * lds));
    gbuf[i].alloc(sizeof(float) * g_elems * (g_cross ? 2 : 1));  // S_hi^T S_hi (upper tiles) followed by the full S_hi^T S_lo
    ssum[i].alloc(sizeof(float) * lds);
    if (!cache_factors) Hbuf[i].alloc(sizeof(double) * static_cast<size_t>(bmax) * bmax);
    if (!cache_factors && custom_solve) Dbuf[i].alloc(sizeof(double) * chol_solve_dinv_doubles(bmax));
  }
  cm.alloc(sizeof(float) * c_elems);
  rhs.alloc(sizeof(double) * static_cast<size_t>(bmax) * k);
  rsum.alloc(sizeof(double) * kpad);
  bop.alloc(es * static_cast<size_t>(kpad) * lds);
  if (x2) {
    slab_lo.reset(new DevBuf[NBUF]);
    for (int i = 0; i < NBUF; ++i) slab_lo[i].alloc(slab[i].bytes);
    for (int i = 0; i < NBUF; ++i) dsq[i].alloc(sizeof(double) * lds);
    if (!src.F && !f16)  // tf32 pairs of generated features: unrounded fp32 block before the split (fp16 pairs come out of the epilogue)
      sf32.alloc(sizeof(float) * static_cast<size_t>(std::max<int64_t>(n_loc, 1) * lds));
    bop_lo.alloc(bop.bytes);
  }
  cbias.alloc(sizeof(float) * kpad);
  samp.alloc(sizeof(double) * (bmax + 1));  // sample column sums + sample row count (generated features)
  std::vector<std::unique_ptr<DevBuf>> factors(nb), dinvs(nb), deltas(nb), shifts(nb);

  // ---- exact column means for materialised features (one pass over F for all blocks)
  if (src.F) {
    c.span_begin(PH_FEATURIZE);
    fsum.alloc(sizeof(double) * static_cast<size_t>(src.F->ld));
    KS_CUDA(cudaMemsetAsync(fsum.p, 0, fsum.bytes, S1));
    launch_colsum(src.F->d, nullptr, src.F->ld, n_loc, static_cast<int>(src.F->cols), fsum.as<double>(), S1);
    c.launches += 1;
    c.allreduce_f64(fsum.as<double>(), static_cast<size_t>(src.F->cols));
    c.span_end();
  }
  KS_CUDA(cudaEventRecord(ev_init, S1));
  KS_CUDA(cudaStreamWaitEvent(S2, ev_init, 0));
  KS_CUDA(cudaStreamWaitEvent(S3, ev_init, 0));

  struct Step { int it, j; };
  std::vector<Step> steps;
  for (int it = 0; it < num_iter; ++it)
    for (int j = 0; j < nb; ++j) steps.push_back({it, j});
  const int T = static_cast<int>(steps.size());
  std::vector<cudaEvent_t> ev_slab(T), ev_fact(T), ev_upd(T), ev_gdone(T), ev_g(T), ev_c(T), ev_solved(T);
  for (int t = 0; t < T; ++t) {
    ev_slab[t] = new_event();
    ev_fact[t] = new_event();
    ev_upd[t] = new_event();
    ev_gdone[t] = new_event();
    ev_g[t] = new_event();
    ev_c[t] = new_event();
    ev_solved[t] = new_event();
  }
  int info_slot = 0;
  double flops = 0;
  const bool shard_solve = c.world > 1 && c.shard_solve && k >= c.world;


  // ---------------- proj(t): shift estimate (first sweep) + slab of step t, on ST
  auto do_proj = [&](int t) {
    const int it = steps[t].it, j = steps[t].j, buf = t % NBUF;
    int64_t c0;
    const int b = block_cols(j, &c0);
    c.span_begin(PH_FEATURIZE, ST);
    if (it == 0) {
      shifts[j] = std::make_unique<DevBuf>();
      shifts[j]->alloc(sizeof(float) * lds);
      KS_CUDA(cudaMemsetAsync(shifts[j]->p, 0, shifts[j]->bytes, ST));
      if (src.F) {
        scale_f64_to_f32_kernel<<<(b + 255) / 256, 256, 0, ST>>>(fsum.as<double>() + c0, 1.0 / n_total_d,
                                                                 shifts[j]->as<float>(), nullptr, b);
        c.launches += 1;
      } else {
        // mean estimate from the first sample_rows rows of every rank; exactness is restored by the rank-1 correction
        // with delta below, the estimate only has to be close enough to avoid cancellation
        const int64_t ns = std::min<int64_t>(n_loc, c.sample_rows);
        KS_CUDA(cudaMemsetAsync(samp.p, 0, samp.bytes, ST));
        KS_CUDA(cudaMemsetAsync(ssum[buf].p, 0, ssum[buf].bytes, ST));
        if (x2 && f16) produce_slab(c, src, c0, b, src.zeros.as<float>(), slab[buf].p, lds, 0, ns, /*round_out=*/false,
                                    ssum[buf].as<float>(), ST, false, true, slab_lo[buf].p);
        else if (x2) produce_slab(c, src, c0, b, src.zeros.as<float>(), sf32.p, lds, 0, ns, /*round_out=*/false, ssum[buf].as<float>(), ST,
                                  false, true);
        else produce_slab(c, src, c0, b, src.zeros.as<float>(), slab[buf].p, lds, 0, ns, /*round_out=*/false,
                          ssum[buf].as<float>(), ST, f16);
        launch_f32_to_f64_rows(ssum[buf].as<float>(), lds, samp.as<double>(), bmax, 1, b, ST);  // 1 x b "matrix"
        c.launches += 1;
        set_f64_kernel<<<1, 1, 0, ST>>>(samp.as<double>() + bmax, static_cast<double>(ns));
        c.launches += 1;
        c.allreduce_on(samp.p, static_cast<size_t>(bmax + 1), true, c.comm2, ST);
        launch_divide_by_count(samp.as<double>(), samp.as<double>() + bmax, shifts[j]->as<float>(), nullptr, b, ST);
        c.launches += 1;
        flops += 2.0 * static_cast<double>(ns) * src.d_in * b;
      }
    }
    KS_CUDA(cudaMemsetAsync(ssum[buf].p, 0, ssum[buf].bytes, ST));
    float* cs = it == 0 ? ssum[buf].as<float>() : nullptr;
    if (x2 && src.F) {  // materialised features: tf32 hi / lo planes straight from F
      launch_center_round(src.F->d, src.F->ld, static_cast<int>(c0), shifts[j]->as<float>(), slab[buf].as<float>(), cs, lds, n_loc, b,
                          ST, slab_lo[buf].as<float>());
      c.launches += 1;
    } else if (x2 && f16) {  // fp16 pairs straight out of the projection's epilogue
      produce_slab(c, src, c0, b, shifts[j]->as<float>(), slab[buf].p, lds, 0, n_loc, /*round_out=*/false, cs, ST, false, true,
                   slab_lo[buf].p);
      flops += 4.0 * static_cast<double>(n_loc) * src.d_in * b;  // two extra product terms of the projection
    } else if (x2) {
      produce_slab(c, src, c0, b, shifts[j]->as<float>(), sf32.p, lds, 0, n_loc, /*round_out=*/false, nullptr, ST, false, true);
      launch_center_round(sf32.as<float>(), lds, 0, src.zeros.as<float>(), slab[buf].as<float>(), cs, lds, n_loc, b, ST,
                          slab_lo[buf].as<float>());  // tf32 pairs
      c.launches += 1;
      flops += 4.0 * static_cast<double>(n_loc) * src.d_in * b;  // two extra product terms of the projection
    } else {
      produce_slab(c, src, c0, b, shifts[j]->as<float>(), slab[buf].p, lds, 0, n_loc, true, cs, ST, f16);
    }
    if (!src.F) flops += 2.0 * static_cast<double>(n_loc) * src.d_in * b;
    if (x2 && it == 0) {  // the diagonal of this block's Gram matrix, exactly (the tensor core's is biased low: aux_kernels.cu)
      KS_CUDA(cudaMemsetAsync(dsq[buf].p, 0, dsq[buf].bytes, ST));
      launch_colsumsq_pair(slab[buf].p, slab_lo[buf].p, f16, lds, n_loc, b, dsq[buf].as<double>(), ST);
      c.launches += 1;
    }
    c.span_end(ST);
    KS_CUDA(cudaEventRecord(ev_slab[t], ST));
  };
  // ---------------- gram(t): G of step t on ST, its all-reduce on SG, the factorisation on SF
  auto do_gram = [&](int t) {
    const int it = steps[t].it, j = steps[t].j, buf = t % NBUF;
    int64_t c0;
    const int b = block_cols(j, &c0);
    if (it != 0) {  // later sweeps reuse the cached factor
      KS_CUDA(cudaEventRecord(ev_fact[t], ST));
      return;
    }
    c.span_begin(PH_GRAM, ST);
    KS_CUDA(cudaMemsetAsync(gbuf[buf].p, 0, gbuf[buf].bytes, ST));
    if (x2 && f16) {  // one pass: upper tiles of S_hi^T S_hi + S_lo^T S_hi + S_hi^T S_lo
      launch_gram_block(c, slab[buf].p, lds, n_loc, b, nullptr, 0, 0, gbuf[buf].as<float>(), ldg, nullptr, 0, true, false, ST, f16,
                        x2_chunk, slab_lo[buf].p);
      flops += 4.0 * n_loc * static_cast<double>(b) * b;
    } else if (x2) {  // one launch: upper tiles of S_hi^T S_hi and all tiles of S_hi^T S_lo (the "C" slot with kcols = b)
      launch_gram_block(c, slab[buf].p, lds, n_loc, b, slab_lo[buf].p, lds, b, gbuf[buf].as<float>(), ldg,
                        gbuf[buf].as<float>() + g_elems, ldg, true, true, ST, f16, x2_chunk);
      flops += 4.0 * n_loc * static_cast<double>(b) * b;
    } else {
      launch_gram_block(c, slab[buf].p, lds, n_loc, b, nullptr, 0, 0, gbuf[buf].as<float>(), ldg, nullptr, 0, true, false, ST, f16);
    }
    flops += 2.0 * n_loc * static_cast<double>(b) * b;
    c.span_end(ST);
    KS_CUDA(cudaEventRecord(ev_gdone[t], ST));
    if (c.world > 1) {
      if (SG != ST) KS_CUDA(cudaStreamWaitEvent(SG, ev_gdone[t], 0));
      c.span_begin(PH_ALLREDUCE, SG);
      c.allreduce_on(gbuf[buf].p, g_elems * (g_cross ? 2 : 1), false, commG, SG);
      c.allreduce_on(ssum[buf].p, static_cast<size_t>(b), false, commG, SG);
      if (x2) c.allreduce_on(dsq[buf].p, static_cast<size_t>(b), true, commG, SG);
      c.span_end(SG);
      KS_CUDA(cudaEventRecord(ev_g[t], SG));
    } else {
      KS_CUDA(cudaEventRecord(ev_g[t], ST));
    }
    // ---- factor(t)
    deltas[j] = std::make_unique<DevBuf>();
    deltas[j]->alloc(sizeof(double) * b);
    double* Hj;
    double* Dj = nullptr;
    if (cache_factors) {
      factors[j] = std::make_unique<DevBuf>();
      factors[j]->alloc(sizeof(double) * static_cast<size_t>(b) * b);
      Hj = factors[j]->as<double>();
      if (custom_solve) {
        dinvs[j] = std::make_unique<DevBuf>();
        dinvs[j]->alloc(sizeof(double) * chol_solve_dinv_doubles(b));
        Dj = dinvs[j]->as<double>();
      }
    } else {
      Hj = Hbuf[buf].as<double>();
      if (custom_solve) Dj = Dbuf[buf].as<double>();
    }
    KS_CUDA(cudaStreamWaitEvent(SF, ev_g[t], 0));
    c.span_begin(PH_SOLVE, SF);
    launch_delta_mean(ssum[buf].as<float>(), shifts[j]->as<float>(), n_total_d, deltas[j]->as<double>(), model->mean[j]->as<double>(), b, SF);
    launch_build_system(gbuf[buf].as<float>(), ldg, deltas[j]->as<double>(), n_total_d, lam, Hj, b, SF,
                        g_cross ? gbuf[buf].as<float>() + g_elems : nullptr, x2 ? dsq[buf].as<double>() : nullptr);
    c.launches += 2;
    c.potrf(Hj, b, info_slot++, SF);
    if (Dj) {  // inverses of the factor's 64 x 64 diagonal tiles: the in-tile substitutions of the solve become DMMA products
      KS_CUDA(launch_tri_inv_tiles(Hj, b, Dj, SF));
      c.launches += 1;
    }
    KS_CUDA(cudaMemsetAsync(model->W[j]->p, 0, model->W[j]->bytes, SF));
    c.span_end(SF);
    KS_CUDA(cudaEventRecord(ev_fact[t], SF));
    flops += static_cast<double>(b) * b * b / 3.0;
  };
  // ---------------- cgram(t): operand copy of R + C = S^T R on SR
  auto do_cgram = [&](int t) {
    const int j = steps[t].j, buf = t % NBUF;
    int64_t c0;
    const int b = block_cols(j, &c0);
    c.span_begin(PH_OTHER, SR);
    KS_CUDA(cudaMemsetAsync(cm.p, 0, sizeof(float) * c_elems, SR));
    KS_CUDA(cudaMemsetAsync(rsum.p, 0, rsum.bytes, SR));
    if (f16) launch_round_colsum16(r_f32.as<float>(), r_op.p, kpad, n_loc, k, rsum.as<double>(), rscale, SR, x2 ? r_lo.p : nullptr,
                                   maxbits + 6);   // scales[6]: fp16 overflow flag of the residual operand
    else launch_round_colsum(r_f32.as<float>(), r_op.as<float>(), kpad, n_loc, k, rsum.as<double>(), SR, x2 ? r_lo.as<float>() : nullptr);
    c.launches += 1;
    c.span_end(SR);
    if (SR != ST) KS_CUDA(cudaStreamWaitEvent(SR, ev_slab[t], 0));
    c.span_begin(PH_UPDATE, SR);  // A^T R part of the Gram (accounted with the residual chain)
    if (x2 && f16) {  // one pass: S_hi^T R_hi + S_lo^T R_hi + S_hi^T R_lo
      launch_gram_block(c, slab[buf].p, lds, n_loc, b, r_op.p, kpad, k, nullptr, 0, cm.as<float>(), ldc, false, true, SR, f16,
                        x2_chunk, slab_lo[buf].p, r_lo.p);
      flops += 4.0 * n_loc * static_cast<double>(b) * k;
    } else {
      launch_gram_block(c, slab[buf].p, lds, n_loc, b, r_op.p, kpad, k, nullptr, 0, cm.as<float>(), ldc, false, true, SR, f16,
                        x2 ? x2_chunk : 0);
    }
    if (x2 && !f16) {  // + S_lo^T R_hi + S_hi^T R_lo, reduce-added into the same C
      launch_gram_block(c, slab_lo[buf].p, lds, n_loc, b, r_op.p, kpad, k, nullptr, 0, cm.as<float>(), ldc, false, true, SR, f16,
                        x2_chunk);
      launch_gram_block(c, slab[buf].p, lds, n_loc, b, r_lo.p, kpad, k, nullptr, 0, cm.as<float>(), ldc, false, true, SR, f16,
                        x2_chunk);
      flops += 4.0 * n_loc * static_cast<double>(b) * k;
    }
    flops += 2.0 * n_loc * static_cast<double>(b) * k;
    c.span_end(SR);
    KS_CUDA(cudaEventRecord(ev_c[t], SR));
  };
  // ---------------- solve(t): all-reduce of C, rhs, triangular solves, W += dW, operand of the update, on SS
  auto do_solve = [&](int t) {
    const int it = steps[t].it, j = steps[t].j, buf = t % NBUF;
    int64_t c0;
    const int b = block_cols(j, &c0);
    if (SS != SR) KS_CUDA(cudaStreamWaitEvent(SS, ev_c[t], 0));
    c.span_begin(PH_ALLREDUCE, SS);
    c.allreduce_f32(cm.as<float>(), c_elems);
    c.allreduce_f64(rsum.as<double>(), k);
    c.span_end(SS);
    KS_CUDA(cudaStreamWaitEvent(SS, ev_fact[t], 0));
    c.span_begin(PH_SOLVE, SS);
    double* Hj = cache_factors ? factors[j]->as<double>() : Hbuf[buf].as<double>();
    launch_build_rhs(cm.as<float>(), ldc, deltas[j]->as<double>(), rsum.as<double>(), n_total_d, lam,
                     it > 0 ? model->W[j]->as<double>() : nullptr, rhs.as<double>(), b, k, SS, f16 ? rscale + 1 : nullptr);
    c.launches += 1;
    const double* Dj = !custom_solve ? nullptr : cache_factors ? dinvs[j]->as<double>() : Dbuf[buf].as<double>();
    auto solve_cols = [&](double* cols, int ncols) {  // (L L^T)^-1 on `ncols` right-hand sides, in place
      if (custom_solve) {
        KS_CUDA(launch_chol_solve(Hj, Dj, b, cols, ncols, SS));  // one launch, runs beside the look-ahead Gram (solve_kernels.cu)
        c.launches += 1;
      } else {
        c.potrs(Hj, b, cols, ncols, info_slot++, SS);
      }
    };
    if (shard_solve) {
      // Column-sharded solve: the right-hand sides are independent, so rank r solves columns [k r / world, k (r+1) / world)
      // in place (column-major: a contiguous slice) and one grouped broadcast per rank hands every slice to everybody.
      // All ranks end up with the same bytes, so the model stays bit-identical across ranks.
      auto col0 = [&](int r) { return static_cast<int64_t>(k) * r / c.world; };
      const int64_t m0 = col0(c.rank), m1 = col0(c.rank + 1);
      solve_cols(rhs.as<double>() + m0 * b, static_cast<int>(m1 - m0));
      KS_NCCL(nccl_api().GroupStart());
      for (int r = 0; r < c.world; ++r) {
        double* slice = rhs.as<double>() + col0(r) * b;
        KS_NCCL(nccl_api().Broadcast(slice, slice, static_cast<size_t>(col0(r + 1) - col0(r)) * b, ncclFloat64, r, c.comm, SS));
      }
      KS_NCCL(nccl_api().GroupEnd());
      c.launches += 1;
    } else {
      solve_cols(rhs.as<double>(), k);
    }
    const double* dw_ptr = rhs.as<double>();
    if (f16) {
      KS_CUDA(cudaMemsetAsync(maxbits + 1, 0, sizeof(unsigned), SS));
      launch_max_abs_f64(dw_ptr, static_cast<int64_t>(b) * k, maxbits + 1, SS);
      launch_pow2_scale(maxbits + 1, 8192.f, dwscale, SS);
      launch_pack_update16(dw_ptr, model->W[j]->as<double>(), deltas[j]->as<double>(), bop.p, static_cast<int>(lds),
                           cbias.as<float>(), b, k, static_cast<int>(kpad), dwscale, SS, x2 ? bop_lo.p : nullptr);
      c.launches += 2;
    } else {
      launch_pack_update(dw_ptr, model->W[j]->as<double>(), deltas[j]->as<double>(), bop.as<float>(), x2 ? bop_lo.as<float>() : nullptr,
                         static_cast<int>(lds), cbias.as<float>(), b, k, static_cast<int>(kpad), SS);
    }
    c.launches += 1;
    flops += 2.0 * static_cast<double>(b) * b * k;
    c.span_end(SS);
    KS_CUDA(cudaEventRecord(ev_solved[t], SS));
    if (it == num_iter - 1 && model->host_valid) {  // W_j and mean_j are final: mirror them to the host while the fit goes on
      KS_CUDA(cudaStreamWaitEvent(S5, ev_solved[t], 0));
      model_block_to_host(*model, j, S5);
    }
  };
  // ---------------- update(t): R -= S dW on SR
  auto do_update = [&](int t) {
    const int j = steps[t].j, buf = t % NBUF;
    int64_t c0;
    const int b = block_cols(j, &c0);
    if (SR != SS) KS_CUDA(cudaStreamWaitEvent(SR, ev_solved[t], 0));
    c.span_begin(PH_UPDATE, SR);
    if (x2 && f16) {  // one pass: R -= S_hi dW_hi + S_lo dW_hi + S_hi dW_lo
      launch_update(c, slab[buf].p, lds, n_loc, b, bop.p, lds, k, r_f32.as<float>(), kpad, cbias.as<float>(), EPI_UPDATE,
                    /*reduce=*/true, SR, f16, dwscale + 1, slab_lo[buf].p, bop_lo.p);
      flops += 4.0 * n_loc * static_cast<double>(b) * k;
    } else {
      launch_update(c, slab[buf].p, lds, n_loc, b, bop.p, lds, k, r_f32.as<float>(), kpad, cbias.as<float>(),
                    EPI_UPDATE, /*reduce=*/true, SR, f16, f16 ? dwscale + 1 : nullptr);
    }
    if (x2 && !f16) {  // - S_lo dW_hi - S_hi dW_lo (the constant delta^T dW is applied once, above)
      launch_update(c, slab_lo[buf].p, lds, n_loc, b, bop.p, lds, k, r_f32.as<float>(), kpad, nullptr, EPI_UPDATE, true, SR, f16,
                    f16 ? dwscale + 1 : nullptr);
      launch_update(c, slab[buf].p, lds, n_loc, b, bop_lo.p, lds, k, r_f32.as<float>(), kpad, nullptr, EPI_UPDATE, true, SR, f16,
                    f16 ? dwscale + 1 : nullptr);
      flops += 4.0 * n_loc * static_cast<double>(b) * k;
    }
    flops += 2.0 * n_loc * static_cast<double>(b) * k;
    c.span_end(SR);
    KS_CUDA(cudaEventRecord(ev_upd[t], SR));
  };

  // Enqueue order: a stream-wait on an event that has not been recorded yet counts as complete, so every wait is enqueued
  // after the corresponding record.
  if (serial) {
    // tensor stream (look-ahead LA, LA + 2 buffers): proj(0..LA) G(0..LA-1) | C(t) G(t+LA) update(t) proj(t+LA+1) | ...
    // (slab (t+LA+1) % (LA+2) was last read by update(t-1), G buffer (t+LA) % (LA+2) by factor(t-2): both precede in stream / event order).  The solve of step t runs beside
    // G(t+1): its CTAs fit on the SMs next to Gram CTAs (solve_kernels.cu), not next to the register-heavy projection kernel,
    // which therefore comes after the update (pipeline = 2 puts it before, for A/B runs).
    for (int t = 0; t < std::min(T, LA + 1); ++t) do_proj(t);
    for (int t = 0; t < std::min(T, LA); ++t) do_gram(t);
    for (int t = 0; t < T; ++t) {
      do_cgram(t);
      do_solve(t);
      if (c.pipeline == 1) {  // C(t), G(t+LA), update(t), proj(t+LA+1): the solve of step t runs beside G(t+LA)
        if (t + LA < T) do_gram(t + LA);
        do_update(t);
        if (t + LA + 1 < T) do_proj(t + LA + 1);
        continue;
      }
      if (c.pipeline == 4) {  // C(t), update(t), G(t+LA), proj(t+LA+1): the tensor stream waits for the solve; nothing shares the
        do_update(t);         // GPU with it except the factor chain of the block ahead
        if (t + LA < T) do_gram(t + LA);
        if (t + LA + 1 < T) do_proj(t + LA + 1);
        continue;
      }
      if (c.pipeline == 3) {  // the solve runs beside the projection (persistent kernel that leaves reserve_sms SMs free)
        if (t + 2 < T) do_proj(t + 2);
        do_update(t);
        if (t + 1 < T) do_gram(t + 1);
        continue;
      }
      if (t + 1 < T) do_gram(t + 1);
      if (c.pipeline == 2 && t + 2 < T) do_proj(t + 2);
      do_update(t);
      if (c.pipeline != 2 && t + 2 < T) do_proj(t + 2);
    }
  } else {
    // proj(t) after update(t - NBUF) released its buffers; G + factor of step t+1 after the chain of step t was enqueued
    for (int t = 0; t < std::min(T, NBUF - 1); ++t) do_proj(t);
    do_gram(0);
    for (int t = 0; t < T; ++t) {
      do_cgram(t);
      do_solve(t);
      do_update(t);
      if (t + 1 < T) do_gram(t + 1);
      if (t + NBUF - 1 < T) {
        if (t >= 1) KS_CUDA(cudaStreamWaitEvent(ST, ev_upd[t - 1], 0));  // step t-1 was the last reader of that slab buffer
        do_proj(t + NBUF - 1);
      }
    }
  }
  KS_CUDA(cudaStreamWaitEvent(S1, ev_upd[T - 1], 0));
  KS_CUDA(cudaStreamWaitEvent(S1, ev_fact[T - 1], 0));
  if (model->host_valid) {
    model_intercept_to_host(*model, S5);
    cudaEvent_t ev_copy = new_event();
    KS_CUDA(cudaEventRecord(ev_copy, S5));
    KS_CUDA(cudaStreamWaitEvent(S1, ev_copy, 0));  // total_ms ends with the whole model on the host
  }
  KS_CUDA(cudaEventRecord(ev1, S1));
  c.check_async("BlockLeastSquaresEstimator.fit");
  c.check_infos(info_slot);
  if (f16) {  // collective by construction: every rank scales alike, but only some may overflow -> all-reduce the flag first
    c.allreduce_max_u32(maxbits + 6, 1);
    unsigned ovf = 0;
    KS_CUDA(cudaMemcpyAsync(&ovf, maxbits + 6, sizeof(unsigned), cudaMemcpyDeviceToHost, S1));
    KS_CUDA(cudaStreamSynchronize(S1));
    if (ovf)
      throw KsError{KS_ERR_INVALID, "the residual left fp16's range during the fit (it grew more than 16x over the centred labels): "
                                    "use KS_PRECISION_TF32 for this problem"};
  }
  float total_ms = 0;
  cudaEventElapsedTime(&total_ms, ev0, ev1);
  double ms[PH_COUNT];
  c.timeline_origin = getenv("KS_TIMELINE") ? ev0 : nullptr;
  c.collect_spans(ms);
  c.timeline_origin = nullptr;
  if (getenv("KS_TIMELINE")) {
    FILE* f = fopen((std::string(getenv("KS_TIMELINE")) + "." + std::to_string(c.rank)).c_str(), "w");
    if (f) { fputs(c.timeline_json.c_str(), f); fclose(f); }
  }
  for (cudaEvent_t e : c.fit_events) c.event_pool.push_back(e);
  c.fit_events.clear();
  std::ostringstream js;
  js << "{\"solver\":\"blockls\",\"n_local\":" << n_loc << ",\"n_total\":" << static_cast<int64_t>(n_total_d) << ",\"d\":" << D
     << ",\"k\":" << k << ",\"block_size\":" << bs << ",\"num_blocks\":" << nb << ",\"num_iter\":" << num_iter
     << ",\"world\":" << c.world << ",\"total_ms\":" << total_ms << ",\"featurize_ms\":" << ms[PH_FEATURIZE]
     << ",\"gram_ms\":" << ms[PH_GRAM] << ",\"allreduce_ms\":" << ms[PH_ALLREDUCE] << ",\"solve_ms\":" << ms[PH_SOLVE]
     << ",\"update_ms\":" << ms[PH_UPDATE] << ",\"other_ms\":" << ms[PH_OTHER] << ",\"local_flops\":" << flops
     << ",\"launches\":" << (c.launches - launches0) << ",\"mma\":\"" << (x2 ? (f16 ? "f16x2" : "tf32x2") : f16 ? "f16" : "tf32x1")
     << "\",\"pipeline\":" << c.pipeline << ",\"lookahead\":" << LA << ",\"host_mirror\":" << (model->host_valid ? 1 : 0) << ",\"solve\":\""
     << (custom_solve ? "dmma-kernel" : "potrs") << (shard_solve ? "-column-sharded" : "") << "\",\"host_ms\":"
     << std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count() << "}";
  c.stats_json = js.str();
  return c.add(std::move(model));
}

// ------------------------------------------------------------------------------------ apply
std::unique_ptr<Matrix> new_matrix(int64_t rows, int64_t cols) {
  auto m = std::make_unique<Matrix>();
  m->rows = rows;
  m->cols = cols;
  m->ld = round_up(std::max<int64_t>(cols, 1), kPadCols);
  m->buf.alloc(sizeof(float) * static_cast<size_t>(std::max<int64_t>(rows, 1) * m->ld));
  m->d = m->buf.as<float>();
  return m;
}

// BlockLinearMapper.apply.  precision KS_PRECISION_F16X2 (the context default): slab and weights are carried as tf32 hi + lo
// pairs and every block costs three GEMMs (hi*hi + lo*hi + hi*lo); otherwise one tf32 GEMM per block.
static std::unique_ptr<Matrix> apply_model(Ctx& c, Model& md, FeatSrc& src, int last_block, bool use_means, int precision) {
  const int nb = static_cast<int>(md.brows.size());
  if (last_block < 0 || last_block >= nb) last_block = nb - 1;
  int64_t dsum = 0;
  for (auto r : md.brows) dsum += r;
  if (dsum > src.D) throw KsError{KS_ERR_INVALID, "model has more features than the input"};
  const int k = static_cast<int>(md.k);
  const int64_t n_loc = src.n_rows;
  auto out = new_matrix(n_loc, k);
  KS_CUDA(cudaMemsetAsync(out->d, 0, out->buf.bytes, c.st));
  int bmax = 0;
  for (auto r : md.brows) bmax = std::max<int>(bmax, static_cast<int>(r));
  const int64_t lds = round_up(std::max(bmax, 1), 32);
  const int64_t kpad = round_up(k, 32);
  const bool x2 = precision == KS_PRECISION_F16X2 && (src.F || src.proj_x2);
  DevBuf slab, slab_lo, sf32, bop, bop_lo, cbias, shift;
  const size_t slab_bytes = sizeof(float) * static_cast<size_t>(std::max<int64_t>(n_loc, 1) * lds);
  slab.alloc(slab_bytes);
  bop.alloc(sizeof(float) * static_cast<size_t>(kpad) * lds);
  if (x2) {
    slab_lo.alloc(slab_bytes);
    bop_lo.alloc(bop.bytes);
    if (!src.F) sf32.alloc(slab_bytes);
  }
  cbias.alloc(sizeof(float) * kpad);
  shift.alloc(sizeof(float) * lds);
  int64_t c0 = 0;
  for (int j = 0; j <= last_block; ++j) {
    const int b = static_cast<int>(md.brows[j]);
    KS_CUDA(cudaMemsetAsync(shift.p, 0, shift.bytes, c.st));
    if (use_means && md.has_mean) {
      launch_f64_to_f32_vec(md.mean[j]->as<double>(), shift.as<float>(), b, c.st);
      c.launches += 1;
    }
    if (x2 && src.F) {
      launch_center_round(src.F->d, src.F->ld, static_cast<int>(c0), shift.as<float>(), slab.as<float>(), nullptr, lds, n_loc, b, c.st,
                          slab_lo.as<float>());
      c.launches += 1;
    } else if (x2) {
      produce_slab(c, src, c0, b, shift.as<float>(), sf32.p, lds, 0, n_loc, /*round_out=*/false, nullptr, c.st, false, true);
      launch_center_round(sf32.as<float>(), lds, 0, src.zeros.as<float>(), slab.as<float>(), nullptr, lds, n_loc, b, c.st,
                          slab_lo.as<float>());
      c.launches += 1;
    } else {
      produce_slab(c, src, c0, b, shift.as<float>(), slab.as<float>(), lds, 0, n_loc);
    }
    // the fp32 rounding of the mean is compensated in the bias: cbias = intercept - (mean - fp32(mean)) . W
    launch_pack_apply(md.W[j]->as<double>(), (use_means && md.has_mean) ? md.mean[j]->as<double>() : nullptr, shift.as<float>(),
                      (j == 0 && md.has_intercept) ? md.intercept.as<double>() : nullptr, bop.as<float>(),
                      x2 ? bop_lo.as<float>() : nullptr, static_cast<int>(lds), cbias.as<float>(), b, k, static_cast<int>(kpad), c.st);
    c.launches += 1;
    launch_update(c, slab.as<float>(), lds, n_loc, b, bop.as<float>(), lds, k, out->d, out->ld, cbias.as<float>(), EPI_APPLY,
                  /*reduce=*/j > 0);
    if (x2) {
      launch_update(c, slab_lo.as<float>(), lds, n_loc, b, bop.as<float>(), lds, k, out->d, out->ld, nullptr, EPI_APPLY, true);
      launch_update(c, slab.as<float>(), lds, n_loc, b, bop_lo.as<float>(), lds, k, out->d, out->ld, nullptr, EPI_APPLY, true);
    }
    c0 += md.block_size;
  }
  c.check_async("BlockLinearMapper.apply");
  return out;
}

}  // namespace ks

// ======================================================================================= C ABI
using namespace ks;

static std::mutex g_mu;
static std::unordered_map<int64_t, std::unique_ptr<Ctx>> g_ctxs;
static int64_t g_next_ctx = 1;
static thread_local std::string g_global_err;

static Ctx* find_ctx(int64_t h) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_ctxs.find(h);
  return it == g_ctxs.end() ? nullptr : it->second.get();
}

// An exception that unwinds a fit returns its workspace to the memory pool while kernels that use it may still be queued on
// the context's streams.  Nothing may be handed out of the pool before those have drained: wait for the whole device
// (the context is single-threaded, so no allocation can have happened in between), then recycle the fit's events.
static void after_error(Ctx& c) {
  cudaDeviceSynchronize();
  cudaGetLastError();
  for (cudaEvent_t e : c.fit_events) c.event_pool.push_back(e);
  c.fit_events.clear();
  for (auto& sp : c.spans) {
    c.event_pool.push_back(sp.a);
    c.event_pool.push_back(sp.b);
  }
  c.spans.clear();
}

template <class Fn>
static int32_t guard(int64_t ctx, Fn&& fn) {
  Ctx* c = find_ctx(ctx);
  if (!c) {
    g_global_err = "unknown context handle " + std::to_string(ctx);
    return KS_ERR_HANDLE;
  }
  try {
    cudaError_t e = cudaSetDevice(c->device);
    if (e != cudaSuccess) throw KsError{KS_ERR_CUDA, std::string("cudaSetDevice: ") + cudaGetErrorString(e)};
    fn(*c);
    return KS_OK;
  } catch (const KsError& e) {
    c->err = e.msg;
    after_error(*c);
    return e.code;
  } catch (const std::exception& e) {
    c->err = std::string("exception: ") + e.what();
    after_error(*c);
    return KS_ERR_INVALID;
  }
}

extern "C" {

KS_API int32_t ks_version(void) { return 100; }

KS_API int32_t ks_nccl_unique_id(uint8_t* out_id) {
  try {
    if (!out_id) throw KsError{KS_ERR_INVALID, "null out_id"};
    static_assert(sizeof(ncclUniqueId) == KS_NCCL_ID_BYTES, "ncclUniqueId size");
    ncclUniqueId id;
    ncclResult_t r = nccl_api().GetUniqueId(&id);
    if (r != ncclSuccess) throw KsError{KS_ERR_NCCL, std::string("ncclGetUniqueId: ") + nccl_api().GetErrorString(r)};
    memcpy(out_id, &id, KS_NCCL_ID_BYTES);
    return KS_OK;
  } catch (const KsError& e) {
    g_global_err = e.msg;
    return e.code;
  }
}

KS_API int32_t ks_ctx_create(int32_t device_id, int32_t rank, int32_t world_size, const uint8_t* nccl_id, int64_t* out_ctx) {
  try {
    if (!out_ctx || world_size < 1 || rank < 0 || rank >= world_size) throw KsError{KS_ERR_INVALID, "bad arguments"};
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
      cudaGetLastError();
      throw KsError{KS_ERR_NO_DEVICE, "no CUDA device: keystone_b200 has no CPU fallback"};
    }
    if (device_id < 0 || device_id >= ndev) throw KsError{KS_ERR_INVALID, "device_id out of range"};
    KS_CUDA(cudaSetDevice(device_id));
    cudaDeviceProp prop;
    KS_CUDA(cudaGetDeviceProperties(&prop, device_id));
    if (prop.major != 9 || prop.minor != 0)
      throw KsError{KS_ERR_NO_DEVICE, std::string("device is sm_") + std::to_string(prop.major) + std::to_string(prop.minor) + "; this library contains sm_90a code only"};
    auto c = std::make_unique<Ctx>();
    c->device = device_id;
    c->rank = rank;
    c->world = world_size;
    c->num_sms = prop.multiProcessorCount;
    // stream priorities: the residual-dependent chain (st) is the critical path of the pipelined fit and mostly small
    // kernels (NCCL, triangular solves); it must not queue behind the look-ahead tensor work of st2
    int prio_least = 0, prio_greatest = 0;
    KS_CUDA(cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest));
    const int prio_mid = (prio_greatest < prio_least) ? prio_greatest + 1 : prio_greatest;
    KS_CUDA(cudaStreamCreateWithPriority(&c->st, cudaStreamNonBlocking, prio_greatest));
    if (const char* e = getenv("KS_GRAM_CHUNK_ROWS")) {
      const long v = atol(e);
      if (v >= kGramStageRows) c->gram_chunk_rows = v;
    }
    if (const char* e = getenv("KS_SHARD_SOLVE")) c->shard_solve = atoi(e) != 0;
    if (const char* e = getenv("KS_PROJ_F16")) c->proj_f16 = atoi(e) != 0;
    if (const char* e = getenv("KS_PRECISION"))
      c->precision = (atoi(e) == 1 || !strcmp(e, "f16")) ? KS_PRECISION_F16 : (atoi(e) == 2 || !strcmp(e, "f16x2") || !strcmp(e, "parity")) ? KS_PRECISION_F16X2 : KS_PRECISION_TF32;
    if (const char* e = getenv("KS_CUSTOM_SOLVE")) c->custom_solve = std::max(-1, std::min(1, atoi(e)));
    if (const char* e = getenv("KS_RESERVE_SMS")) c->reserve_sms = std::max(0, std::min(140, atoi(e)));
    if (const char* e = getenv("KS_PIPELINE")) c->pipeline = std::max(0, std::min(4, atoi(e)));
    if (const char* e = getenv("KS_HOST_MIRROR")) c->host_mirror = atoi(e) != 0;
    if (const char* e = getenv("KS_LOOKAHEAD")) c->lookahead = std::max(0, std::min(6, atoi(e)));
    KS_CUDA(cudaStreamCreateWithPriority(&c->st2, cudaStreamNonBlocking, prio_least));
    KS_CUDA(cudaStreamCreateWithPriority(&c->st3, cudaStreamNonBlocking, prio_mid));
    KS_CUDA(cudaStreamCreateWithPriority(&c->st4, cudaStreamNonBlocking, prio_mid));
    KS_CUDA(cudaStreamCreateWithPriority(&c->st5, cudaStreamNonBlocking, prio_mid));
    if (world_size > 1) {
      if (!nccl_id) throw KsError{KS_ERR_INVALID, "nccl_id required for world_size > 1"};
      ncclUniqueId id;
      memcpy(&id, nccl_id, KS_NCCL_ID_BYTES);
      KS_NCCL(nccl_api().CommInitRank(&c->comm, world_size, id, rank));
      c->comm2 = c->comm;
      c->comm3 = c->comm;
      if (nccl_api().CommSplit) {  // one communicator per stream so that collectives of different streams never interleave
        ncclComm_t c2 = nullptr, c3 = nullptr;
        if (nccl_api().CommSplit(c->comm, 0, rank, &c2, nullptr) == ncclSuccess && c2) c->comm2 = c2;
        if (nccl_api().CommSplit(c->comm, 0, rank, &c3, nullptr) == ncclSuccess && c3) c->comm3 = c3;
      }
    }
    std::lock_guard<std::mutex> lk(g_mu);
    const int64_t h = g_next_ctx++;
    g_ctxs[h] = std::move(c);
    *out_ctx = h;
    return KS_OK;
  } catch (const KsError& e) {
    g_global_err = e.msg;
    return e.code;
  }
}

KS_API int32_t ks_ctx_destroy(int64_t ctx) {
  std::unique_ptr<Ctx> c;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_ctxs.find(ctx);
    if (it == g_ctxs.end()) return KS_ERR_HANDLE;
    c = std::move(it->second);
    g_ctxs.erase(it);
  }
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->st);
  if (c->st2) cudaStreamSynchronize(c->st2);
  if (c->st3) cudaStreamSynchronize(c->st3);
  if (c->st4) cudaStreamSynchronize(c->st4);
  if (c->st5) cudaStreamSynchronize(c->st5);
  c->matrices.clear();
  c->rfs.clear();
  c->models.clear();
  c->kernels.clear();
  c->convs.clear();
  c->tile_cache.clear();
  for (auto e : c->event_pool) cudaEventDestroy(e);
  for (auto& ln : c->lanes) {
    if (ln->s) cudaStreamSynchronize(ln->s);
    if (ln->h) solver_api().Destroy(ln->h);
    ln->work.release();
    if (ln->s) cudaStreamDestroy(ln->s);
  }
  c->lanes.clear();
  if (c->solver) solver_api().Destroy(c->solver);
  if (c->solver2) solver_api().Destroy(c->solver2);
  if (c->comm3 && c->comm3 != c->comm) nccl_api().CommDestroy(c->comm3);
  if (c->comm2 && c->comm2 != c->comm) nccl_api().CommDestroy(c->comm2);
  if (c->comm) nccl_api().CommDestroy(c->comm);
  c->solver_work.release();
  c->dev_info.release();
  c->tile_counters.release();
  cudaStreamDestroy(c->st);
  if (c->st2) cudaStreamDestroy(c->st2);
  if (c->st3) cudaStreamDestroy(c->st3);
  if (c->st4) cudaStreamDestroy(c->st4);
  if (c->st5) cudaStreamDestroy(c->st5);
  c.reset();
  bool last;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    last = g_ctxs.empty();
  }
  if (last) {
    pool_release_all();
    host_pool_release_all();
  }
  return KS_OK;
}

KS_API const char* ks_last_error(int64_t ctx) {
  Ctx* c = find_ctx(ctx);
  return c ? c->err.c_str() : g_global_err.c_str();
}

KS_API int32_t ks_ctx_synchronize(int64_t ctx) {
  return guard(ctx, [&](Ctx& c) { c.check_async("synchronize"); });
}

KS_API int32_t ks_ctx_set_option(int64_t ctx, const char* name, int64_t value) {
  return guard(ctx, [&](Ctx& c) {
    const std::string n = name ? name : "";
    if (n == "gram_chunk_rows" && (value == 0 || value >= kGramStageRows)) c.gram_chunk_rows = value;
    else if (n == "split_chunk_rows" && value >= kGramStageRows && value % kGramStageRows == 0) c.split_chunk_rows = value;
    else if (n == "sample_rows" && value >= 1) c.sample_rows = value;
    else if (n == "shard_solve") c.shard_solve = value != 0;
    else if (n == "proj_f16") c.proj_f16 = value != 0;
    else if (n == "precision" && (value == KS_PRECISION_TF32 || value == KS_PRECISION_F16 || value == KS_PRECISION_F16X2)) c.precision = static_cast<int>(value);
    else if (n == "custom_solve" && value >= -1 && value <= 1) c.custom_solve = static_cast<int>(value);
    else if (n == "reserve_sms" && value >= 0 && value < c.num_sms) c.reserve_sms = static_cast<int>(value);
    else if (n == "pipeline" && value >= 0 && value <= 4) c.pipeline = static_cast<int>(value);
    else if (n == "dyn_tiles") c.dyn_tiles = value != 0;
    else if (n == "lookahead" && value >= 0 && value <= 6) c.lookahead = static_cast<int>(value);
    else if (n == "solve_lanes" && value >= 1 && value <= 16) c.solve_lanes = static_cast<int>(value);
    else if (n == "host_mirror") c.host_mirror = value != 0;
    else if (n == "timing") c.timing = value != 0;
    else throw KsError{KS_ERR_INVALID, "unknown option or bad value: " + n};
  });
}

KS_API int32_t ks_ctx_launch_count(int64_t ctx, int64_t* out_count) {
  return guard(ctx, [&](Ctx& c) { *out_count = c.launches; });
}

// ---------------------------------------------------------------- matrices
static void upload_rows(Ctx& c, Matrix& m, const void* host, int64_t ld, bool is_f64) {
  if (m.rows == 0) return;
  const size_t esz = is_f64 ? sizeof(double) : sizeof(float);
  if (!is_f64 && ld == m.cols && m.ld == m.cols) {  // same layout on both sides: one 1-D copy
    KS_CUDA(cudaMemcpyAsync(m.d, host, esz * static_cast<size_t>(m.rows * m.cols), cudaMemcpyHostToDevice, c.st));
    KS_CUDA(cudaStreamSynchronize(c.st));
    return;
  }
  // Dense chunks of rows land in two alternating staging buffers by 1-D copies (2-D only when the host rows are themselves
  // strided); a device kernel converts / re-pitches each chunk and zeroes the padding columns.  Everything is ordered on one
  // stream, so a staging buffer is rewritten only after the kernel that read it; one synchronize at the end.
  const int64_t chunk_rows =
      std::min(m.rows, std::max<int64_t>(1, (int64_t(128) << 20) / static_cast<int64_t>(esz * std::max<int64_t>(m.cols, 1))));
  DevBuf stage[2];
  for (auto& sb : stage) sb.alloc(esz * static_cast<size_t>(chunk_rows * m.cols));
  const char* h = static_cast<const char*>(host);
  int which = 0;
  for (int64_t r0 = 0; r0 < m.rows; r0 += chunk_rows, which ^= 1) {
    const int64_t nr = std::min(chunk_rows, m.rows - r0);
    const char* src = h + static_cast<size_t>(r0 * ld) * esz;
    if (ld == m.cols)
      KS_CUDA(cudaMemcpyAsync(stage[which].p, src, esz * static_cast<size_t>(nr * m.cols), cudaMemcpyHostToDevice, c.st));
    else
      KS_CUDA(cudaMemcpy2DAsync(stage[which].p, esz * m.cols, src, esz * ld, esz * m.cols, nr, cudaMemcpyHostToDevice, c.st));
    if (is_f64) launch_f64_to_f32_rows(stage[which].as<double>(), m.cols, m.d + r0 * m.ld, m.ld, nr, m.cols, c.st);
    else launch_f32_repitch_rows(stage[which].as<float>(), m.cols, m.d + r0 * m.ld, m.ld, nr, m.cols, c.st);
    c.launches += 1;
  }
  KS_CUDA(cudaStreamSynchronize(c.st));
}

KS_API int32_t ks_matrix_from_host_f64(int64_t ctx, const double* rowmajor, int64_t n_rows, int64_t n_cols, int64_t ld, int64_t* out_m) {
  return guard(ctx, [&](Ctx& c) {
    if (n_rows < 0 || n_cols <= 0 || ld < n_cols || (!rowmajor && n_rows > 0) || !out_m) throw KsError{KS_ERR_INVALID, "bad matrix arguments"};
    auto m = new_matrix(n_rows, n_cols);
    upload_rows(c, *m, rowmajor, ld, true);
    *out_m = c.add(std::move(m));
  });
}
KS_API int32_t ks_matrix_from_host_f32(int64_t ctx, const float* rowmajor, int64_t n_rows, int64_t n_cols, int64_t ld, int64_t* out_m) {
  return guard(ctx, [&](Ctx& c) {
    if (n_rows < 0 || n_cols <= 0 || ld < n_cols || (!rowmajor && n_rows > 0) || !out_m) throw KsError{KS_ERR_INVALID, "bad matrix arguments"};
    auto m = new_matrix(n_rows, n_cols);
    upload_rows(c, *m, rowmajor, ld, false);
    *out_m = c.add(std::move(m));
  });
}
// An empty (zero) matrix that is then filled by row ranges: the shape a Spark executor needs to upload the rows of its
// partitions one partition at a time (mapPartitionsWithIndex) without first concatenating them on the JVM heap.
KS_API int32_t ks_matrix_create(int64_t ctx, int64_t n_rows, int64_t n_cols, int64_t* out_m) {
  return guard(ctx, [&](Ctx& c) {
    if (n_rows < 0 || n_cols <= 0 || !out_m) throw KsError{KS_ERR_INVALID, "bad matrix arguments"};
    auto m = new_matrix(n_rows, n_cols);
    KS_CUDA(cudaMemsetAsync(m->d, 0, m->buf.bytes, c.st));
    KS_CUDA(cudaStreamSynchronize(c.st));
    *out_m = c.add(std::move(m));
  });
}
static void write_rows(Ctx& c, Matrix& m, int64_t row0, const void* host, int64_t n, int64_t ld, bool is_f64) {
  if (row0 < 0 || n < 0 || row0 + n > m.rows || ld < m.cols || (!host && n > 0)) throw KsError{KS_ERR_INVALID, "bad row range"};
  if (n == 0) return;
  Matrix view;  // a window onto rows [row0, row0 + n) of m (borrowed pointer: view.buf stays empty)
  view.d = m.d + row0 * m.ld;
  view.rows = n;
  view.cols = m.cols;
  view.ld = m.ld;
  upload_rows(c, view, host, ld, is_f64);  // padding columns of the window are rewritten with zeros, as they already were
}
KS_API int32_t ks_matrix_write_rows_f64(int64_t ctx, int64_t m, int64_t row0, const double* rowmajor, int64_t n_rows, int64_t ld) {
  return guard(ctx, [&](Ctx& c) { write_rows(c, c.matrix(m), row0, rowmajor, n_rows, ld, true); });
}
KS_API int32_t ks_matrix_write_rows_f32(int64_t ctx, int64_t m, int64_t row0, const float* rowmajor, int64_t n_rows, int64_t ld) {
  return guard(ctx, [&](Ctx& c) { write_rows(c, c.matrix(m), row0, rowmajor, n_rows, ld, false); });
}
KS_API int32_t ks_matrix_synthetic_normal(int64_t ctx, int64_t n_rows, int64_t n_cols, uint64_t seed, int64_t global_row_offset,
                                   double mean, double stddev, int64_t* out_m) {
  return guard(ctx, [&](Ctx& c) {
    if (n_rows < 0 || n_cols <= 0 || !out_m) throw KsError{KS_ERR_INVALID, "bad matrix arguments"};
    auto m = new_matrix(n_rows, n_cols);
    launch_normal_f32(m->d, m->ld, n_rows, static_cast<int>(n_cols), seed, global_row_offset, static_cast<float>(mean),
                      static_cast<float>(stddev), c.st);
    c.launches += 1;
    c.check_async("synthetic_normal");
    *out_m = c.add(std::move(m));
  });
}
KS_API int32_t ks_labels_from_classes(int64_t ctx, const int32_t* classes, int64_t n_rows, int32_t num_classes, int64_t* out_m) {
  return guard(ctx, [&](Ctx& c) {
    if (n_rows < 0 || num_classes <= 0 || (!classes && n_rows > 0) || !out_m) throw KsError{KS_ERR_INVALID, "bad label arguments"};
    for (int64_t i = 0; i < n_rows; ++i)
      if (classes[i] < 0 || classes[i] >= num_classes) throw KsError{KS_ERR_INVALID, "class index out of range at row " + std::to_string(i)};
    auto m = new_matrix(n_rows, num_classes);
    DevBuf cls;
    cls.alloc(sizeof(int32_t) * static_cast<size_t>(std::max<int64_t>(n_rows, 1)));
    KS_CUDA(cudaMemcpyAsync(cls.p, classes, sizeof(int32_t) * n_rows, cudaMemcpyHostToDevice, c.st));
    launch_labels_from_classes(cls.as<int32_t>(), m->d, m->ld, n_rows, num_classes, c.st);
    c.launches += 1;
    c.check_async("labels_from_classes");
    *out_m = c.add(std::move(m));
  });
}
KS_API int32_t ks_matrix_shape(int64_t ctx, int64_t m, int64_t* n_rows, int64_t* n_cols) {
  return guard(ctx, [&](Ctx& c) {
    Matrix& mm = c.matrix(m);
    if (n_rows) *n_rows = mm.rows;
    if (n_cols) *n_cols = mm.cols;
  });
}
KS_API int32_t ks_matrix_to_host_f32(int64_t ctx, int64_t m, float* out, int64_t ld) {
  return guard(ctx, [&](Ctx& c) {
    Matrix& mm = c.matrix(m);
    if (!out || ld < mm.cols) throw KsError{KS_ERR_INVALID, "bad output buffer"};
    if (mm.rows == 0) return;
    KS_CUDA(cudaMemcpy2DAsync(out, sizeof(float) * ld, mm.d, sizeof(float) * mm.ld, sizeof(float) * mm.cols, mm.rows,
                              cudaMemcpyDeviceToHost, c.st));
    c.check_async("matrix_to_host_f32");
  });
}
KS_API int32_t ks_matrix_to_host_f64(int64_t ctx, int64_t m, double* out, int64_t ld) {
  return guard(ctx, [&](Ctx& c) {
    Matrix& mm = c.matrix(m);
    if (!out || ld < mm.cols) throw KsError{KS_ERR_INVALID, "bad output buffer"};
    if (mm.rows == 0) return;
    const int64_t chunk_rows = std::max<int64_t>(1, (int64_t(256) << 20) / (8 * mm.cols));
    DevBuf stage;
    stage.alloc(sizeof(double) * static_cast<size_t>(std::min(chunk_rows, mm.rows) * mm.cols));
    for (int64_t r0 = 0; r0 < mm.rows; r0 += chunk_rows) {
      const int64_t nr = std::min(chunk_rows, mm.rows - r0);
      launch_f32_to_f64_rows(mm.d + r0 * mm.ld, mm.ld, stage.as<double>(), mm.cols, nr, mm.cols, c.st);
      c.launches += 1;
      KS_CUDA(cudaMemcpy2DAsync(out + r0 * ld, sizeof(double) * ld, stage.p, sizeof(double) * mm.cols, sizeof(double) * mm.cols, nr,
                                cudaMemcpyDeviceToHost, c.st));
      KS_CUDA(cudaStreamSynchronize(c.st));
    }
  });
}
KS_API int32_t ks_matrix_destroy(int64_t ctx, int64_t m) {
  return guard(ctx, [&](Ctx& c) {
    if (!c.matrices.erase(m)) throw KsError{KS_ERR_HANDLE, "unknown matrix handle"};
  });
}

// ---------------------------------------------------------------- CosineRandomFeatures
KS_API int32_t ks_cosine_rf_create(int64_t ctx, const double* W_colmajor, const double* b, int64_t n_out, int64_t n_in, int64_t* out_rf) {
  return guard(ctx, [&](Ctx& c) {
    if (!W_colmajor || !b || n_out <= 0 || n_in <= 0 || !out_rf) throw KsError{KS_ERR_INVALID, "bad CosineRandomFeatures arguments"};
    auto r = std::make_unique<CosRF>();
    r->n_out = n_out;
    r->n_in = n_in;
    r->ld = round_up(n_in, kPadCols);
    r->wbuf.alloc(sizeof(float) * static_cast<size_t>(n_out * r->ld));
    r->bbuf.alloc(sizeof(float) * static_cast<size_t>(n_out));
    r->wfbuf.alloc(r->wbuf.bytes);
    r->W = r->wbuf.as<float>();
    r->Wfull = r->wfbuf.as<float>();
    r->bias = r->bbuf.as<float>();
    DevBuf stage;
    stage.alloc(sizeof(double) * static_cast<size_t>(n_out * n_in + n_out));
    KS_CUDA(cudaMemcpyAsync(stage.p, W_colmajor, sizeof(double) * n_out * n_in, cudaMemcpyHostToDevice, c.st));
    KS_CUDA(cudaMemcpyAsync(stage.as<double>() + n_out * n_in, b, sizeof(double) * n_out, cudaMemcpyHostToDevice, c.st));
    launch_w_to_operand(stage.as<double>(), n_out, n_in, r->W, r->ld, c.st);
    launch_w_to_operand(stage.as<double>(), n_out, n_in, r->Wfull, r->ld, c.st, /*round=*/false);
    launch_f64_to_f32_vec(stage.as<double>() + n_out * n_in, r->bias, n_out, c.st);
    c.launches += 2;
    c.check_async("cosine_rf_create");
    const int64_t id = c.next_id++;
    c.rfs[id] = std::move(r);
    *out_rf = id;
  });
}
// RandomSignNode -> PaddedFFT [-> LinearRectifier] as ONE dense feature map (the real part of the FFT of a sign-flipped,
// zero-padded real vector is a fixed cosine-matrix product): usable wherever a CosineRandomFeatures handle is.
KS_API int32_t ks_padded_fft_create(int64_t ctx, const double* signs_or_null, int64_t n_in, int32_t rectify, double max_val,
                                    double alpha, int64_t* out_rf) {
  return guard(ctx, [&](Ctx& c) {
    if (n_in <= 0 || !out_rf) throw KsError{KS_ERR_INVALID, "bad PaddedFFT arguments"};
    int64_t P = 1;
    while (P < n_in) P <<= 1;   // nextPositivePowerOfTwo (PaddedFFT.scala:20)
    if (P < 2) P = 2;
    auto r = std::make_unique<CosRF>();
    r->n_out = P / 2;
    r->n_in = n_in;
    r->ld = round_up(n_in, kPadCols);
    r->kind = 1;
    r->rect_floor = rectify ? static_cast<float>(max_val) : -INFINITY;
    r->wbuf.alloc(sizeof(float) * static_cast<size_t>(r->n_out * r->ld));
    r->wfbuf.alloc(r->wbuf.bytes);
    r->bbuf.alloc(sizeof(float) * static_cast<size_t>(r->n_out));
    r->W = r->wbuf.as<float>();
    r->Wfull = r->wfbuf.as<float>();
    r->bias = r->bbuf.as<float>();
    DevBuf sg;
    if (signs_or_null) {
      sg.alloc(sizeof(double) * static_cast<size_t>(n_in));
      KS_CUDA(cudaMemcpyAsync(sg.p, signs_or_null, sizeof(double) * n_in, cudaMemcpyHostToDevice, c.st));
    }
    launch_fft_real_matrix(signs_or_null ? sg.as<double>() : nullptr, n_in, P, r->W, r->Wfull, r->ld, c.st);
    launch_fill_f32(r->bias, r->n_out, rectify ? static_cast<float>(alpha) : 0.f, c.st);
    c.launches += 2;
    c.check_async("padded_fft_create");
    const int64_t id = c.next_id++;
    c.rfs[id] = std::move(r);
    *out_rf = id;
  });
}
// out = x .* colvec (op 0: RandomSignNode on a batch) or max(a, x - b) (op 1: LinearRectifier on a batch), as a new matrix
KS_API int32_t ks_matrix_map(int64_t ctx, int64_t m, int32_t op, const double* colvec_or_null, double a, double b, int64_t* out_m) {
  return guard(ctx, [&](Ctx& c) {
    Matrix& in = c.matrix(m);
    if (!out_m || (op != 0 && op != 1) || (op == 0 && !colvec_or_null)) throw KsError{KS_ERR_INVALID, "bad matrix_map arguments"};
    auto out = new_matrix(in.rows, in.cols);
    DevBuf cv64, cv32;
    if (op == 0) {
      cv64.alloc(sizeof(double) * static_cast<size_t>(in.cols));
      cv32.alloc(sizeof(float) * static_cast<size_t>(in.cols));
      KS_CUDA(cudaMemcpyAsync(cv64.p, colvec_or_null, sizeof(double) * in.cols, cudaMemcpyHostToDevice, c.st));
      launch_f64_to_f32_vec(cv64.as<double>(), cv32.as<float>(), in.cols, c.st);
    }
    launch_matrix_map(in.d, out->d, in.ld, in.rows, static_cast<int>(in.cols), op, cv32.as<float>(), static_cast<float>(a),
                      static_cast<float>(b), c.st);
    c.launches += 2;
    c.check_async("matrix_map");
    *out_m = c.add(std::move(out));
  });
}
// ---------------------------------------------------------------- Convolver / SymmetricRectifier / Pooler (CIFAR random-patch featurizer)
KS_API int32_t ks_convolver_create(int64_t ctx, const double* filters_colmajor, int32_t n_filters, int32_t x_dim, int32_t y_dim,
                                   int32_t channels, int32_t conv_size, const double* whitener_means_or_null, int32_t normalize_patches,
                                   double var_constant, int64_t* out_conv) {
  return guard(ctx, [&](Ctx& c) {
    const int pd = conv_size * conv_size * channels;
    if (!filters_colmajor || n_filters <= 0 || x_dim < conv_size || y_dim < conv_size || channels <= 0 || conv_size <= 0 || pd > 256 ||
        static_cast<int64_t>(x_dim) * y_dim * channels > 12288 || !out_conv)
      throw KsError{KS_ERR_INVALID, "bad Convolver arguments (patch dimension <= 256, image <= 12288 values)"};
    auto cv = std::make_unique<ConvPool>();
    cv->x_dim = x_dim; cv->y_dim = y_dim; cv->ch = channels; cv->conv = conv_size; cv->n_filters = n_filters;
    cv->normalize = normalize_patches ? 1 : 0;
    cv->var_constant = static_cast<float>(var_constant);
    cv->pd = pd;
    cv->ld1 = round_up(pd, 64);
    cv->ld3 = round_up(3 * pd, 64);
    // filters: DenseMatrix (n_filters x pd) column-major fp64 -> fp32 row-major [n_filters][ldf] (unrounded) -> scaled fp16 operands
    const int64_t ldf = round_up(pd, kPadCols);
    DevBuf stage, f32;
    stage.alloc(sizeof(double) * static_cast<size_t>(n_filters) * pd);
    f32.alloc(sizeof(float) * static_cast<size_t>(n_filters) * ldf);
    KS_CUDA(cudaMemcpyAsync(stage.p, filters_colmajor, sizeof(double) * static_cast<size_t>(n_filters) * pd, cudaMemcpyHostToDevice, c.st));
    launch_w_to_operand(stage.as<double>(), n_filters, pd, f32.as<float>(), ldf, c.st, /*round=*/false);
    cv->wscale.alloc(sizeof(float) * 8);   // [1] max bits, [2,3] {2^e, 2^-e}
    KS_CUDA(cudaMemsetAsync(cv->wscale.p, 0, cv->wscale.bytes, c.st));
    launch_max_abs_f32(f32.as<float>(), ldf, n_filters, pd, cv->wscale.as<unsigned>() + 1, c.st);
    launch_pow2_scale(cv->wscale.as<unsigned>() + 1, 4096.f, cv->wscale.as<float>() + 2, c.st);
    cv->w16.alloc(2 * static_cast<size_t>(n_filters) * cv->ld1);
    cv->w3.alloc(2 * static_cast<size_t>(n_filters) * cv->ld3);
    launch_f32_to_f16_rows(f32.as<float>(), ldf, cv->w16.p, cv->ld1, n_filters, pd, c.st, cv->wscale.as<float>() + 2);
    launch_split_concat3(f32.as<float>(), ldf, n_filters, pd, cv->wscale.as<float>() + 2, cv->w3.p, cv->ld3, 1, c.st);
    if (whitener_means_or_null) {
      DevBuf m64;
      m64.alloc(sizeof(double) * pd);
      cv->wmeans.alloc(sizeof(float) * pd);
      KS_CUDA(cudaMemcpyAsync(m64.p, whitener_means_or_null, sizeof(double) * pd, cudaMemcpyHostToDevice, c.st));
      launch_f64_to_f32_vec(m64.as<double>(), cv->wmeans.as<float>(), pd, c.st);
      cv->has_means = true;
      c.check_async("convolver_create");
    }
    c.launches += 6;
    c.check_async("convolver_create");
    const int64_t id = c.next_id++;
    c.convs[id] = std::move(cv);
    *out_conv = id;
  });
}
KS_API int32_t ks_convolver_destroy(int64_t ctx, int64_t conv) {
  return guard(ctx, [&](Ctx& c) {
    if (!c.convs.erase(conv)) throw KsError{KS_ERR_HANDLE, "unknown Convolver handle"};
  });
}
// images: (n x x_dim*y_dim*channels) matrix in ImageVectorizer order (c + x*C + y*C*x_dim, K/utils/images/Image.scala:47-65).
// pool_size == 0: Convolver.apply alone -> (n x resW*resH*n_filters), the convolved images in the same vectorised order.
// pool_size  > 0: Convolver andThen SymmetricRectifier(max_val, alpha) andThen Pooler(stride, pool_size, identity, sum) andThen
//                 ImageVectorizer, fused -> (n x nPoolsX*nPoolsY*2*n_filters); the convolved maps never reach HBM.
// Operands: fp16 (context precision F16 / TF32) or split fp16 pairs concatenated along K (F16X2, the default).
KS_API int32_t ks_convolver_apply(int64_t ctx, int64_t conv, int64_t images, int32_t pool_stride, int32_t pool_size, double max_val,
                                  double alpha, int64_t* out_features) {
  return guard(ctx, [&](Ctx& c) {
    if (!out_features) throw KsError{KS_ERR_INVALID, "null output"};
    auto it = c.convs.find(conv);
    if (it == c.convs.end()) throw KsError{KS_ERR_HANDLE, "unknown Convolver handle"};
    ConvPool& cv = *it->second;
    Matrix& im = c.matrix(images);
    if (im.cols != static_cast<int64_t>(cv.x_dim) * cv.y_dim * cv.ch) throw KsError{KS_ERR_INVALID, "image size does not match the Convolver"};
    const int rw = cv.x_dim - cv.conv + 1, rh = cv.y_dim - cv.conv + 1, ppi = rw * rh;
    const bool pooled = pool_size > 0;
    int npx = 0, npy = 0;
    std::vector<unsigned> mask(ppi, 0u);
    if (pooled) {
      if (pool_stride <= 0) throw KsError{KS_ERR_INVALID, "bad pool stride"};
      const int s0 = pool_size / 2;                                   // Pooler.scala:27, :36-37
      npx = (rw - s0 + pool_stride - 1) / pool_stride;
      npy = (rh - s0 + pool_stride - 1) / pool_stride;
      if (npx <= 0 || npy <= 0 || npx * npy > 16) throw KsError{KS_ERR_INVALID, "Pooler geometry unsupported (1..16 pools per image)"};
      for (int px = 0; px < npx; ++px)
        for (int py = 0; py < npy; ++py) {
          const int cx = s0 + px * pool_stride, cy = s0 + py * pool_stride;
          for (int x = cx - pool_size / 2; x < std::min(cx + pool_size / 2, rw); ++x)
            for (int y = cy - pool_size / 2; y < std::min(cy + pool_size / 2, rh); ++y) mask[x + y * rw] |= 1u << (px + py * npx);
        }
    }
    const bool x2 = c.precision == KS_PRECISION_F16X2;
    const int64_t ldp = x2 ? cv.ld3 : cv.ld1;
    const int kdepth = x2 ? 3 * cv.pd : cv.pd;
    const int64_t out_cols = pooled ? static_cast<int64_t>(npx) * npy * 2 * cv.n_filters : static_cast<int64_t>(ppi) * cv.n_filters;
    auto out = new_matrix(im.rows, out_cols);
    KS_CUDA(cudaMemsetAsync(out->d, 0, out->buf.bytes, c.st));
    DevBuf maskd, patches;
    maskd.alloc(sizeof(unsigned) * ppi);
    KS_CUDA(cudaMemcpyAsync(maskd.p, mask.data(), sizeof(unsigned) * ppi, cudaMemcpyHostToDevice, c.st));
    // image chunks bound the patch matrix (ppi * ldp * 2 B per image) to ~4 GB
    const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(im.rows, (int64_t(4) << 30) / (static_cast<int64_t>(ppi) * ldp * 2)));
    patches.alloc(2 * static_cast<size_t>(chunk) * ppi * ldp);
    for (int64_t i0 = 0; i0 < im.rows; i0 += chunk) {
      const int64_t ni = std::min(chunk, im.rows - i0);
      launch_im2col_normalize(im.d + i0 * im.ld, im.ld, ni, cv.x_dim, cv.y_dim, cv.ch, cv.conv, cv.normalize, cv.var_constant,
                              cv.has_means ? cv.wmeans.as<float>() : nullptr, patches.p, ldp, x2 ? 1 : 0, c.st);
      KmLaunch k;
      const int64_t m_rows = ni * ppi;
      tmap16_or_throw(&k.tmA, patches.p, m_rows, kdepth, ldp, 64, 128, TMAP_SW128);
      tmap16_or_throw(&k.tmB, x2 ? cv.w3.p : cv.w16.p, cv.n_filters, kdepth, ldp, 64, 128, TMAP_SW128);
      k.f16 = 1;
      k.p.acc_scale_ptr = cv.wscale.as<float>() + 3;      // 2^-e of the filter scale
      k.p.M = static_cast<int>(m_rows);
      k.p.N = cv.n_filters;
      k.p.K = kdepth;
      k.p.vec0 = nullptr;
      k.p.vec1 = nullptr;
      k.p.colsum = nullptr;
      k.num_sms = c.num_sms;
      if (c.dyn_tiles) k.p.tile_counter = c.next_tile_counter(c.st);
      if (pooled) {
        k.epi = EPI_POOL;
        k.p.flags = 0;
        k.p.pool_mask = maskd.as<unsigned>();
        k.p.pool_out = out->d + i0 * out->ld;
        k.p.pool_out_ld = out->ld;
        k.p.patches_per_image = ppi;
        k.p.n_pools = npx * npy;
        k.p.pool_alpha = static_cast<float>(alpha);
        k.p.rect_floor = static_cast<float>(max_val);
        tmap_or_throw(&k.tmOut, out->d, im.rows, std::min<int64_t>(out_cols, 32), out->ld, 32);  // unused by this epilogue
      } else {
        // the convolved image of image i is rows [i * ppi, (i+1) * ppi) x n_filters of the product: view the output as that matrix
        k.epi = EPI_APPLY;
        k.p.flags = 0;
        if (out->ld != out_cols) throw KsError{KS_ERR_INVALID, "Convolver.apply alone needs resW*resH*n_filters to be a multiple of 32"};
        tmap_or_throw(&k.tmOut, out->d + i0 * out->ld, m_rows, cv.n_filters, cv.n_filters, 32);
      }
      KS_CUDA(launch_kmajor(k, c.st));
      c.launches += 2;
      KS_CUDA(cudaStreamSynchronize(c.st));   // the patch buffer is reused by the next chunk
    }
    c.check_async("Convolver.apply");
    *out_features = c.add(std::move(out));
  });
}

KS_API int32_t ks_cosine_rf_apply(int64_t ctx, int64_t rf, int64_t x_in, int64_t* out_features) {
  return guard(ctx, [&](Ctx& c) {
    if (!out_features) throw KsError{KS_ERR_INVALID, "null output"};
    FeatSrc src;
    make_feat_src(c, 0, x_in, &rf, 1, src, c.precision);
    auto out = new_matrix(src.n_rows, src.D);
    KS_CUDA(cudaMemsetAsync(out->d, 0, out->buf.bytes, c.st));
    // parity mode: split fp16 projection operands (hi*hi + lo*hi + hi*lo in one GEMM of depth 3 d_in); else tf32 operands
    produce_slab(c, src, 0, src.D, src.zeros.as<float>(), out->d, out->ld, 0, src.n_rows, /*round_out=*/false, nullptr, nullptr, false,
                 src.proj_x2);
    c.check_async("CosineRandomFeatures.apply");
    *out_features = c.add(std::move(out));
  });
}
KS_API int32_t ks_cosine_rf_destroy(int64_t ctx, int64_t rf) {
  return guard(ctx, [&](Ctx& c) {
    if (!c.rfs.erase(rf)) throw KsError{KS_ERR_HANDLE, "unknown CosineRandomFeatures handle"};
  });
}

// ---------------------------------------------------------------- estimators
// the per-call precision_mode is authoritative; KS_PRECISION_DEFAULT means "the context's setting" (option "precision")
static int resolve_precision(Ctx& c, int32_t precision_mode) {
  if (precision_mode == KS_PRECISION_DEFAULT) return c.precision;
  if (precision_mode != KS_PRECISION_TF32 && precision_mode != KS_PRECISION_F16 && precision_mode != KS_PRECISION_F16X2)
    throw KsError{KS_ERR_INVALID, "unsupported precision_mode"};
  return precision_mode;
}
KS_API int32_t ks_blockls_fit(int64_t ctx, int64_t features, int64_t x_in, const int64_t* rfs, int32_t n_rfs, int64_t labels,
                       int32_t block_size, int32_t num_iter, double lambda, int64_t num_features_or_0, int32_t precision_mode,
                       int64_t* out_model) {
  return guard(ctx, [&](Ctx& c) {
    if (!out_model) throw KsError{KS_ERR_INVALID, "null out_model"};
    const int prec = resolve_precision(c, precision_mode);
    FeatSrc src;
    make_feat_src(c, features, x_in, rfs, n_rfs, src, prec);
    *out_model = fit_blockls(c, src, c.matrix(labels), block_size, num_iter, lambda, num_features_or_0, prec);
  });
}

KS_API int32_t ks_blockwls_fit(int64_t ctx, int64_t features, int64_t x_in, const int64_t* rfs, int32_t n_rfs, int64_t labels,
                        int32_t block_size, int32_t num_iter, double lambda, double mixture_weight, int64_t num_features_or_0,
                        int32_t precision_mode, int64_t* out_model) {
  return guard(ctx, [&](Ctx& c) {
    if (!out_model) throw KsError{KS_ERR_INVALID, "null out_model"};
    const int prec = resolve_precision(c, precision_mode);
    FeatSrc src;
    make_feat_src(c, features, x_in, rfs, n_rfs, src, prec);
    *out_model = fit_bwls(c, src, c.matrix(labels), block_size, num_iter, lambda, mixture_weight, num_features_or_0, prec);
  });
}

KS_API int32_t ks_lbfgs_fit(int64_t ctx, int64_t features, int64_t x_in, const int64_t* rfs, int32_t n_rfs, int64_t labels,
                            int32_t fit_intercept, int32_t num_corrections, double convergence_tol, int32_t num_iterations,
                            double reg_param, int32_t precision_mode, int64_t* out_model) {
  return guard(ctx, [&](Ctx& c) {
    if (!out_model) throw KsError{KS_ERR_INVALID, "null out_model"};
    const int prec = resolve_precision(c, precision_mode);
    FeatSrc src;
    make_feat_src(c, features, x_in, rfs, n_rfs, src, prec);
    *out_model = fit_lbfgs(c, src, c.matrix(labels), fit_intercept != 0, num_corrections, convergence_tol, num_iterations, reg_param,
                           prec);
  });
}

KS_API int32_t ks_linear_map_fit(int64_t ctx, int64_t features, int64_t labels, int32_t has_lambda, double lambda, int64_t* out_model) {
  return guard(ctx, [&](Ctx& c) {
    if (!out_model) throw KsError{KS_ERR_INVALID, "null out_model"};
    FeatSrc src;
    make_feat_src(c, features, 0, nullptr, 0, src);
    // one block spanning every feature, one pass: exactly (A^T A [+ lambda I]) \ A^T y on centred data; the operand mode is the
    // context's ("precision" option; the default is the split-operand parity mode)
    *out_model = fit_blockls(c, src, c.matrix(labels), static_cast<int>(src.D), 1, has_lambda ? lambda : 0.0, 0, c.precision);
  });
}

// ---------------------------------------------------------------- models
KS_API int32_t ks_model_from_host(int64_t ctx, const double* const* xs, const int64_t* block_rows, int32_t n_blocks, int64_t k,
                           const double* b_or_null, const double* const* means_or_null, int32_t block_size, int64_t* out_model) {
  return guard(ctx, [&](Ctx& c) {
    if (!xs || !block_rows || n_blocks <= 0 || k <= 0 || block_size <= 0 || !out_model) throw KsError{KS_ERR_INVALID, "bad model arguments"};
    auto m = std::make_unique<Model>();
    m->block_size = block_size;
    m->k = k;
    m->has_mean = means_or_null != nullptr;
    m->has_intercept = b_or_null != nullptr;
    for (int j = 0; j < n_blocks; ++j) {
      const int64_t b = block_rows[j];
      if (b <= 0 || b > block_size) throw KsError{KS_ERR_INVALID, "block_rows out of range"};
      auto W = std::make_unique<DevBuf>();
      W->alloc(sizeof(double) * static_cast<size_t>(b * k));
      KS_CUDA(cudaMemcpyAsync(W->p, xs[j], sizeof(double) * b * k, cudaMemcpyHostToDevice, c.st));
      m->W.push_back(std::move(W));
      m->brows.push_back(b);
      if (m->has_mean) {
        auto mu = std::make_unique<DevBuf>();
        mu->alloc(sizeof(double) * static_cast<size_t>(b));
        KS_CUDA(cudaMemcpyAsync(mu->p, means_or_null[j], sizeof(double) * b, cudaMemcpyHostToDevice, c.st));
        m->mean.push_back(std::move(mu));
      }
    }
    m->intercept.alloc(sizeof(double) * static_cast<size_t>(k));
    if (b_or_null) KS_CUDA(cudaMemcpyAsync(m->intercept.p, b_or_null, sizeof(double) * k, cudaMemcpyHostToDevice, c.st));
    KS_CUDA(cudaStreamSynchronize(c.st));
    *out_model = c.add(std::move(m));
  });
}
KS_API int32_t ks_model_num_blocks(int64_t ctx, int64_t model, int32_t* n_blocks, int64_t* k, int32_t* block_size) {
  return guard(ctx, [&](Ctx& c) {
    Model& m = c.model(model);
    if (n_blocks) *n_blocks = static_cast<int32_t>(m.brows.size());
    if (k) *k = m.k;
    if (block_size) *block_size = m.block_size;
  });
}
KS_API int32_t ks_model_block_rows(int64_t ctx, int64_t model, int32_t j, int64_t* rows) {
  return guard(ctx, [&](Ctx& c) {
    Model& m = c.model(model);
    if (j < 0 || j >= static_cast<int>(m.brows.size()) || !rows) throw KsError{KS_ERR_INVALID, "block index out of range"};
    *rows = m.brows[j];
  });
}
KS_API int32_t ks_model_get_block(int64_t ctx, int64_t model, int32_t j, double* W_out, double* mean_out, int32_t* has_mean) {
  return guard(ctx, [&](Ctx& c) {
    Model& m = c.model(model);
    if (j < 0 || j >= static_cast<int>(m.brows.size())) throw KsError{KS_ERR_INVALID, "block index out of range"};
    if (has_mean) *has_mean = m.has_mean ? 1 : 0;
    if (m.host_valid) {  // the fit already mirrored the block into pinned host memory
      const uint8_t* h = static_cast<const uint8_t*>(m.host.p);
      if (W_out) memcpy(W_out, h + m.host_w_off[j], sizeof(double) * m.brows[j] * m.k);
      if (mean_out && m.has_mean) memcpy(mean_out, h + m.host_mean_off[j], sizeof(double) * m.brows[j]);
      return;
    }
    if (W_out) KS_CUDA(cudaMemcpyAsync(W_out, m.W[j]->p, sizeof(double) * m.brows[j] * m.k, cudaMemcpyDeviceToHost, c.st));
    if (mean_out && m.has_mean) KS_CUDA(cudaMemcpyAsync(mean_out, m.mean[j]->p, sizeof(double) * m.brows[j], cudaMemcpyDeviceToHost, c.st));
    KS_CUDA(cudaStreamSynchronize(c.st));
  });
}
static void ensure_host_mirror(Ctx& c, Model& m) {
  if (m.host_valid) return;
  model_alloc_host(m);
  for (int q = 0; q < static_cast<int>(m.brows.size()); ++q) model_block_to_host(m, q, c.st);
  model_intercept_to_host(m, c.st);
  KS_CUDA(cudaStreamSynchronize(c.st));
}
KS_API int32_t ks_model_host_view(int64_t ctx, int64_t model, int32_t j, const double** W_ptr, const double** mean_ptr,
                                  const double** intercept_ptr) {
  return guard(ctx, [&](Ctx& c) {
    Model& m = c.model(model);
    if (j < 0 || j >= static_cast<int>(m.brows.size())) throw KsError{KS_ERR_INVALID, "block index out of range"};
    ensure_host_mirror(c, m);  // models that were not fitted with the mirror on (or came from the host): mirror now
    const uint8_t* h = static_cast<const uint8_t*>(m.host.p);
    if (W_ptr) *W_ptr = reinterpret_cast<const double*>(h + m.host_w_off[j]);
    if (mean_ptr) *mean_ptr = m.has_mean ? reinterpret_cast<const double*>(h + m.host_mean_off[j]) : nullptr;
    if (intercept_ptr) *intercept_ptr = m.has_intercept ? reinterpret_cast<const double*>(h + m.host_b_off) : nullptr;
  });
}
// KernelBlockLinearMapper: applied to raw input rows (features) only
static std::unique_ptr<Matrix> apply_kernel_model(Ctx& c, Model& m, int64_t features, int64_t x_in, int32_t n_rfs) {
  if (x_in != 0 || n_rfs != 0 || features == 0)
    throw KsError{KS_ERR_INVALID, "a kernel model is applied to raw input rows: pass them as features, without x_in / rfs"};
  return kernel_model_apply(c, m, c.matrix(features));
}
static void reject_kernel_model(const Model& m, const char* what) {
  if (m.kernel) throw KsError{KS_ERR_INVALID, std::string(what) + " is not available for kernel models (KernelBlockLinearMapper)"};
}
// Flat model file (little endian): "KSB2MDL1", int32 block_size, int32 n_blocks, int64 k, int32 has_mean, int32 has_intercept,
// int64 rows[n_blocks], then per block W (rows x k fp64, column-major) [+ rows means], then k intercepts.  Replaces the
// Java-serialised FittedPipeline of the reference (K/workflow/FittedPipeline.scala:18-22) for the BlockLinearMapper stage.
KS_API int32_t ks_model_save(int64_t ctx, int64_t model, const char* path) {
  return guard(ctx, [&](Ctx& c) {
    if (!path) throw KsError{KS_ERR_INVALID, "null path"};
    Model& m = c.model(model);
    reject_kernel_model(m, "save (kernel models hold the training rows and are not persisted)");
    ensure_host_mirror(c, m);
    FILE* f = fopen(path, "wb");
    if (!f) throw KsError{KS_ERR_INVALID, std::string("cannot open ") + path + " for writing"};
    const int32_t hdr[2] = {m.block_size, static_cast<int32_t>(m.brows.size())};
    const int64_t k = m.k;
    const int32_t flags[2] = {m.has_mean ? 1 : 0, m.has_intercept ? 1 : 0};
    bool ok = fwrite("KSB2MDL1", 1, 8, f) == 8 && fwrite(hdr, sizeof(hdr), 1, f) == 1 && fwrite(&k, sizeof(k), 1, f) == 1 &&
              fwrite(flags, sizeof(flags), 1, f) == 1 && fwrite(m.brows.data(), sizeof(int64_t), m.brows.size(), f) == m.brows.size();
    const uint8_t* h = static_cast<const uint8_t*>(m.host.p);
    for (size_t j = 0; ok && j < m.brows.size(); ++j) {
      const size_t nw = static_cast<size_t>(m.brows[j]) * m.k;
      ok = fwrite(h + m.host_w_off[j], sizeof(double), nw, f) == nw;
      if (ok && m.has_mean) ok = fwrite(h + m.host_mean_off[j], sizeof(double), m.brows[j], f) == static_cast<size_t>(m.brows[j]);
    }
    if (ok && m.has_intercept) ok = fwrite(h + m.host_b_off, sizeof(double), m.k, f) == static_cast<size_t>(m.k);
    ok = (fclose(f) == 0) && ok;
    if (!ok) throw KsError{KS_ERR_INVALID, std::string("short write to ") + path};
  });
}
KS_API int32_t ks_model_load(int64_t ctx, const char* path, int64_t* out_model) {
  return guard(ctx, [&](Ctx& c) {
    if (!path || !out_model) throw KsError{KS_ERR_INVALID, "null argument"};
    FILE* f = fopen(path, "rb");
    if (!f) throw KsError{KS_ERR_INVALID, std::string("cannot open ") + path};
    struct Closer { FILE* f; ~Closer() { fclose(f); } } closer{f};
    char magic[8];
    int32_t hdr[2], flags[2];
    int64_t k = 0;
    if (fread(magic, 1, 8, f) != 8 || memcmp(magic, "KSB2MDL1", 8) != 0) throw KsError{KS_ERR_INVALID, "not a keystone_b200 model file"};
    if (fread(hdr, sizeof(hdr), 1, f) != 1 || fread(&k, sizeof(k), 1, f) != 1 || fread(flags, sizeof(flags), 1, f) != 1 ||
        hdr[0] <= 0 || hdr[1] <= 0 || hdr[1] > (1 << 20) || k <= 0)
      throw KsError{KS_ERR_INVALID, "corrupt model header"};
    auto m = std::make_unique<Model>();
    m->block_size = hdr[0];
    m->k = k;
    m->has_mean = flags[0] != 0;
    m->has_intercept = flags[1] != 0;
    m->brows.resize(hdr[1]);
    if (fread(m->brows.data(), sizeof(int64_t), m->brows.size(), f) != m->brows.size()) throw KsError{KS_ERR_INVALID, "truncated model file"};
    for (auto r : m->brows)
      if (r <= 0 || r > m->block_size) throw KsError{KS_ERR_INVALID, "corrupt model header (block rows)"};
    for (size_t j = 0; j < m->brows.size(); ++j) {
      auto W = std::make_unique<DevBuf>();
      W->alloc(sizeof(double) * static_cast<size_t>(m->brows[j]) * k);
      m->W.push_back(std::move(W));
      if (m->has_mean) {
        auto mu = std::make_unique<DevBuf>();
        mu->alloc(sizeof(double) * static_cast<size_t>(m->brows[j]));
        m->mean.push_back(std::move(mu));
      }
    }
    m->intercept.alloc(sizeof(double) * static_cast<size_t>(k));
    model_alloc_host(*m);   // the file is read straight into the pinned mirror, then copied to the device
    uint8_t* h = static_cast<uint8_t*>(m->host.p);
    for (size_t j = 0; j < m->brows.size(); ++j) {
      const size_t nw = static_cast<size_t>(m->brows[j]) * k;
      if (fread(h + m->host_w_off[j], sizeof(double), nw, f) != nw) throw KsError{KS_ERR_INVALID, "truncated model file"};
      KS_CUDA(cudaMemcpyAsync(m->W[j]->p, h + m->host_w_off[j], sizeof(double) * nw, cudaMemcpyHostToDevice, c.st));
      if (m->has_mean) {
        if (fread(h + m->host_mean_off[j], sizeof(double), m->brows[j], f) != static_cast<size_t>(m->brows[j]))
          throw KsError{KS_ERR_INVALID, "truncated model file"};
        KS_CUDA(cudaMemcpyAsync(m->mean[j]->p, h + m->host_mean_off[j], sizeof(double) * m->brows[j], cudaMemcpyHostToDevice, c.st));
      }
    }
    if (m->has_intercept) {
      if (fread(h + m->host_b_off, sizeof(double), k, f) != static_cast<size_t>(k)) throw KsError{KS_ERR_INVALID, "truncated model file"};
      KS_CUDA(cudaMemcpyAsync(m->intercept.p, h + m->host_b_off, sizeof(double) * k, cudaMemcpyHostToDevice, c.st));
    } else {
      KS_CUDA(cudaMemsetAsync(m->intercept.p, 0, sizeof(double) * k, c.st));
    }
    KS_CUDA(cudaStreamSynchronize(c.st));
    *out_model = c.add(std::move(m));
  });
}
KS_API int32_t ks_model_get_intercept(int64_t ctx, int64_t model, double* b_out, int32_t* has_intercept) {
  return guard(ctx, [&](Ctx& c) {
    Model& m = c.model(model);
    if (has_intercept) *has_intercept = m.has_intercept ? 1 : 0;
    if (b_out && m.has_intercept) {
      KS_CUDA(cudaMemcpyAsync(b_out, m.intercept.p, sizeof(double) * m.k, cudaMemcpyDeviceToHost, c.st));
      KS_CUDA(cudaStreamSynchronize(c.st));
    }
  });
}
KS_API int32_t ks_model_apply(int64_t ctx, int64_t model, int64_t features, int64_t x_in, const int64_t* rfs, int32_t n_rfs, int64_t* out) {
  return guard(ctx, [&](Ctx& c) {
    if (!out) throw KsError{KS_ERR_INVALID, "null output"};
    if (c.model(model).kernel) {
      *out = c.add(apply_kernel_model(c, c.model(model), features, x_in, n_rfs));
      return;
    }
    FeatSrc src;
    make_feat_src(c, features, x_in, rfs, n_rfs, src, c.precision);
    *out = c.add(apply_model(c, c.model(model), src, -1, true, c.precision));
  });
}
KS_API int32_t ks_model_apply_partial(int64_t ctx, int64_t model, int64_t features, int64_t x_in, const int64_t* rfs, int32_t n_rfs,
                               int32_t last_block, int64_t* out) {
  return guard(ctx, [&](Ctx& c) {
    if (!out) throw KsError{KS_ERR_INVALID, "null output"};
    reject_kernel_model(c.model(model), "apply_partial");
    FeatSrc src;
    make_feat_src(c, features, x_in, rfs, n_rfs, src, c.precision);
    *out = c.add(apply_model(c, c.model(model), src, last_block, true, c.precision));
  });
}
KS_API int32_t ks_model_apply_argmax(int64_t ctx, int64_t model, int64_t features, int64_t x_in, const int64_t* rfs, int32_t n_rfs,
                              int32_t* host_out) {
  return guard(ctx, [&](Ctx& c) {
    if (!host_out) throw KsError{KS_ERR_INVALID, "null output"};
    std::unique_ptr<Matrix> y;
    if (c.model(model).kernel) {
      y = apply_kernel_model(c, c.model(model), features, x_in, n_rfs);
    } else {
      FeatSrc src;
      make_feat_src(c, features, x_in, rfs, n_rfs, src, c.precision);
      y = apply_model(c, c.model(model), src, -1, true, c.precision);
    }
    DevBuf idx;
    idx.alloc(sizeof(int32_t) * static_cast<size_t>(std::max<int64_t>(y->rows, 1)));
    launch_argmax_rows(y->d, y->ld, y->rows, static_cast<int>(y->cols), idx.as<int32_t>(), c.st);
    c.launches += 1;
    KS_CUDA(cudaMemcpyAsync(host_out, idx.p, sizeof(int32_t) * y->rows, cudaMemcpyDeviceToHost, c.st));
    c.check_async("apply_argmax");
  });
}
KS_API int32_t ks_model_confusion_matrix(int64_t ctx, int64_t model, int64_t features, int64_t x_in, const int64_t* rfs,
                                         int32_t n_rfs, int64_t labels, double* out_counts) {
  return guard(ctx, [&](Ctx& c) {
    if (!out_counts) throw KsError{KS_ERR_INVALID, "null output"};
    Model& m = c.model(model);
    Matrix& L = c.matrix(labels);
    std::unique_ptr<Matrix> y;
    if (m.kernel) {
      if (features == 0 || L.rows != c.matrix(features).rows || L.cols != m.k) throw KsError{KS_ERR_INVALID, "labels shape mismatch"};
      y = apply_kernel_model(c, m, features, x_in, n_rfs);
    } else {
      FeatSrc src;
      make_feat_src(c, features, x_in, rfs, n_rfs, src, c.precision);
      if (L.rows != src.n_rows || L.cols != m.k) throw KsError{KS_ERR_INVALID, "labels shape mismatch"};
      y = apply_model(c, m, src, -1, true, c.precision);
    }
    const int k = static_cast<int>(m.k);
    DevBuf pred, act, counts;
    pred.alloc(sizeof(int32_t) * static_cast<size_t>(std::max<int64_t>(y->rows, 1)));
    act.alloc(pred.bytes);
    counts.alloc(sizeof(unsigned long long) * static_cast<size_t>(k) * k);
    KS_CUDA(cudaMemsetAsync(counts.p, 0, counts.bytes, c.st));
    launch_argmax_rows(y->d, y->ld, y->rows, k, pred.as<int32_t>(), c.st);   // MaxClassifier on the predictions ...
    launch_argmax_rows(L.d, L.ld, L.rows, k, act.as<int32_t>(), c.st);       // ... and on the +-1 indicator labels
    launch_confusion(pred.as<int32_t>(), act.as<int32_t>(), y->rows, k, counts.as<unsigned long long>(), c.st);
    c.launches += 3;
    if (c.world > 1)
      KS_NCCL(nccl_api().AllReduce(counts.p, counts.p, static_cast<size_t>(k) * k, ncclUint64, ncclSum, c.comm, c.st));
    std::vector<unsigned long long> h(static_cast<size_t>(k) * k);
    KS_CUDA(cudaMemcpyAsync(h.data(), counts.p, counts.bytes, cudaMemcpyDeviceToHost, c.st));
    c.check_async("confusion_matrix");
    for (size_t i = 0; i < h.size(); ++i) out_counts[i] = static_cast<double>(h[i]);
  });
}
KS_API int32_t ks_model_cost(int64_t ctx, int64_t model, int64_t features, int64_t x_in, const int64_t* rfs, int32_t n_rfs,
                      int64_t labels, double lambda, double* out_cost) {
  return guard(ctx, [&](Ctx& c) {
    if (!out_cost) throw KsError{KS_ERR_INVALID, "null output"};
    Model& m = c.model(model);
    reject_kernel_model(m, "computeCost");
    Matrix& L = c.matrix(labels);
    FeatSrc src;
    make_feat_src(c, features, x_in, rfs, n_rfs, src, c.precision);
    if (L.rows != src.n_rows || L.cols != m.k) throw KsError{KS_ERR_INVALID, "labels shape mismatch"};
    auto y = apply_model(c, m, src, -1, /*use_means=*/false, c.precision);  // computeCost applies no feature scalers (:149-156)
    DevBuf acc;  // [0] squared error, [1] row count, [2] ||W||^2
    acc.alloc(sizeof(double) * 3);
    KS_CUDA(cudaMemsetAsync(acc.p, 0, acc.bytes, c.st));
    launch_sq_err(y->d, y->ld, L.d, L.ld, L.rows, static_cast<int>(m.k), acc.as<double>(), c.st);
    c.launches += 1;
    const double nl = static_cast<double>(L.rows);
    KS_CUDA(cudaMemcpyAsync(acc.as<double>() + 1, &nl, sizeof(double), cudaMemcpyHostToDevice, c.st));
    KS_CUDA(cudaStreamSynchronize(c.st));
    c.allreduce_f64(acc.as<double>(), 2);
    for (size_t j = 0; j < m.W.size(); ++j) {
      sumsq_f64_kernel<<<64, 256, 0, c.st>>>(m.W[j]->as<double>(), m.brows[j] * m.k, acc.as<double>() + 2);
      c.launches += 1;
    }
    double h[3];
    KS_CUDA(cudaMemcpyAsync(h, acc.p, sizeof(h), cudaMemcpyDeviceToHost, c.st));
    c.check_async("computeCost");
    *out_cost = h[0] / (2.0 * h[1]) + (lambda == 0 ? 0.0 : lambda / 2.0 * h[2]);
  });
}
KS_API int32_t ks_model_destroy(int64_t ctx, int64_t model) {
  return guard(ctx, [&](Ctx& c) {
    if (!c.models.erase(model)) throw KsError{KS_ERR_HANDLE, "unknown model handle"};
  });
}

// ---------------------------------------------------------------- Gaussian kernel ridge regression (krr.cu)
static std::shared_ptr<GaussKernel> find_kernel(Ctx& c, int64_t h) {
  auto it = c.kernels.find(h);
  if (it == c.kernels.end()) throw KsError{KS_ERR_HANDLE, "unknown Gaussian kernel handle " + std::to_string(h)};
  return it->second;
}
KS_API int32_t ks_gaussian_kernel_create(int64_t ctx, int64_t x_train, double gamma, int64_t* out_kernel) {
  return guard(ctx, [&](Ctx& c) {
    if (!out_kernel) throw KsError{KS_ERR_INVALID, "null out_kernel"};
    *out_kernel = gaussian_kernel_create(c, c.matrix(x_train), gamma);
  });
}
KS_API int32_t ks_gaussian_kernel_block(int64_t ctx, int64_t kernel, int64_t x, int64_t col0, int64_t cols, int64_t* out_m) {
  return guard(ctx, [&](Ctx& c) {
    if (!out_m) throw KsError{KS_ERR_INVALID, "null out_m"};
    auto K = find_kernel(c, kernel);
    *out_m = c.add(gaussian_kernel_block(c, *K, c.matrix(x), col0, cols));
  });
}
KS_API int32_t ks_gaussian_kernel_shape(int64_t ctx, int64_t kernel, int64_t* n_train, int64_t* dim) {
  return guard(ctx, [&](Ctx& c) {
    auto K = find_kernel(c, kernel);
    if (n_train) *n_train = K->n;
    if (dim) *dim = K->d;
  });
}
KS_API int32_t ks_gaussian_kernel_destroy(int64_t ctx, int64_t kernel) {
  return guard(ctx, [&](Ctx& c) {
    if (!c.kernels.erase(kernel)) throw KsError{KS_ERR_HANDLE, "unknown Gaussian kernel handle"};
  });
}
KS_API int32_t ks_krr_fit(int64_t ctx, int64_t kernel, int64_t labels, double lambda, int32_t block_size, int32_t num_epochs,
                          const int32_t* block_order_or_null, int64_t* out_model) {
  return guard(ctx, [&](Ctx& c) {
    if (!out_model) throw KsError{KS_ERR_INVALID, "null out_model"};
    auto K = find_kernel(c, kernel);
    *out_model = fit_krr(c, K, c.matrix(labels), lambda, block_size, num_epochs, block_order_or_null);
  });
}
KS_API int32_t ks_kernel_model_from_host(int64_t ctx, int64_t kernel, const double* const* xs_colmajor, const int64_t* block_rows,
                                         int32_t n_blocks, int64_t k, int32_t block_size, int64_t* out_model) {
  return guard(ctx, [&](Ctx& c) {
    if (!out_model) throw KsError{KS_ERR_INVALID, "null out_model"};
    *out_model = kernel_model_from_host(c, find_kernel(c, kernel), xs_colmajor, block_rows, n_blocks, k, block_size);
  });
}

KS_API int32_t ks_last_fit_stats_json_size(int64_t ctx, int64_t* out_bytes) {
  return guard(ctx, [&](Ctx& c) {
    if (!out_bytes) throw KsError{KS_ERR_INVALID, "null out_bytes"};
    *out_bytes = static_cast<int64_t>(c.stats_json.size()) + 1;
  });
}
KS_API int32_t ks_last_fit_stats_json(int64_t ctx, char* buf, int64_t buflen) {
  return guard(ctx, [&](Ctx& c) {
    if (!buf || buflen <= 0) throw KsError{KS_ERR_INVALID, "bad buffer"};
    const std::string& s = c.stats_json;
    if (static_cast<int64_t>(s.size()) + 1 > buflen) throw KsError{KS_ERR_INVALID, "buffer too small"};
    memcpy(buf, s.c_str(), s.size() + 1);
  });
}

// ---------------------------------------------------------------- debug / micro-benchmarks
// With the context option precision = KS_PRECISION_F16 the operands are first converted to fp16 and the fp16 kernel runs;
// with KS_PRECISION_F16X2 they are split into fp16 pairs hi + lo and the split kernel runs (G = A^T A keeps
// hi^T hi + lo^T hi + hi^T lo); with KS_PRECISION_TF32 the fp32 operands go to the tf32 kernel as they are.
struct DebugGramOps {
  DevBuf a16, b16, a16lo, b16lo;
  const void* A = nullptr;
  const void* B = nullptr;
  const void* Alo = nullptr;
  const void* Blo = nullptr;
  bool f16 = false;
};
__global__ void split_f16_pair_kernel(const float* __restrict__ src, int64_t ld, int64_t rows, int cols, __half* __restrict__ hi,
                                      __half* __restrict__ lo) {
  const int64_t total = rows * cols;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / cols, o = r * ld + (i - r * cols);
    const float v = src[o];
    const __half h = __float2half_rn(v);
    hi[o] = h;
    lo[o] = __float2half_rn(v - __half2float(h));
  }
}
static void debug_split_f16(Ctx& c, Matrix& M, DevBuf& hi, DevBuf& lo) {
  const size_t bytes = 2 * static_cast<size_t>(std::max<int64_t>(M.rows, 1) * M.ld);
  hi.alloc(bytes);
  lo.alloc(bytes);
  KS_CUDA(cudaMemsetAsync(hi.p, 0, bytes, c.st));  // pad columns stay zero
  KS_CUDA(cudaMemsetAsync(lo.p, 0, bytes, c.st));
  const int64_t total = M.rows * M.cols;
  if (total > 0) {
    const unsigned grid = static_cast<unsigned>(std::min<int64_t>((total + 255) / 256, 4096));
    split_f16_pair_kernel<<<grid, 256, 0, c.st>>>(M.d, M.ld, M.rows, static_cast<int>(M.cols), hi.as<__half>(), lo.as<__half>());
    c.launches += 1;
  }
}
static void debug_gram_run(Ctx& c, Matrix& A, Matrix& B, DevBuf& gc, int* ldg, int* ldc, DebugGramOps& ops) {
  if (A.rows != B.rows) throw KsError{KS_ERR_INVALID, "row mismatch"};
  ops.f16 = c.precision == KS_PRECISION_F16 || c.precision == KS_PRECISION_F16X2;
  ops.A = A.d;
  ops.B = B.d;
  if (c.precision == KS_PRECISION_F16X2) {
    debug_split_f16(c, A, ops.a16, ops.a16lo);
    debug_split_f16(c, B, ops.b16, ops.b16lo);
    ops.A = ops.a16.p;
    ops.B = ops.b16.p;
    ops.Alo = ops.a16lo.p;
    ops.Blo = ops.b16lo.p;
  } else if (ops.f16) {
    ops.a16.alloc(2 * static_cast<size_t>(std::max<int64_t>(A.rows, 1) * A.ld));
    ops.b16.alloc(2 * static_cast<size_t>(std::max<int64_t>(B.rows, 1) * B.ld));
    launch_f32_to_f16_rows(A.d, A.ld, ops.a16.p, A.ld, A.rows, A.cols, c.st);
    launch_f32_to_f16_rows(B.d, B.ld, ops.b16.p, B.ld, B.rows, B.cols, c.st);
    ops.A = ops.a16.p;
    ops.B = ops.b16.p;
  }
  const int b = static_cast<int>(A.cols), kc = static_cast<int>(B.cols);
  *ldg = static_cast<int>(round_up(b, 32));
  *ldc = static_cast<int>(round_up(kc, 32));
  const size_t ge = static_cast<size_t>(b) * *ldg, ce = static_cast<size_t>(b) * *ldc;
  gc.alloc(sizeof(float) * (ge + ce));
  KS_CUDA(cudaMemsetAsync(gc.p, 0, gc.bytes, c.st));
  launch_gram_block(c, ops.A, A.ld, A.rows, b, ops.B, B.ld, kc, gc.as<float>(), *ldg, gc.as<float>() + ge, *ldc, true, true,
                    nullptr, ops.f16, 0, ops.Alo, ops.Blo);
}
KS_API int32_t ks_debug_gram(int64_t ctx, int64_t a, int64_t b, double* out_g, int64_t ld_g, double* out_c, int64_t ld_c) {
  return guard(ctx, [&](Ctx& c) {
    Matrix& A = c.matrix(a);
    Matrix& B = c.matrix(b);
    DevBuf gc;
    DebugGramOps ops;
    int ldg, ldc;
    debug_gram_run(c, A, B, gc, &ldg, &ldc, ops);
    c.check_async("debug_gram");
    const int m = static_cast<int>(A.cols), kc = static_cast<int>(B.cols);
    std::vector<float> h(gc.bytes / sizeof(float));
    KS_CUDA(cudaMemcpy(h.data(), gc.p, gc.bytes, cudaMemcpyDeviceToHost));
    const float* G = h.data();
    const float* C = h.data() + static_cast<size_t>(m) * ldg;
    if (out_g)
      for (int r = 0; r < m; ++r)
        for (int q = 0; q < m; ++q) out_g[r * ld_g + q] = G[static_cast<size_t>(std::min(r, q)) * ldg + std::max(r, q)];
    if (out_c)
      for (int r = 0; r < m; ++r)
        for (int q = 0; q < kc; ++q) out_c[r * ld_c + q] = C[static_cast<size_t>(r) * ldc + q];
  });
}
KS_API int32_t ks_debug_time_gram(int64_t ctx, int64_t a, int64_t b, int32_t iters, double* out_ms) {
  return guard(ctx, [&](Ctx& c) {
    Matrix& A = c.matrix(a);
    Matrix& B = c.matrix(b);
    DevBuf gc;
    DebugGramOps ops;
    int ldg, ldc;
    debug_gram_run(c, A, B, gc, &ldg, &ldc, ops);  // warm-up + allocation
    const size_t ge = static_cast<size_t>(A.cols) * ldg;
    cudaEvent_t e0 = c.get_event(), e1 = c.get_event();
    KS_CUDA(cudaEventRecord(e0, c.st));
    for (int i = 0; i < iters; ++i)
      launch_gram_block(c, ops.A, A.ld, A.rows, static_cast<int>(A.cols), ops.B, B.ld, static_cast<int>(B.cols), gc.as<float>(),
                        ldg, gc.as<float>() + ge, ldc, true, true, nullptr, ops.f16, 0, ops.Alo, ops.Blo);
    KS_CUDA(cudaEventRecord(e1, c.st));
    c.check_async("debug_time_gram");
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    c.event_pool.push_back(e0);
    c.event_pool.push_back(e1);
    *out_ms = ms / std::max(iters, 1);
  });
}

KS_API int32_t ks_debug_chol_solve(int64_t ctx, const double* H_colmajor, int32_t n, const double* B_colmajor, int32_t k,
                                   int32_t use_cusolver, double* X_out, double* out_ms) {
  return guard(ctx, [&](Ctx& c) {
    if (!H_colmajor || !B_colmajor || !X_out || n <= 0 || k <= 0) throw KsError{KS_ERR_INVALID, "bad arguments"};
    DevBuf H, B, Dv;
    H.alloc(sizeof(double) * static_cast<size_t>(n) * n);
    B.alloc(sizeof(double) * static_cast<size_t>(n) * k);
    Dv.alloc(sizeof(double) * chol_solve_dinv_doubles(n));
    KS_CUDA(cudaMemcpyAsync(H.p, H_colmajor, sizeof(double) * static_cast<size_t>(n) * n, cudaMemcpyHostToDevice, c.st));
    c.potrf(H.as<double>(), n, 0, c.st);
    KS_CUDA(launch_tri_inv_tiles(H.as<double>(), n, Dv.as<double>(), c.st));
    float best = 1e30f;
    for (int rep = 0; rep < 3; ++rep) {
      KS_CUDA(cudaMemcpyAsync(B.p, B_colmajor, sizeof(double) * static_cast<size_t>(n) * k, cudaMemcpyHostToDevice, c.st));
      cudaEvent_t e0 = c.get_event(), e1 = c.get_event();
      KS_CUDA(cudaEventRecord(e0, c.st));
      if (use_cusolver) c.potrs(H.as<double>(), n, B.as<double>(), k, 1, c.st);
      else KS_CUDA(launch_chol_solve(H.as<double>(), Dv.as<double>(), n, B.as<double>(), k, c.st));
      KS_CUDA(cudaEventRecord(e1, c.st));
      c.check_async("debug_chol_solve");
      float ms = 0;
      cudaEventElapsedTime(&ms, e0, e1);
      best = std::min(best, ms);
      c.event_pool.push_back(e0);
      c.event_pool.push_back(e1);
    }
    c.check_infos(2);
    KS_CUDA(cudaMemcpy(X_out, B.p, sizeof(double) * static_cast<size_t>(n) * k, cudaMemcpyDeviceToHost));
    if (out_ms) *out_ms = best;
  });
}

}  // extern "C"
