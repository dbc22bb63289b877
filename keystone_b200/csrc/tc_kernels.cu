// Tensor-core kernels of the block least-squares hot path (sm_90a: TMA + mbarrier pipelines feeding wgmma).
//
//   gram_tn_kernel    D[M x N] += A^T B over a chunk of rows, A [rows x M] and B [rows x N] both
//                     row-major (contraction over the slow axis => both operands MN-major).
//                     Replaces the per-partition (A^T A, A^T R) + treeReduce of the reference
//                     (K/nodes/learning/BlockWeightedLeastSquares.scala:212-214 and the mlmatrix
//                     NormalEquations called from K/nodes/learning/BlockLinearMapper.scala:236-239).
//   gemm_kmajor_kernel D[M x N] = A B^T, A [M x K] and B [N x K] row-major (K-major operands),
//                     persistent, with fused epilogues:
//                       EPI_COS     out  = tf32(cos(acc + bias) - shift)     (CosineRandomFeatures.scala:30-32)
//                       EPI_UPDATE  R   += -acc + cbias                      (BlockWeightedLeastSquares.scala:287-290)
//                       EPI_APPLY   Y [+]= acc + cbias                       (BlockLinearMapper.scala:55-70)
//                       EPI_POOL    Convolver -> SymmetricRectifier -> sum Pooler (Convolver.scala, Pooler.scala)
//                       EPI_RBF     out  = exp(-gamma (n_i + n_j - 2 acc))   (KernelGenerator.scala:160-176)
//
// Both kernels are 128 x 128 output tiles on 384 threads: warpgroup 0 issues the TMA loads of a 4-stage mbarrier ring,
// warpgroups 1 and 2 each own 64 output rows (one m64n128 wgmma accumulator, 64 fp32 registers per thread) and run the
// epilogue.  The accumulator goes registers -> shared memory (transposed so that lane i holds row i of a 32 x 32 chunk) ->
// epilogue math -> 128 B-swizzled staging -> TMA store / TMA reduce-add, so global memory only sees full 128 B rows.
// wgmma accepts tf32 operands only K-major, so the tf32 Gram (MN-major) builds warp-level mma.sync fragments from the same
// TMA-filled stages instead.
// The slab producers (EPI_COS, EPI_RBF) add a fourth warpgroup that runs the epilogue while the MMA warpgroups go on to the next
// tile (KmSmem).
// SPLIT variants (parity mode, fp16 pairs; Gram and EPI_UPDATE): each stage holds the hi and lo planes of both operands and one
// pass issues hi·hi, lo·hi and hi·lo into two accumulators, so the operands are fetched and the output is reduce-added once.
#include <algorithm>
#include <type_traits>

#include "tc_common.cuh"
#include "kernels.h"

namespace ks {

static constexpr int kThreads = 384;
static constexpr int kTileM = 128, kTileN = 128;
static constexpr int kStages = 4;
static constexpr int kRawLd = 65;  // odd row pitch: lane i reading row i of the transpose buffer hits bank (i + col) % 32
static constexpr int kRawBytes = 2 * 64 * kRawLd * 4;   // one 64 x 64 slab per consumer warpgroup
static constexpr int kStagingBytes = 8 * 4096;          // one 32 x 32 fp32 chunk per consumer warp
static constexpr int kVecBytes = 8 * 64 * 4;            // per-warp copies of 32 columns of vec0 and vec1
static constexpr int kEpiBytes = kStagingBytes + kRawBytes + kVecBytes;
static constexpr int kStageBytes = 32768;               // A and B tiles of one stage (128 x 128 B each)
static constexpr int kSmemBytes = kStages * kStageBytes + kEpiBytes + 1024 /*align*/ + 256 /*barriers*/;
static_assert(kSmemBytes <= 227 * 1024, "shared memory per block");

struct SmemLayout {
  uint8_t* stages;
  uint8_t* staging;  // 8 x 4 KB, 1024 B aligned
  float* raw;        // 2 x [64][kRawLd]
  float* vec;        // 8 x 64
  uint64_t* full_bar;
  uint64_t* empty_bar;
  uint64_t* ring_bar;  // [8]
  int* tile_ring;      // [8]
};
__device__ __forceinline__ SmemLayout carve_smem(uint8_t* smem_raw) {
  SmemLayout L;
  L.stages = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  L.staging = L.stages + kStages * kStageBytes;
  L.raw = reinterpret_cast<float*>(L.staging + kStagingBytes);
  L.vec = L.raw + 2 * 64 * kRawLd;
  L.full_bar = reinterpret_cast<uint64_t*>(L.vec + 8 * 64);
  L.empty_bar = L.full_bar + kStages;
  L.ring_bar = L.empty_bar + kStages;
  L.tile_ring = reinterpret_cast<int*>(L.ring_bar + 8);
  return L;
}

// Slab producers (EPI_COS, EPI_RBF) run their epilogue in separate warps, so that the MMA warpgroups go straight on to the next
// tile: they dump the accumulator into a whole-tile fp32 buffer and hand it over with the tile id (tile_full), and the epilogue
// warps give the buffer back (tile_empty) once they have read it.  Their epilogue per element (range-reduced cosine or exp, the
// hi / lo split, the fp16 staging, column sums) costs about as much as the tile's MMA at K ~ 1000, so it now hides under the next
// tile's main loop.  Eight epilogue warps, two per SM sub-partition (one warp each leaves the epilogue's latencies exposed and
// makes it slower than the MMA): the three warps of the producer warpgroup that issue no TMA, warpgroup 3 and a 17th warp, 544
// threads (120 registers each).  Each takes two 32 x 32 chunks of a tile.  Shared memory: 4 stages, the 128 x 129 tile buffer,
// one 4 KB staging chunk per epilogue warp and one copy of the tile's vec0 / vec1 columns for all of them.
__host__ __device__ constexpr bool km_async(int epi) { return epi == EPI_COS || epi == EPI_RBF; }
__host__ __device__ constexpr int km_threads(int epi) { return km_async(epi) ? 544 : kThreads; }
static constexpr int kEpiWarps = 8;
static constexpr int kTileLd = 129;  // odd row pitch, as kRawLd
static constexpr int kTileBufBytes = kTileM * kTileLd * 4;
static constexpr int kAsyncStagingBytes = kEpiWarps * 4096;
static constexpr int kAsyncVecBytes = 2 * kTileN * 4;  // vec0 and vec1 of the tile's 128 columns, [chunk][vec0 32 | vec1 32]
static constexpr int kAsyncSmemBytes =
    kStages * kStageBytes + kAsyncStagingBytes + kTileBufBytes + kAsyncVecBytes + 1024 /*align*/ + 256 /*barriers*/;
static_assert(kAsyncSmemBytes <= 227 * 1024, "shared memory per block");
__host__ __device__ constexpr int km_smem_bytes(int epi) { return km_async(epi) ? kAsyncSmemBytes : kSmemBytes; }

struct KmSmem : SmemLayout {
  float* tile = nullptr;  // [kTileM][kTileLd]: the accumulator of one tile (async epilogue only)
  uint64_t* tile_full = nullptr;
  uint64_t* tile_empty = nullptr;
  int* tile_id = nullptr;  // id of the tile in the buffer (-1: no more tiles)
};
template <bool ASYNC>
__device__ __forceinline__ KmSmem carve_km_smem(uint8_t* smem_raw) {
  KmSmem L;
  if (!ASYNC) {
    static_cast<SmemLayout&>(L) = carve_smem(smem_raw);
    return L;
  }
  L.stages = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  L.staging = L.stages + kStages * kStageBytes;
  L.tile = reinterpret_cast<float*>(L.staging + kAsyncStagingBytes);
  L.raw = nullptr;
  L.vec = L.tile + kTileM * kTileLd;
  L.full_bar = reinterpret_cast<uint64_t*>(L.vec + kAsyncVecBytes / 4);
  L.empty_bar = L.full_bar + kStages;
  L.ring_bar = L.empty_bar + kStages;
  L.tile_full = L.ring_bar + 8;
  L.tile_empty = L.tile_full + 1;
  L.tile_ring = reinterpret_cast<int*>(L.tile_empty + 1);
  L.tile_id = L.tile_ring + 8;
  return L;
}

// Accumulator of one warpgroup (m64n128 wgmma layout: register 4j + e of thread (warp w, lane l) is row 16w + l/4 + 8(e/2),
// column 8j + 2(l%4) + e%2) -> columns [64 slab, +64) of the warpgroup's transpose buffer.
__device__ __forceinline__ void wgmma_acc_to_raw(const float (&acc)[64], float* raw, int slab, int w, int lane) {
#pragma unroll
  for (int jj = 0; jj < 8; ++jj)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int r = 16 * w + (lane >> 2) + 8 * (e >> 1);
      const int c = 8 * jj + 2 * (lane & 3) + (e & 1);
      raw[r * kRawLd + c] = acc[4 * (8 * slab + jj) + e];
    }
}
// Shared-memory accesses of the whole-tile buffer by 32-bit address: through a generic pointer the compiler keeps one 64-bit
// address per element live and runs out of the 128 registers a 512-thread CTA allows.
__device__ __forceinline__ void sts_f32(uint32_t addr, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v)); }
__device__ __forceinline__ float lds_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
// The same transpose for all 128 columns at once: warpgroup g's accumulator -> rows [64 g, +64) of the whole-tile buffer.
__device__ __forceinline__ void wgmma_acc_to_tile(const float (&acc)[64], uint32_t tile, int g, int w, int lane) {
  const uint32_t base = tile + 4 * ((64 * g + 16 * w + (lane >> 2)) * kTileLd + 2 * (lane & 3));
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) sts_f32(base + 4 * ((8 * (e >> 1)) * kTileLd + 8 * j + (e & 1)), acc[4 * j + e]);
}

// Epilogue walk shared by both kernels.  For each 64-column slab the warpgroup's accumulator goes through the transpose
// buffer; warp w then holds rows 32 (w % 2) + lane and columns 32 (w / 2) + i of the slab as o[i] and calls
// chunk(o, slab, row offset in the warpgroup, column offset in the tile).
template <typename ToRaw, typename Chunk>
__device__ __forceinline__ void epilogue_slabs(float* raw, int g, int w, int lane, ToRaw to_raw, Chunk chunk) {
#pragma unroll  // constant slab: the accumulator registers are indexed statically
  for (int slab = 0; slab < kTileN / 64; ++slab) {
    to_raw(raw, slab);
    named_bar_sync(1 + g, 128);
    float o[32];
    const float* src = raw + (32 * (w & 1) + lane) * kRawLd + 32 * (w >> 1);
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = src[i];
    named_bar_sync(1 + g, 128);  // the buffer is free for the next slab
    chunk(o, slab, 32 * (w & 1), slab * 64 + 32 * (w >> 1));
  }
}

// =====================================================================================
// Gram / A^T B kernel (MN-major operands, split over row chunks, TMA reduce-add epilogue)
// =====================================================================================
// F16: fp16 operands, 64-column (128 B) x 64-row TMA boxes, wgmma with both operands MN-major (K = 16 per instruction);
// tf32: fp32 containers, 32-column x 32-row boxes, mma.sync m16n8k8 fragments (K = 8).  Either way a stage holds the 128
// columns of A and of B for SR rows of the contraction: 32 KB.
// SPLIT (fp16 pairs): a stage holds the four tiles A_hi, A_lo, B_hi, B_lo of 32 rows each (64 x 32 boxes), still 32 KB.
template <bool F16, bool SPLIT = false>
struct GramCfg {
  static constexpr int PLANES = SPLIT ? 4 : 2;   // operand tiles per stage
  static constexpr int SR = SPLIT ? 32 : F16 ? 64 : 32;  // rows (K) per stage
  static constexpr int CW = F16 ? 64 : 32;       // columns per TMA box (128 B)
  static constexpr int NBOX = kTileM / CW;       // boxes per 128 operand columns
  static constexpr int BOX_BYTES = SR * 128;
  static constexpr int A_BYTES = NBOX * BOX_BYTES;
  static_assert(PLANES * A_BYTES == kStageBytes, "stage size");
  static_assert(!SPLIT || F16, "split operands are fp16 pairs");
  static_assert(!SPLIT || NBOX == 2, "each CTA of a pair fetches one box of each shared plane");
};

// tf32 element (column c, row r) of one MN-major operand tile: 32-column boxes of SR rows, 128 B swizzle
template <int BOX_BYTES>
__device__ __forceinline__ uint32_t ld_mn_tf32(const uint8_t* tile, int c, int r) {
  return *reinterpret_cast<const uint32_t*>(tile + (c >> 5) * BOX_BYTES + r * 128 + (((((c & 31) >> 2) ^ (r & 7))) << 4) +
                                            ((c & 3) << 2));
}

// SPLIT: D += A_hi^T B_hi + A_lo^T B_hi + A_hi^T B_lo in one pass.  The hi x hi product accumulates in its own registers
// with the same instruction sequence as the single-product kernel; the two cross products (~2^-11 smaller) share a second
// accumulator; the two are added (fp32, round-to-nearest) before the epilogue, so each chunk is reduce-added once.
template <bool F16, bool SPLIT>
__global__ void __launch_bounds__(kThreads, 1)
gram_tn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB0,
               const __grid_constant__ CUtensorMap tmB1, const __grid_constant__ CUtensorMap tmOut0,
               const __grid_constant__ CUtensorMap tmOut1, const __grid_constant__ CUtensorMap tmAlo,
               const __grid_constant__ CUtensorMap tmB0lo, const __grid_constant__ CUtensorMap tmB1lo,
               const GramTile* __restrict__ tiles, int num_tiles, int rows, int chunk_rows, int n_valid0, int n_valid1) {
  using Cfg = GramCfg<F16, SPLIT>;
  constexpr int SR = Cfg::SR;
  extern __shared__ uint8_t smem_raw[];
  const SmemLayout L = carve_smem(smem_raw);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  // SPLIT: clusters of two CTAs, one pair of tiles each; entry 2 p + rank of the list is this CTA's tile of pair p
  const uint32_t rank = SPLIT ? cl_ctarank() : 0;
  const int pairs = num_tiles / 2;
  const GramTile tile = SPLIT ? tiles[2 * ((blockIdx.x >> 1) % pairs) + rank] : tiles[blockIdx.x % num_tiles];
  const int chunk = SPLIT ? (blockIdx.x >> 1) / pairs : blockIdx.x / num_tiles;
  const bool idle = SPLIT && (tile.pair & GRAM_IDLE);
  const bool share_b = SPLIT && (tile.pair & GRAM_SHARE_B);
  const int row0 = chunk * chunk_rows;
  const int nrows = min(chunk_rows, rows - row0);
  const int ksteps = (nrows + SR - 1) / SR;
  const int m0 = tile.m_blk * kTileM;
  const int n0 = tile.n_blk * kTileN;
  const CUtensorMap* tmB = tile.which ? &tmB1 : &tmB0;
  const CUtensorMap* tmBlo = tile.which ? &tmB1lo : &tmB0lo;
  const CUtensorMap* tmOut = tile.which ? &tmOut1 : &tmOut0;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(tmB);
    if (SPLIT) {
      tma_prefetch_desc(&tmAlo);
      tma_prefetch_desc(tmBlo);
    }
    tma_prefetch_desc(tmOut);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&L.full_bar[s], 1);
      mbar_init(&L.empty_bar[s], SPLIT ? 16 : 8);  // one arrive per consumer warp (SPLIT: of both CTAs of the pair)
    }
    fence_barrier_init();
  }
  if (SPLIT) cl_sync();  // the partner's barriers are initialised before anything lands in or arrives on them
  else __syncthreads();

  if (wg == 0) {
    if (SPLIT) setmaxnreg_dec<40>();  // two accumulators per consumer thread
    if (warp == 0 && elect_one()) {
      for (int ks = 0; ks < ksteps; ++ks) {
        const int s = ks % kStages;
        const uint32_t ph = (ks / kStages) & 1;
        mbar_wait(&L.empty_bar[s], ph ^ 1);  // SPLIT: released by the consumers of both CTAs (the multicast writes into both)
        mbar_arrive_expect_tx(&L.full_bar[s], idle ? kStageBytes / 2 : kStageBytes);
        uint8_t* sA = L.stages + s * kStageBytes;
        const int r = row0 + ks * SR;
        // tiles in stage order: A, B (SPLIT: A_hi, A_lo, B_hi, B_lo)
        const CUtensorMap* maps[4] = {&tmA, SPLIT ? &tmAlo : tmB, tmB, tmBlo};
#pragma unroll
        for (int pl = 0; pl < Cfg::PLANES; ++pl) {
          const int c0 = (pl < Cfg::PLANES / 2) ? m0 : n0;
          if (SPLIT && (pl >= Cfg::PLANES / 2) == share_b) {
            // the shared panel: this CTA fetches box `rank` of the plane for both CTAs of the pair
            tma_load_2d_mc(sA + pl * Cfg::A_BYTES + rank * Cfg::BOX_BYTES, maps[pl], &L.full_bar[s], c0 + Cfg::CW * rank, r, 0x3);
            continue;
          }
          if (idle) continue;
#pragma unroll
          for (int i = 0; i < Cfg::NBOX; ++i)
            tma_load_2d(sA + pl * Cfg::A_BYTES + i * Cfg::BOX_BYTES, maps[pl], &L.full_bar[s], c0 + Cfg::CW * i, r);
        }
      }
    }
    if (SPLIT) {
      __syncwarp();
      cl_sync();  // neither CTA exits while the other may still write into its stages or arrive on its barriers
    }
    return;
  }
  if (SPLIT) setmaxnreg_inc<232>();

  const int g = wg - 1;  // output rows [64 g, +64) of the tile
  const int w = warp & 3;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;

  if (SPLIT) {
    float acc_x[64];  // lo^T hi + hi^T lo
#pragma unroll
    for (int i = 0; i < 64; ++i) acc_x[i] = 0.f;
    wgmma_fence_acc(acc);
    wgmma_fence_acc(acc_x);
    // a stage is released to the producers of both CTAs: each of them refills part of it
    const uint32_t peer_empty = cl_map_shared(smem_u32(L.empty_bar), rank ^ 1);
    auto release = [&](int s) {
      mbar_arrive(&L.empty_bar[s]);
      mbar_arrive_remote(peer_empty + 8 * s);
    };
    int prev = -1;
    for (int ks = 0; ks < ksteps; ++ks) {
      const int s = ks % kStages;
      mbar_wait(&L.full_bar[s], (ks / kStages) & 1);
      if (idle) {  // the partner's tile alone: hand the stage back once its half of the shared panel has landed here
        if (lane == 0) release(s);
        continue;
      }
      const uint32_t st = smem_u32(L.stages + s * kStageBytes);
      const uint32_t sAhi = st + g * Cfg::BOX_BYTES, sAlo = sAhi + Cfg::A_BYTES;  // this warpgroup's 64 columns of A
      const uint32_t sBhi = st + 2 * Cfg::A_BYTES, sBlo = st + 3 * Cfg::A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < SR / 16; ++kk)
        wgmma_f16_n128<1, 1>(acc, make_wgmma_desc(sAhi + kk * 2048, Cfg::BOX_BYTES, 1024),
                             make_wgmma_desc(sBhi + kk * 2048, Cfg::BOX_BYTES, 1024), 1);
#pragma unroll
      for (int kk = 0; kk < SR / 16; ++kk) {
        wgmma_f16_n128<1, 1>(acc_x, make_wgmma_desc(sAlo + kk * 2048, Cfg::BOX_BYTES, 1024),
                             make_wgmma_desc(sBhi + kk * 2048, Cfg::BOX_BYTES, 1024), 1);
        wgmma_f16_n128<1, 1>(acc_x, make_wgmma_desc(sAhi + kk * 2048, Cfg::BOX_BYTES, 1024),
                             make_wgmma_desc(sBlo + kk * 2048, Cfg::BOX_BYTES, 1024), 1);
      }
      wgmma_commit();
      if (prev >= 0) {
        wgmma_wait<1>();
        if (lane == 0) release(prev);
      }
      prev = s;
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    wgmma_fence_acc(acc_x);
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = __fadd_rn(acc[i], acc_x[i]);
  } else if (F16) {
    wgmma_fence_acc(acc);
    int prev = -1;
    for (int ks = 0; ks < ksteps; ++ks) {
      const int s = ks % kStages;
      mbar_wait(&L.full_bar[s], (ks / kStages) & 1);
      const uint32_t sA = smem_u32(L.stages + s * kStageBytes) + g * Cfg::BOX_BYTES;  // this warpgroup's 64 columns of A
      const uint32_t sB = smem_u32(L.stages + s * kStageBytes) + Cfg::A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < SR / 16; ++kk) {
        // 16 rows of K per instruction = two 8-row groups 1024 B apart (SBO); B's two 64-column blocks are a box apart (LBO)
        const uint64_t ad = make_wgmma_desc(sA + kk * 2048, Cfg::BOX_BYTES, 1024);
        const uint64_t bd = make_wgmma_desc(sB + kk * 2048, Cfg::BOX_BYTES, 1024);
        wgmma_f16_n128<1, 1>(acc, ad, bd, 1);
      }
      wgmma_commit();
      if (prev >= 0) {
        wgmma_wait<1>();  // the previous stage's wgmmas have finished reading it
        if (lane == 0) mbar_arrive(&L.empty_bar[prev]);
      }
      prev = s;
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
  } else {
    // warp tile: rows [32 (w % 2), +32) of the warpgroup's 64, columns [64 (w / 2), +64): 2 x 8 m16n8 fragments
    const int mrow = 64 * g + 32 * (w & 1);
    const int ncol = 64 * (w >> 1);
    const int gq = lane >> 2, tq = lane & 3;
    for (int ks = 0; ks < ksteps; ++ks) {
      const int s = ks % kStages;
      mbar_wait(&L.full_bar[s], (ks / kStages) & 1);
      const uint8_t* sA = L.stages + s * kStageBytes;
      const uint8_t* sB = sA + Cfg::A_BYTES;
#pragma unroll
      for (int k = 0; k < SR; k += 8) {
        uint32_t a[2][4], b[8][2];
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) {
          const int m = mrow + 16 * mi + gq;
          a[mi][0] = ld_mn_tf32<Cfg::BOX_BYTES>(sA, m, k + tq);
          a[mi][1] = ld_mn_tf32<Cfg::BOX_BYTES>(sA, m + 8, k + tq);
          a[mi][2] = ld_mn_tf32<Cfg::BOX_BYTES>(sA, m, k + tq + 4);
          a[mi][3] = ld_mn_tf32<Cfg::BOX_BYTES>(sA, m + 8, k + tq + 4);
        }
#pragma unroll
        for (int ni = 0; ni < 8; ++ni) {
          const int n = ncol + 8 * ni + gq;
          b[ni][0] = ld_mn_tf32<Cfg::BOX_BYTES>(sB, n, k + tq);
          b[ni][1] = ld_mn_tf32<Cfg::BOX_BYTES>(sB, n, k + tq + 4);
        }
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
          for (int ni = 0; ni < 8; ++ni) mma_tf32_16x8x8(&acc[(mi * 8 + ni) * 4], a[mi], b[ni]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&L.empty_bar[s]);
    }
  }

  // epilogue: every 32 x 32 chunk of the partial tile is added to the fp32 output with one TMA reduce-add (clipped at the
  // matrix edge by the map); whole chunks beyond n_valid are skipped
  const int n_valid = tile.which ? n_valid1 : n_valid0;
  uint8_t* buf = L.staging + (warp - 4) * 4096;
  float* raw = L.raw + g * 64 * kRawLd;
  auto to_raw = [&](float* rw, int slab) {
    if (F16) {
      wgmma_acc_to_raw(acc, rw, slab, w, lane);
    } else if ((w >> 1) == slab) {  // the two warps whose 64 columns are this slab
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 8; ++ni)
#pragma unroll
          for (int e = 0; e < 4; ++e)
            rw[(32 * (w & 1) + 16 * mi + (lane >> 2) + 8 * (e >> 1)) * kRawLd + 8 * ni + 2 * (lane & 3) + (e & 1)] =
                acc[(mi * 8 + ni) * 4 + e];
    }
  };
  auto chunk_fn = [&](float (&o)[32], int, int r_off, int c_off) {
    const int col = n0 + c_off;
    if (col >= n_valid) return;  // warp-uniform
    if (lane == 0) bulk_wait_read0();  // previous chunk's reduce has finished reading the staging buffer
    __syncwarp();
    stage_row_sw128(buf, lane, o);
    fence_proxy_async();
    __syncwarp();
    if (lane == 0) {
      tma_reduce_add_2d(tmOut, buf, col, m0 + 64 * g + r_off);
      bulk_commit();
    }
  };
  if (!idle) epilogue_slabs(raw, g, w, lane, to_raw, chunk_fn);
  if (lane == 0) bulk_wait0();
  if (SPLIT) {
    __syncwarp();
    cl_sync();  // the producers' cl_sync: all remote arrivals on and multicast writes into this CTA are done
  }
}

// =====================================================================================
// K-major GEMM with fused epilogues (persistent)
// =====================================================================================
__device__ __forceinline__ float cos_reduced(float x) {
  // Cody-Waite reduction to [-pi, pi] (round-to-nearest multiple of 2 pi via the 1.5 * 2^23 trick: FMA pipe only),
  // then the SFU cosine (abs err ~ 5e-7 on the reduced range)
  const float kInv2Pi = 0.15915494309189535f;
  const float k2PiHi = 6.2831854820251465f;      // fp32(2*pi)
  const float k2PiLo = -1.7484555314695172e-7f;  // 2*pi - fp32(2*pi)
  const float kMagic = 12582912.0f;              // 1.5 * 2^23
  const float k = __fadd_rn(__fmaf_rn(x, kInv2Pi, kMagic), -kMagic);
  float r = fmaf(-k, k2PiHi, x);
  r = fmaf(-k, k2PiLo, r);
  return __cosf(r);
}

// fp16 flavour of the staging: thread `lane` owns row `lane` of a 32 x 32 chunk, stored as 64 B rows without swizzle
// (the matching tensor map is {32, 32} fp16, SWIZZLE_NONE).
__device__ __forceinline__ void stage_row_f16(uint8_t* buf, int lane, const float (&o)[32]) {
  uint4* row = reinterpret_cast<uint4*>(buf + lane * 64);
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    __half2 h0 = __floats2half2_rn(o[8 * c + 0], o[8 * c + 1]);
    __half2 h1 = __floats2half2_rn(o[8 * c + 2], o[8 * c + 3]);
    __half2 h2 = __floats2half2_rn(o[8 * c + 4], o[8 * c + 5]);
    __half2 h3 = __floats2half2_rn(o[8 * c + 6], o[8 * c + 7]);
    uint4 v;
    v.x = *reinterpret_cast<uint32_t*>(&h0);
    v.y = *reinterpret_cast<uint32_t*>(&h1);
    v.z = *reinterpret_cast<uint32_t*>(&h2);
    v.w = *reinterpret_cast<uint32_t*>(&h3);
    row[c] = v;
  }
}

// split flavour: v = hi + lo with hi = fp16(v), lo = fp16(v - hi); hi rows at buf, lo rows at buf + 2048 (same 64 B row layout)
__device__ __forceinline__ void stage_row_f16x2(uint8_t* buf, int lane, const float (&o)[32]) {
  uint4* row_hi = reinterpret_cast<uint4*>(buf + lane * 64);
  uint4* row_lo = reinterpret_cast<uint4*>(buf + 2048 + lane * 64);
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    uint32_t wh[4], wl[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float a = o[8 * c + 2 * e], b = o[8 * c + 2 * e + 1];
      const __half2 h = __floats2half2_rn(a, b);
      const float2 hf = __half22float2(h);
      const __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
      wh[e] = *reinterpret_cast<const uint32_t*>(&h);
      wl[e] = *reinterpret_cast<const uint32_t*>(&l);
    }
    row_hi[c] = make_uint4(wh[0], wh[1], wh[2], wh[3]);
    row_lo[c] = make_uint4(wl[0], wl[1], wl[2], wl[3]);
  }
}

// One 32 x 32 chunk of the K-major epilogue: lane holds row row0 + lane, columns col0 + i, as the raw accumulator a[i];
// vs[0, 32) / vs[32, 64) are vec0 / vec1 of those columns.  slot alternates the two 2 KB halves of the staging buffer for
// single fp16 outputs, so that one store may still be reading while the next chunk is staged.
template <int EPI, int OUT16>
__device__ __forceinline__ void km_chunk(const KmParams& p, const CUtensorMap* tmOut, const CUtensorMap* tmOut2, const float (&a)[32],
                                         const float* vs, uint8_t* sbuf, int slot, int row0, int col0, int lane, float ascale) {
  const float* v0s = vs;
  const float* v1s = vs + 32;
  float o[32];
  if (EPI == EPI_COS) {
    // cosine random feature, or (KM_FLAG_RECT) a rectified linear feature max(floor, z - alpha): PaddedFFT + LinearRectifier.
    // The value summed into colsum must be exactly the stored one: tf32 rounding here; the fp16 slab is rounded once,
    // by the packed conversion of the staging step, and its column sums are taken from the staged halfs.
    if (p.flags & KM_FLAG_RECT) {
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const float val = fmaxf(p.rect_floor, fmaf(a[i], ascale, -v0s[i])) - v1s[i];
        o[i] = OUT16 ? val : ((p.flags & KM_FLAG_NO_ROUND) ? val : round_tf32(val));
      }
    } else if (p.flags & KM_FLAG_NO_ROUND) {  // unrounded output (parity mode, materialised features): exact range reduction
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] = cos_reduced(fmaf(a[i], ascale, v0s[i])) - v1s[i];
    } else {
      // 10-bit slabs: cos.approx on the raw argument (its own range reduction costs ~6e-8 |z| of phase: 1e-6 at |z| = 16,
      // three orders below the operand rounding) saves the four Cody-Waite instructions per element
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const float val = __cosf(fmaf(a[i], ascale, v0s[i])) - v1s[i];
        o[i] = OUT16 ? val : round_tf32(val);
      }
    }
  } else if (EPI == EPI_UPDATE) {
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = v0s[i] - a[i] * ascale;
  } else if (EPI == EPI_APPLY) {
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = v0s[i] + a[i] * ascale;
  } else if (EPI == EPI_RBF) {
    // squared distance from the norms and the cross product; full-precision expf (the value is stored as a 21-bit pair)
    const float ni = row0 + lane < p.M ? __ldg(p.row_vec + row0 + lane) : 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = expf(-p.gamma * fmaxf(0.f, ni + v0s[i] - 2.f * a[i] * ascale));
  }
  if (EPI == EPI_POOL) {
    // Convolver -> SymmetricRectifier -> sum Pooler: the chunk (32 patch rows x 32 filters) is transposed through the staging
    // buffer; lane c then owns filter column c and walks the 32 rows, adding max(floor, +-v - alpha) into the pools the row's
    // patch position belongs to (bit mask per position; rows of a chunk may belong to two images), and flushes the pool
    // sums of an image with fp32 atomics into out[img][pool * 2 N + {0, N} + filter] (the ImageVectorizer order).
    uint8_t* buf = sbuf;
    const int grow = row0 + lane;
    const int my_img = grow / p.patches_per_image;
    const unsigned my_mask = grow < p.M ? __ldg(p.pool_mask + (grow - my_img * p.patches_per_image)) : 0u;
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = a[i] * ascale;
    __syncwarp();
    stage_row_sw128(buf, lane, o);
    __syncwarp();
    const int f = col0 + lane;
    // pool loops are compile-time unrolled over 4 (the CIFAR geometry: 2 x 2 pools) or 16 accumulator pairs
    auto run = [&](auto np_tag) {
      constexpr int NP = decltype(np_tag)::value;
      float ap[NP], an[NP];
#pragma unroll
      for (int pl = 0; pl < NP; ++pl) ap[pl] = an[pl] = 0.f;
      int cur = __shfl_sync(0xffffffffu, my_img, 0);
      unsigned touched = 0;
      auto flush = [&](int img) {
        if (f < p.N && touched) {
          float* dst = p.pool_out + static_cast<int64_t>(img) * p.pool_out_ld + f;
#pragma unroll
          for (int pl = 0; pl < NP; ++pl)
            if (touched >> pl & 1) {
              atomicAdd(dst + static_cast<int64_t>(pl) * 2 * p.N, ap[pl]);
              atomicAdd(dst + static_cast<int64_t>(pl) * 2 * p.N + p.N, an[pl]);
              ap[pl] = an[pl] = 0.f;
            }
        }
        touched = 0;
      };
#pragma unroll 1
      for (int r = 0; r < 32; ++r) {
        const int im = __shfl_sync(0xffffffffu, my_img, r);
        const unsigned mk = __shfl_sync(0xffffffffu, my_mask, r);
        if (im != cur) {  // warp-uniform
          flush(cur);
          cur = im;
        }
        if (mk) {
          const float val = *reinterpret_cast<const float*>(buf + r * 128 + ((((lane >> 2) ^ (r & 7)) << 4) | ((lane & 3) << 2)));
          const float pos = fmaxf(p.rect_floor, val - p.pool_alpha), neg = fmaxf(p.rect_floor, -val - p.pool_alpha);
#pragma unroll
          for (int pl = 0; pl < NP; ++pl)
            if (mk >> pl & 1) {
              ap[pl] += pos;
              an[pl] += neg;
            }
          touched |= mk;
        }
      }
      flush(cur);
    };
    if (p.n_pools <= 4) run(std::integral_constant<int, 4>{});
    else run(std::integral_constant<int, 16>{});
    __syncwarp();
    return;  // no TMA store for this epilogue
  }
  if (EPI == EPI_COS && p.colsum != nullptr && row0 + lane >= p.M) {
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;  // rows past the end must not pollute the column sums
  }
  uint8_t* buf = OUT16 == 1 ? sbuf + slot * 2048 : sbuf;  // an fp16 chunk is 2 KB; the hi + lo pair fills both halves
  if (lane == 0) {  // the store that last used this staging slot has finished reading it
    if (OUT16 == 1) bulk_wait_read1();
    else bulk_wait_read0();
  }
  __syncwarp();
  if (OUT16 == 2) stage_row_f16x2(buf, lane, o);
  else if (OUT16 == 1) stage_row_f16(buf, lane, o);
  else stage_row_sw128(buf, lane, o);
  fence_proxy_async();
  __syncwarp();
  if (lane == 0) {
    if (OUT16 == 2) {
      tma_store_2d(tmOut, buf, col0, row0);
      tma_store_2d(tmOut2, buf + 2048, col0, row0);
    } else if (p.flags & KM_FLAG_REDUCE) {
      tma_reduce_add_2d(tmOut, buf, col0, row0);
    } else {
      tma_store_2d(tmOut, buf, col0, row0);
    }
    bulk_commit();
  }
  if (EPI == EPI_COS && p.colsum != nullptr) {
    // column sums of the chunk straight from the staged copy: lane c adds column c over the 32 rows
    float cs = 0.f;
    if (OUT16 == 2) {
      // p.colsumsq: the exact Gram diagonal, sum of (hi + lo)^2 in fp64 (two partial sums: half the dependent DFMA chain)
      double sq[2] = {0.0, 0.0};
#pragma unroll
      for (int r = 0; r < 32; ++r) {
        const float h = __half2float(*reinterpret_cast<const __half*>(buf + r * 64 + lane * 2));
        const float l = __half2float(*reinterpret_cast<const __half*>(buf + 2048 + r * 64 + lane * 2));
        cs += h + l;
        if (p.colsumsq != nullptr) {
          const double v = static_cast<double>(h) + static_cast<double>(l);
          sq[r & 1] = fma(v, v, sq[r & 1]);
        }
      }
      if (p.colsumsq != nullptr && col0 + lane < p.N) atomicAdd(p.colsumsq + col0 + lane, sq[0] + sq[1]);
    } else if (OUT16 == 1) {
#pragma unroll
      for (int r = 0; r < 32; ++r) cs += __half2float(*reinterpret_cast<const __half*>(buf + r * 64 + lane * 2));
    } else {
      // (row r keeps 16 B chunk j at (j ^ (r & 7)): 32 lanes read 32 distinct words of one 128 B row, no conflicts)
#pragma unroll
      for (int r = 0; r < 32; ++r)
        cs += *reinterpret_cast<const float*>(buf + r * 128 + ((((lane >> 2) ^ (r & 7)) << 4) | ((lane & 3) << 2)));
    }
    const int n = col0 + lane;
    if (n < p.N) atomicAdd(p.colsum + n, cs);
  }
}

// F16: fp16 operands (64 K-elements per 128 B row, K = 16 per wgmma), else tf32 (32 per row, K = 8).  A stage is the
// 128 x 128 B A tile and the 128 x 128 B B tile, both K-major with 128 B swizzle.  OUT16 (EPI_COS only): 1 = the slab is
// written as fp16 (tmOut: {32, 32} fp16 boxes, no swizzle), 2 = as two fp16 planes hi + lo of the unrounded value
// (tmOut / tmOut2), the operand pair of the split-operand Gram and update.
// SPLIT (fp16 pairs): a stage holds A_hi, A_lo, B_hi, B_lo with 32 K-elements each (64 B rows, 64 B swizzle, 8 KB per tile);
// A_hi B_hi^T accumulates on its own, A_lo B_hi^T + A_hi B_lo^T in a second accumulator, and their fp32 sum goes through the
// epilogue once.
// Slab producers (km_async): 512 threads, warpgroup 3 runs the epilogue (see KmSmem).
template <int EPI, bool F16, int OUT16, bool SPLIT>
__global__ void __launch_bounds__(km_threads(EPI), 1)
gemm_kmajor_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   const __grid_constant__ CUtensorMap tmOut, const __grid_constant__ CUtensorMap tmOut2,
                   const __grid_constant__ CUtensorMap tmAlo, const __grid_constant__ CUtensorMap tmBlo, KmParams p) {
  static_assert(!SPLIT || F16, "split operands are fp16 pairs");
  constexpr bool ASYNC = km_async(EPI);
  static_assert(!(ASYNC && SPLIT), "the split update keeps its in-place epilogue");
  constexpr int ROW_BYTES = SPLIT ? 64 : 128;     // one swizzle row of K
  constexpr int BK = ROW_BYTES / (F16 ? 2 : 4);   // K elements per stage
  constexpr int A_BYTES = kTileM * ROW_BYTES;
  extern __shared__ uint8_t smem_raw[];
  const KmSmem L = carve_km_smem<ASYNC>(smem_raw);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int m_tiles = (p.M + kTileM - 1) / kTileM;
  const int n_tiles = (p.N + kTileN - 1) / kTileN;
  // SPLIT: clusters of two CTAs walk pairs of tiles (m, 2 q) and (m, 2 q + 1), which share the slab rows A_m; rank r computes
  // tile (m, 2 q + r), or nothing when that column tile is past the end (odd n_tiles)
  // (in a 1D grid of (2, 1, 1) clusters the rank is blockIdx.x & 1: a special register read, which the compiler may repeat instead
  // of keeping it live beside the two accumulators)
  const int n_pairs = (n_tiles + 1) / 2;
  const uint32_t rank = SPLIT ? (blockIdx.x & 1) : 0;
  const int total_tiles = SPLIT ? m_tiles * n_pairs : m_tiles * n_tiles;
  const int ksteps = (p.K + BK - 1) / BK;
  auto tile_m0 = [&](int t) { return (t / (SPLIT ? n_pairs : n_tiles)) * kTileM; };
  auto tile_n0 = [&](int t) { return SPLIT ? (2 * (t % n_pairs) + static_cast<int>(rank)) * kTileN : (t % n_tiles) * kTileN; };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (SPLIT) {
      tma_prefetch_desc(&tmAlo);
      tma_prefetch_desc(&tmBlo);
    }
    tma_prefetch_desc(&tmOut);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&L.full_bar[s], 1);
      mbar_init(&L.empty_bar[s], SPLIT ? 16 : 8);  // one arrive per consumer warp (SPLIT: of both CTAs of the pair)
    }
    for (int r = 0; r < 8; ++r) mbar_init(&L.ring_bar[r], 1);
    if (ASYNC) {
      mbar_init(L.tile_full, 256);   // every MMA thread, after its part of the accumulator
      mbar_init(L.tile_empty, 32 * kEpiWarps);  // every epilogue thread, after its last read of the buffer
    }
    fence_barrier_init();
  }
  if (SPLIT) cl_sync();  // the partner's barriers are initialised before anything lands in or arrives on them
  else __syncthreads();

  // Tile schedule.  With p.tile_counter the CTAs draw tiles from a global counter: a CTA that got its SM late (this kernel is
  // persistent and shares the GPU with the factor / solve chains' kernels) simply takes fewer tiles instead of stretching the
  // whole launch by its late start.  Without a counter the tiles are strided statically.  Either way the producer publishes
  // every tile id (then -1) in an 8-slot ring; the stage ring keeps it within ~kStages tiles of the consumers, so slots are free.
  if (ASYNC && ((warp >= 1 && warp < 4) || warp >= 12)) {
    // epilogue warp e (warps 1-3 -> 0-2, warps 12-16 -> 3-7): rows [32 (e % 4), +32) and chunks 2 (e / 4), 2 (e / 4) + 1 of each tile
    const int e = warp < 4 ? warp - 1 : warp - 9;
    const int rb = e & 3, cb = 2 * (e >> 2);
    uint8_t* sbuf = L.staging + e * 4096;
    const float ascale = p.acc_scale_ptr ? __ldg(p.acc_scale_ptr) * p.acc_scale : p.acc_scale;
    uint32_t staged = 0;  // chunks this warp has stored: single fp16 outputs alternate the two halves of sbuf
    for (uint32_t tl = 0;; ++tl) {
      mbar_wait(L.tile_full, tl & 1);
      const int t = *L.tile_id;
      if (t < 0) break;
      const int m0 = (t / n_tiles) * kTileM;
      const int n0 = (t % n_tiles) * kTileN;
      {  // the tile's vec0 / vec1 columns, once for all epilogue warps (after all of them are done with the previous tile's)
        named_bar_sync(1, 32 * kEpiWarps);
        const int te = 32 * e + lane, which = te >> 7, c = (te >> 5) & 3;
        const float* v = which ? p.vec1 : p.vec0;
        const int n = n0 + 32 * c + lane;
        L.vec[64 * c + 32 * which + lane] = (v && n < p.N) ? __ldg(v + n) : 0.f;
        named_bar_sync(1, 32 * kEpiWarps);
      }
      const uint32_t src = smem_u32(L.tile + (32 * rb + lane) * kTileLd);
#pragma unroll 1
      for (int k = 0; k < 2; ++k) {
        const int c = cb + k;
        const int col0 = n0 + 32 * c;
        if (col0 >= p.N) {  // warp-uniform; columns only run out in the last chunks of a tile
          if (k == 1) mbar_arrive(L.tile_empty);
          continue;
        }
        float o[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) o[i] = lds_f32(src + 4 * (32 * c + i));
        if (k == 1) mbar_arrive(L.tile_empty);  // the MMA warpgroups may dump the next tile
        km_chunk<EPI, OUT16>(p, &tmOut, &tmOut2, o, L.vec + 64 * c, sbuf, staged & 1, m0 + 32 * rb, col0, lane, ascale);
        ++staged;
      }
    }
    if (lane == 0) bulk_wait0();
    return;
  }
  if (wg == 0) {
    if (warp == 0 && elect_one()) {
      uint32_t it = 0, tl = 0;
      // SPLIT: pairs strided statically over the clusters; both CTAs of a cluster walk the same sequence
      int next = SPLIT ? static_cast<int>(blockIdx.x >> 1)
                       : p.tile_counter ? atomicAdd(p.tile_counter, 1) : static_cast<int>(blockIdx.x);
      for (;; ++tl) {
        const int t = next < total_tiles ? next : -1;
        L.tile_ring[tl & 7] = t;
        mbar_arrive(&L.ring_bar[tl & 7]);
        if (t < 0) break;
        next = SPLIT ? t + static_cast<int>(gridDim.x >> 1)
                     : p.tile_counter ? atomicAdd(p.tile_counter, 1) : t + static_cast<int>(gridDim.x);  // latency hides under this tile
        const int m0 = tile_m0(t);
        const int n0 = tile_n0(t);
        const bool idle = SPLIT && n0 >= p.N;
        for (int ks = 0; ks < ksteps; ++ks, ++it) {
          const int s = it % kStages;
          const uint32_t ph = (it / kStages) & 1;
          mbar_wait(&L.empty_bar[s], ph ^ 1);  // SPLIT: released by the consumers of both CTAs (the multicast writes into both)
          mbar_arrive_expect_tx(&L.full_bar[s], idle ? kStageBytes / 2 : kStageBytes);
          uint8_t* sA = L.stages + s * kStageBytes;
          if (SPLIT) {  // A_hi, A_lo, B_hi, B_lo; rank 0 fetches A_hi and rank 1 A_lo for both CTAs of the pair
            if (rank == 0) tma_load_2d_mc(sA, &tmA, &L.full_bar[s], ks * BK, m0, 0x3);
            else tma_load_2d_mc(sA + A_BYTES, &tmAlo, &L.full_bar[s], ks * BK, m0, 0x3);
            if (!idle) {
              tma_load_2d(sA + 2 * A_BYTES, &tmB, &L.full_bar[s], ks * BK, n0);
              tma_load_2d(sA + 3 * A_BYTES, &tmBlo, &L.full_bar[s], ks * BK, n0);
            }
          } else {
            tma_load_2d(sA, &tmA, &L.full_bar[s], ks * BK, m0);
            tma_load_2d(sA + A_BYTES, &tmB, &L.full_bar[s], ks * BK, n0);
          }
        }
      }
    }
    if (SPLIT) {
      __syncwarp();
      cl_sync();  // neither CTA exits while the other may still write into its stages or arrive on its barriers
    }
    return;
  }

  const int g = wg - 1;  // output rows [64 g, +64) of each tile
  const int w = warp & 3;
  float* raw = L.raw + g * 64 * kRawLd;
  float* vs = L.vec + (warp - 4) * 64;
  uint8_t* sbuf = L.staging + (warp - 4) * 4096;
  const float ascale = p.acc_scale_ptr ? __ldg(p.acc_scale_ptr) * p.acc_scale : p.acc_scale;
  uint32_t it = 0;
  for (uint32_t tl = 0;; ++tl) {
    mbar_wait(&L.ring_bar[tl & 7], (tl >> 3) & 1);
    const int t = L.tile_ring[tl & 7];
    if (ASYNC && t < 0) {  // no more tiles: tell the epilogue warpgroup once it has read the last one
      mbar_wait(L.tile_empty, (tl & 1) ^ 1);
      if (threadIdx.x == 128) *L.tile_id = -1;
      mbar_arrive(L.tile_full);
      return;
    }
    if (t < 0) break;
    const int m0 = tile_m0(t);
    const int n0 = tile_n0(t);

    // SPLIT: a stage is released to the producers of both CTAs: each of them refills part of it (the partner's barrier address
    // is formed at the arrive: nothing more stays live beside the two accumulators)
    auto release = [&](int s) {
      mbar_arrive(&L.empty_bar[s]);
      if (SPLIT) mbar_arrive_remote(cl_map_shared(smem_u32(&L.empty_bar[s]), rank ^ 1));
    };
    if (SPLIT && n0 >= p.N) {  // the partner's tile alone: hand each stage back once this CTA's copy of A has landed
      for (int ks = 0; ks < ksteps; ++ks, ++it) {
        const int s = it % kStages;
        mbar_wait(&L.full_bar[s], (it / kStages) & 1);
        if (lane == 0) release(s);
      }
      continue;
    }

    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    if (SPLIT) {
      float acc_x[64];  // A_lo B_hi^T + A_hi B_lo^T
#pragma unroll
      for (int i = 0; i < 64; ++i) acc_x[i] = 0.f;
      wgmma_fence_acc(acc);
      wgmma_fence_acc(acc_x);
      int prev = -1;
      for (int ks = 0; ks < ksteps; ++ks, ++it) {
        const int s = it % kStages;
        mbar_wait(&L.full_bar[s], (it / kStages) & 1);
        const uint32_t sAhi = smem_u32(L.stages + s * kStageBytes) + g * 64 * ROW_BYTES;  // this warpgroup's 64 rows of A
        const uint32_t sAlo = sAhi + A_BYTES;
        const uint32_t sBhi = smem_u32(L.stages + s * kStageBytes) + 2 * A_BYTES, sBlo = sBhi + A_BYTES;
        wgmma_fence();
        // K-major, 64 B swizzle: 8-row groups are 512 B apart (SBO); K advances 32 B (16 fp16) per instruction
#pragma unroll
        for (int kk = 0; kk < 2; ++kk)
          wgmma_f16_n128<0, 0>(acc, make_wgmma_desc<2>(sAhi + kk * 32, 16, 512), make_wgmma_desc<2>(sBhi + kk * 32, 16, 512), 1);
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {
          wgmma_f16_n128<0, 0>(acc_x, make_wgmma_desc<2>(sAlo + kk * 32, 16, 512), make_wgmma_desc<2>(sBhi + kk * 32, 16, 512), 1);
          wgmma_f16_n128<0, 0>(acc_x, make_wgmma_desc<2>(sAhi + kk * 32, 16, 512), make_wgmma_desc<2>(sBlo + kk * 32, 16, 512), 1);
        }
        wgmma_commit();
        if (prev >= 0) {
          wgmma_wait<1>();
          if (lane == 0) release(prev);
        }
        prev = s;
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      wgmma_fence_acc(acc_x);
      if (prev >= 0 && lane == 0) release(prev);
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = __fadd_rn(acc[i], acc_x[i]);
    } else {
      wgmma_fence_acc(acc);
      int prev = -1;
      for (int ks = 0; ks < ksteps; ++ks, ++it) {
        const int s = it % kStages;
        mbar_wait(&L.full_bar[s], (it / kStages) & 1);
        const uint32_t sA = smem_u32(L.stages + s * kStageBytes) + g * 64 * 128;  // this warpgroup's 64 rows of A
        const uint32_t sB = smem_u32(L.stages + s * kStageBytes) + A_BYTES;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          // K-major, 128 B swizzle: 8-row groups are 1024 B apart (SBO); K advances 32 B (8 tf32 / 16 fp16) per instruction
          const uint64_t ad = make_wgmma_desc(sA + kk * 32, 16, 1024);
          const uint64_t bd = make_wgmma_desc(sB + kk * 32, 16, 1024);
          if (F16) wgmma_f16_n128<0, 0>(acc, ad, bd, 1);
          else wgmma_tf32_n128(acc, ad, bd, 1);
        }
        wgmma_commit();
        if (prev >= 0) {
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&L.empty_bar[prev]);
        }
        prev = s;
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (prev >= 0 && lane == 0) mbar_arrive(&L.empty_bar[prev]);
    }

    if (ASYNC) {
      mbar_wait(L.tile_empty, (tl & 1) ^ 1);  // the epilogue warpgroup has read the previous tile
      wgmma_acc_to_tile(acc, smem_u32(L.tile), g, w, lane);
      if (threadIdx.x == 128) *L.tile_id = t;
      mbar_arrive(L.tile_full);
      continue;
    }
    auto to_raw = [&](float* rw, int slab) { wgmma_acc_to_raw(acc, rw, slab, w, lane); };
    auto chunk_fn = [&](float (&o)[32], int slab, int r_off, int c_off) {
      const int col0 = n0 + c_off;
      if (col0 >= p.N) return;  // warp-uniform
      __syncwarp();  // the previous chunk's reads of vs are done
      vs[lane] = (p.vec0 && col0 + lane < p.N) ? __ldg(p.vec0 + col0 + lane) : 0.f;
      vs[32 + lane] = (p.vec1 && col0 + lane < p.N) ? __ldg(p.vec1 + col0 + lane) : 0.f;
      __syncwarp();
      km_chunk<EPI, OUT16>(p, &tmOut, &tmOut2, o, vs, sbuf, slab & 1, m0 + 64 * g + r_off, col0, lane, ascale);
    };
    epilogue_slabs(raw, g, w, lane, to_raw, chunk_fn);
  }
  if (lane == 0) bulk_wait0();
  if (SPLIT) {
    __syncwarp();
    cl_sync();  // the producers' cl_sync: all remote arrivals on and multicast writes into this CTA are done
  }
}

// =====================================================================================
// Host-side launchers
// =====================================================================================
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// 2D fp32 row-major matrix [rows x cols], leading dimension ld (floats); box = {32 floats, box_rows}, 128B swizzle
int make_tmap_2d(CUtensorMap* out, const float* base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  return make_tmap_any(out, base, rows, cols, ld, 32, box_rows, 4, TMAP_SW128);
}

// General form: elem_bytes 4 (fp32 / tf32) or 2 (fp16); ld in elements; box {box_cols, box_rows}.
int make_tmap_any(CUtensorMap* out, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_cols, int box_rows,
                  int elem_bytes, int swizzle) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return -1;
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * static_cast<cuuint64_t>(elem_bytes)};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1u, 1u};
  const CUtensorMapSwizzle sw = swizzle == TMAP_SW128  ? CU_TENSOR_MAP_SWIZZLE_128B
                                : swizzle == TMAP_SW64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                       : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = fn(out, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                  const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -static_cast<int>(r) - 1000;
}

// The kernels of one family share a signature, so the "attribute set" flag lives in each launcher instantiation.
template <typename K>
static cudaError_t set_smem_attr_once(K kern, bool& done, int bytes = kSmemBytes) {
  if (!done) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return e;
    done = true;
  }
  return cudaSuccess;
}

static cudaLaunchConfig_t pair_config(unsigned grid, int smem, cudaStream_t st, cudaLaunchAttribute* attr) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = static_cast<size_t>(smem);
  cfg.stream = st;
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cfg;
}
// The split kernels run as clusters of two CTAs (grid even).
template <typename K, typename... Args>
static cudaError_t launch_pairs(K kern, unsigned grid, int smem, cudaStream_t st, Args... args) {
  cudaLaunchAttribute attr[1];
  const cudaLaunchConfig_t cfg = pair_config(grid, smem, st, attr);
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, args...);
  return e != cudaSuccess ? e : cudaGetLastError();
}
// How many pairs of a kernel can be resident at once: a cluster's two CTAs sit in one GPC, so on a GPC with an odd number of
// free SMs one SM stays out and the count may be below num_sms / 2.  The persistent split update takes no more, or the pairs
// that did not fit would start only when others finish, after a whole launch's worth of tiles.
template <typename K>
static cudaError_t resident_pairs(K kern, int smem, int num_sms, int* pairs) {
  cudaLaunchAttribute attr[1];
  const cudaLaunchConfig_t cfg = pair_config(static_cast<unsigned>(std::max(2, num_sms & ~1)), smem, nullptr, attr);
  int n = 0;
  const cudaError_t e = cudaOccupancyMaxActiveClusters(&n, kern, &cfg);
  if (e != cudaSuccess) return e;
  *pairs = std::max(1, std::min(n, num_sms / 2));
  return cudaSuccess;
}

template <bool F16, bool SPLIT>
static cudaError_t launch_gram_t(const GramLaunch& g, cudaStream_t st) {
  if (g.chunk_rows % GramCfg<F16, SPLIT>::SR != 0) return cudaErrorInvalidValue;
  auto kern = gram_tn_kernel<F16, SPLIT>;
  static bool attr_done = false;
  cudaError_t e = set_smem_attr_once(kern, attr_done);
  if (e != cudaSuccess) return e;
  const int chunks = (g.rows + g.chunk_rows - 1) / g.chunk_rows;
  const unsigned grid = static_cast<unsigned>(chunks) * static_cast<unsigned>(g.num_tiles);
  if (grid == 0) return cudaSuccess;
  if (SPLIT) {  // CTA pairs: g.tiles holds two entries per pair, so the grid is chunks x pairs x 2
    if (g.num_tiles % 2 != 0) return cudaErrorInvalidValue;
    return launch_pairs(kern, grid, kSmemBytes, st, g.tmA, g.tmB0, g.tmB1, g.tmOut0, g.tmOut1, g.tmAlo, g.tmB0lo, g.tmB1lo, g.tiles,
                        g.num_tiles, g.rows, g.chunk_rows, g.n_valid0, g.n_valid1);
  }
  kern<<<grid, kThreads, kSmemBytes, st>>>(g.tmA, g.tmB0, g.tmB1, g.tmOut0, g.tmOut1, SPLIT ? g.tmAlo : g.tmA, SPLIT ? g.tmB0lo : g.tmB0,
                                           SPLIT ? g.tmB1lo : g.tmB1, g.tiles, g.num_tiles, g.rows, g.chunk_rows, g.n_valid0, g.n_valid1);
  return cudaGetLastError();
}

cudaError_t launch_gram(const GramLaunch& g, cudaStream_t st) {
  if (g.split) return g.f16 ? launch_gram_t<true, true>(g, st) : cudaErrorInvalidValue;
  return g.f16 ? launch_gram_t<true, false>(g, st) : launch_gram_t<false, false>(g, st);
}

template <int EPI, bool F16, int OUT16, bool SPLIT = false>
static cudaError_t launch_km_t(const KmLaunch& k, cudaStream_t st) {
  auto kern = gemm_kmajor_kernel<EPI, F16, OUT16, SPLIT>;
  static bool attr_done = false;
  cudaError_t e = set_smem_attr_once(kern, attr_done, km_smem_bytes(EPI));
  if (e != cudaSuccess) return e;
  const int m_tiles = (k.p.M + kTileM - 1) / kTileM;
  const int n_tiles = (k.p.N + kTileN - 1) / kTileN;
  const long long total = static_cast<long long>(m_tiles) * n_tiles;
  if (total == 0) return cudaSuccess;
  if (SPLIT) {  // clusters of two CTAs, one pair of column tiles at a time, at most as many as fit on the GPU at once
    if (k.p.tile_counter) return cudaErrorInvalidValue;  // the pairs are strided statically
    static int fit = 0;
    if (!fit) {
      e = resident_pairs(kern, km_smem_bytes(EPI), k.num_sms, &fit);
      if (e != cudaSuccess) return e;
    }
    const long long pairs = static_cast<long long>(m_tiles) * ((n_tiles + 1) / 2);
    const unsigned grid = 2u * static_cast<unsigned>(std::min<long long>(pairs, std::min(fit, std::max(1, k.num_sms / 2))));
    return launch_pairs(kern, grid, km_smem_bytes(EPI), st, k.tmA, k.tmB, k.tmOut, k.tmOut, k.tmAlo, k.tmBlo, k.p);
  }
  const unsigned grid = static_cast<unsigned>(total < k.num_sms ? total : k.num_sms);
  kern<<<grid, km_threads(EPI), km_smem_bytes(EPI), st>>>(k.tmA, k.tmB, k.tmOut, OUT16 == 2 ? k.tmOut2 : k.tmOut, SPLIT ? k.tmAlo : k.tmA,
                                           SPLIT ? k.tmBlo : k.tmB, k.p);
  return cudaGetLastError();
}

cudaError_t launch_kmajor(const KmLaunch& k, cudaStream_t st) {
  if (k.split) return (k.f16 && k.epi == EPI_UPDATE) ? launch_km_t<EPI_UPDATE, true, 0, true>(k, st) : cudaErrorInvalidValue;
  if (k.epi == EPI_POOL) return k.f16 ? launch_km_t<EPI_POOL, true, 0>(k, st) : cudaErrorInvalidValue;
  if (k.epi == EPI_RBF) return (k.f16 && k.out16 == 2) ? launch_km_t<EPI_RBF, true, 2>(k, st) : cudaErrorInvalidValue;
  if (k.f16 && k.epi == EPI_APPLY) return launch_km_t<EPI_APPLY, true, 0>(k, st);
  if (k.f16 && k.epi == EPI_UPDATE) return launch_km_t<EPI_UPDATE, true, 0>(k, st);
  if (k.out16 == 2 && k.epi == EPI_COS) return k.f16 ? launch_km_t<EPI_COS, true, 2>(k, st) : cudaErrorInvalidValue;
  if (k.out16 && k.f16 && k.epi == EPI_COS) return launch_km_t<EPI_COS, true, 1>(k, st);
  if (k.f16 && k.epi == EPI_COS) return launch_km_t<EPI_COS, true, 0>(k, st);  // fp16 operands, fp32 slab (split mode, tf32 pairs)
  if (k.out16 && k.epi == EPI_COS) return launch_km_t<EPI_COS, false, 1>(k, st);
  switch (k.epi) {
    case EPI_COS: return launch_km_t<EPI_COS, false, 0>(k, st);
    case EPI_UPDATE: return launch_km_t<EPI_UPDATE, false, 0>(k, st);
    case EPI_APPLY: return launch_km_t<EPI_APPLY, false, 0>(k, st);
    default: return cudaErrorInvalidValue;
  }
}

unsigned int read_wait_timeout_flag() {
  unsigned int v = 0;
  cudaMemcpyFromSymbol(&v, g_wait_timeout_flag, sizeof(v));
  return v;
}

}  // namespace ks
