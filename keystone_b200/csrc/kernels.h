// Internal (C++) interface between the host engine (engine.cu) and the CUDA kernels.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ks {

static constexpr int kGramStageRows = 32;  // rows per TMA stage of the Gram kernel
static constexpr int kPadCols = 32;        // every device matrix has ld % 32 == 0 (128 B rows)

enum { EPI_COS = 0, EPI_UPDATE = 1, EPI_APPLY = 2, EPI_POOL = 3, EPI_RBF = 4 };

// Split Gram: its CTAs run in pairs (clusters of two) whose tiles share one operand panel, and the list holds two entries per
// pair in rank order.  pair = 0: the two tiles share A's panel (same m_blk); GRAM_SHARE_B: they share B's (same n_blk, same
// which); GRAM_IDLE: the entry has no tile of its own (a lone tile's partner) and repeats its partner's tile.
enum { GRAM_SHARE_B = 1, GRAM_IDLE = 2 };
struct GramTile {
  int m_blk;  // 128-wide block of A's columns
  int n_blk;  // 128-wide block of B's columns
  int which;  // 0: B = tmB0 -> out0,  1: B = tmB1 -> out1
  int pair;   // split Gram only: GRAM_SHARE_B | GRAM_IDLE
};
struct GramLaunch {
  CUtensorMap tmA, tmB0, tmB1;   // operands: tf32 box {32, kGramStageRows}, fp16 box {64, 64} (split: {64, 32}); SWIZZLE_128B
  CUtensorMap tmOut0, tmOut1;    // outputs:  box {32, 32}, SWIZZLE_128B; dims clip the reduce-add at the matrix edge
  CUtensorMap tmAlo, tmB0lo, tmB1lo;  // split only: the lo planes of A, B0, B1 (same geometry as the hi maps)
  const GramTile* tiles;         // device
  int num_tiles;                 // entries of tiles (split: two per CTA pair)
  int rows;        // contraction length (rows of A and B)
  int chunk_rows;  // split of the contraction across CTAs (multiple of the stage rows)
  int n_valid0, n_valid1;  // valid output columns per target (whole 32-column chunks beyond are skipped)
  int f16 = 0;             // 1: operands are fp16 (wgmma, 64-row stages), 0: tf32 (mma.sync, 32-row stages)
  int split = 0;           // 1 (f16 only): operands are fp16 pairs hi + lo, one pass computes hi^T hi + lo^T hi + hi^T lo
};
enum { KM_FLAG_NO_ROUND = 1, KM_FLAG_REDUCE = 2, KM_FLAG_RECT = 8 };
struct KmParams {
  const float* vec0;  // EPI_COS: bias (KM_FLAG_RECT: alpha);  EPI_UPDATE / EPI_APPLY: per-column constant
  float rect_floor = 0.f;   // KM_FLAG_RECT: the feature is max(rect_floor, acc - alpha) instead of cos(acc + bias)
  const float* vec1;  // EPI_COS: shift
  float* colsum;      // EPI_COS: if non-null, colsum[n] += sum over valid rows of the stored values (fp32 atomics)
  float acc_scale = 1.f;    // the accumulator is multiplied by this before the epilogue (undoes power-of-two operand scaling)
  const float* acc_scale_ptr = nullptr;  // optional device scalar multiplied into acc_scale (scale chosen on the device)
  // EPI_POOL (Convolver -> SymmetricRectifier -> sum Pooler -> ImageVectorizer, fused): rows are image patches (patches_per_image
  // consecutive rows per image), columns are filters; out[img][pool * 2 N + {0, N} + filter] += max(floor, +-acc - alpha)
  const unsigned* pool_mask = nullptr;  // [patches_per_image] bit p set: the patch position lies in pool p (pools may overlap)
  union {
    float* pool_out = nullptr;
    // EPI_COS with the fp16 pair output (out16 == 2) and colsum: if non-null, colsumsq[n] += sum over valid rows of (hi + lo)^2
    // in fp64, the exact Gram diagonal of the slab.  It shares pool_out's slot so that KmParams, and with it the code of every
    // other instantiation, stays as it was.
    double* colsumsq;
  };
  int64_t pool_out_ld = 0;
  int patches_per_image = 0, n_pools = 0;
  float pool_alpha = 0.f;
  int* tile_counter = nullptr;  // persistent single-CTA kernel: zeroed device counter the CTAs draw their tiles from (null: static stride)
  // EPI_RBF (Gaussian kernel block): out = exp(-gamma * max(0, row_vec[m] + vec0[n] - 2 acc)), row_vec / vec0 the squared norms
  // of the rows of A / B
  const float* row_vec = nullptr;
  float gamma = 0.f;
  int M, N, K;
  int flags;  // KM_FLAG_NO_ROUND: EPI_COS keeps fp32;  KM_FLAG_REDUCE: add into the output instead of overwriting it
};
struct KmLaunch {
  CUtensorMap tmA, tmB;  // operands: box {32, 128} (tf32) / {64, 128} (fp16), SWIZZLE_128B
  CUtensorMap tmOut;     // output: box {32, 32}, SWIZZLE_128B
  CUtensorMap tmOut2;    // out16 == 2 only: the lo plane (same geometry as tmOut)
  CUtensorMap tmAlo, tmBlo;  // split only: lo planes of A and B; then every operand map has box {32, 128}, SWIZZLE_64B
  KmParams p;
  int epi;
  int num_sms;
  int f16 = 0;   // 1: fp16 operands
  int split = 0; // 1 (EPI_UPDATE, f16 only): operands are fp16 pairs, one pass computes A_hi B_hi^T + A_lo B_hi^T + A_hi B_lo^T
  int out16 = 0; // EPI_COS (EPI_RBF: 2 only): 1 = the slab is written as fp16 (tmOut: {32, 32} fp16 boxes, no swizzle); 2 = as the fp16 pair hi + lo
                 // of the unrounded value (tmOut, tmOut2)
};

int make_tmap_2d(CUtensorMap* out, const float* base, int64_t rows, int64_t cols, int64_t ld, int box_rows);
enum { TMAP_SW128 = 0, TMAP_SW64 = 1, TMAP_NONE = 2 };
int make_tmap_any(CUtensorMap* out, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_cols, int box_rows,
                  int elem_bytes, int swizzle);
cudaError_t launch_gram(const GramLaunch& g, cudaStream_t st);
cudaError_t launch_kmajor(const KmLaunch& k, cudaStream_t st);
unsigned int read_wait_timeout_flag();
// B (n x k, column-major, ld = n) <- (L L^T)^-1 B with L the lower triangle of a column-major n x n matrix and Dinv the inverses
// of its 64 x 64 diagonal tiles (launch_tri_inv_tiles; chol_solve_dinv_doubles(n) doubles) -- solve_kernels.cu
cudaError_t launch_chol_solve(const double* L, const double* Dinv, int n, double* B, int k, cudaStream_t st);
cudaError_t launch_tri_inv_tiles(const double* L, int n, double* Dinv, cudaStream_t st);
size_t chol_solve_dinv_doubles(int n);

// ---- element-wise / reduction helpers (aux_kernels.cu) ----
void launch_f32_repitch_rows(const float* src, int64_t src_ld, float* dst, int64_t dst_ld, int64_t rows, int64_t cols,
                             cudaStream_t st);
void launch_f64_to_f32_rows(const double* src, int64_t src_ld, float* dst, int64_t dst_ld, int64_t rows, int64_t cols,
                            cudaStream_t st);
void launch_f32_to_f64_rows(const float* src, int64_t src_ld, double* dst, int64_t dst_ld, int64_t rows, int64_t cols,
                            cudaStream_t st);
void launch_labels_from_classes(const int32_t* cls, float* dst, int64_t ld, int64_t rows, int k, cudaStream_t st);
// column sums of [rows x cols] (optionally hi + lo planes) accumulated into fp64 sums[cols] (must be zeroed)
void launch_colsum(const float* hi, const float* lo, int64_t ld, int64_t rows, int cols, double* sums, cudaStream_t st);
// residual initialisation: R[:, :k] = Y - ymean (fp32 master copy), other columns 0
void launch_init_residual(const float* Y, int64_t ldy, const double* ymean, float* R, int64_t ldr, int64_t rows, int k,
                          cudaStream_t st);
// Rr[:, :k] = tf32_rn(R[:, :k]) (the Gram's MN-major operand), Rr[:, k] = 1 (ones column), Rr[:, > k] = 0, and
// sums[c] += column sums of R (fp64; must be zeroed) -- one pass over R per block
void launch_round_colsum(const float* R, float* Rr, int64_t ld, int64_t rows, int k, double* sums, cudaStream_t st,
                         float* Rlo = nullptr);  // Rlo (split-operand mode): tf32(R - Rr)
// slab[:, :cols] = tf32(F[:, c0:c0+cols] - shift); if colsum != null, colsum[c] += column sums of the slab (fp32 atomics)
void launch_center_round(const float* F, int64_t ldf, int c0, const float* shift, float* slab, float* colsum, int64_t lds,
                         int64_t rows, int cols, cudaStream_t st, float* slab_lo = nullptr);  // slab_lo: tf32(v - slab), split mode
// out[i] = float(sums[i] / *count) (and out64 if non-null); the count lives on the device (no host round trip)
void launch_divide_by_count(const double* sums, const double* count, float* out, double* out64, int n, cudaStream_t st);
// delta[i] = double(ssum[i]) / n_total ; mean[i] = shift[i] + delta[i]
void launch_delta_mean(const float* ssum, const float* shift, double n_total, double* delta, double* mean, int b, cudaStream_t st);
// H (fp64, column-major b x b, ld = b) = sym(G) - n * delta delta^T + lam * I
void launch_build_system(const float* G, int ldg, const double* delta, double n_total, double lam, double* H, int b,
                         cudaStream_t st, const float* cross = nullptr,  // cross: S_hi^T S_lo (full b x b, ld = ldg), split mode
                         const double* exact_diag = nullptr);            // split mode: the diagonal from launch_colsumsq_pair
// out[c] (fp64, zeroed) += sum_r (hi[r][c] + lo[r][c])^2: the Gram diagonal of a split slab (fp16 or fp32 planes, ld elements)
void launch_colsumsq_pair(const void* hi, const void* lo, bool f16, int64_t ld, int64_t rows, int cols, double* out, cudaStream_t st);
// RHS (fp64 column-major b x k, ld = b) = C[:, :k] - n * delta * rbar^T - lam * Wold
void launch_build_rhs(const float* C, int ldc, const double* delta, const double* rsum, double n_total, double lam,
                      const double* Wold, double* rhs, int b, int k, cudaStream_t st, const float* c_scale = nullptr);
// Wmodel += dW;  Bop_hi/lo [kpad x ldb] = split(dW^T);  cbias[c] = sum_f delta[f] dW[f][c]
void launch_pack_update(const double* dW, double* Wmodel, const double* delta, float* bop_hi, float* bop_lo, int ldb,
                        float* cbias, int b, int k, int kpad, cudaStream_t st);
// Bop hi (/ lo) [kpad x ldb] = split(W^T) for apply; cbias[c] = (intercept ? intercept[c] : 0) - sum_f (mean[f] - shift32[f]) W[f][c]
void launch_pack_apply(const double* W, const double* mean_or_null, const float* shift32, const double* intercept_or_null,
                       float* bop_hi, float* bop_lo, int ldb, float* cbias, int b, int k, int kpad, cudaStream_t st);
void launch_argmax_rows(const float* Y, int64_t ld, int64_t rows, int k, int32_t* out, cudaStream_t st);
// counts[actual * k + predicted] += 1 over n samples (counts must be zeroed); out-of-range classes are skipped
void launch_confusion(const int32_t* pred, const int32_t* act, int64_t n, int k, unsigned long long* counts, cudaStream_t st);
void launch_sq_err(const float* Y, int64_t ldy, const float* L, int64_t ldl, int64_t rows, int k, double* out,
                   cudaStream_t st);
void launch_fill_f32(float* p, int64_t n, float v, cudaStream_t st);
void launch_normal_f32(float* dst, int64_t ld, int64_t rows, int cols, uint64_t seed, int64_t row_offset, float mean,
                       float stddev, cudaStream_t st);
void launch_w_to_operand(const double* W_colmajor, int64_t n_out, int64_t n_in, float* dst, int64_t ld, cudaStream_t st,
                         bool round = true);  // round: tf32 round-to-nearest (MMA operand); false: plain fp32
void launch_f64_to_f32_vec(const double* src, float* dst, int64_t n, cudaStream_t st);
// Convolver.makePatches + Stats.normalizeRows + whitener means (K/nodes/images/Convolver.scala:152-203, K/utils/Stats.scala:112-123):
// images [n][x_dim * y_dim * ch] fp32 in ImageVectorizer order (c + x*ch + y*ch*x_dim) -> fp16 patch rows [n * resW * resH][ld],
// row = img * resW * resH + x + y * resW, column c + pox*ch + poy*ch*conv; concat3: [hi | lo | hi] along K (split-operand mode)
void launch_im2col_normalize(const float* images, int64_t ld_img, int64_t n_images, int x_dim, int y_dim, int ch, int conv, int normalize,
                             float var_constant, const float* whitener_means, void* out16, int64_t ld_out, int concat3, cudaStream_t st);
// PaddedFFT as a dense map: W[f][n] = signs[n] * cos(2 pi f n / P), f < P / 2, n < n_in (signs may be null = all ones), written
// twice: tf32-rounded (dst) and plain fp32 (dst_full); both [P/2][ld]
void launch_fft_real_matrix(const double* signs, int64_t n_in, int64_t P, float* dst, float* dst_full, int64_t ld, cudaStream_t st);
// elementwise maps on a matrix: op 0: out = x * colvec[c];  op 1: out = max(a, x - b)
void launch_matrix_map(const float* src, float* dst, int64_t ld, int64_t rows, int cols, int op, const float* colvec, float a, float b,
                       cudaStream_t st);
// ---- fp16 operand path: device-chosen power-of-two scales (scale[0] = 2^e, scale[1] = 2^-e) and fp16 operand packers
void launch_max_abs_f32(const float* p, int64_t ld, int64_t rows, int cols, unsigned* maxbits, cudaStream_t st);
void launch_max_abs_f64(const double* p, int64_t n, unsigned* maxbits, cudaStream_t st);
void launch_pow2_scale(const unsigned* maxbits, float target, float* scale, cudaStream_t st);
void launch_f32_to_f16_rows(const float* src, int64_t src_ld, void* dst, int64_t dst_ld, int64_t rows, int64_t cols, cudaStream_t st,
                            const float* scale = nullptr);  // optional device scalar multiplied in before the conversion
void launch_round_colsum16(const float* R, void* R16, int64_t ld, int64_t rows, int k, double* sums, const float* scale,
                           cudaStream_t st, void* R16lo = nullptr, unsigned* overflow = nullptr);  // *overflow = 1 if |R * scale| left fp16's range
void launch_pack_update16(const double* dW, double* Wmodel, const double* delta, void* bop16, int ldb, float* cbias, int b, int k,
                          int kpad, const float* scale, cudaStream_t st, void* bop16_lo = nullptr);
// split-operand mode: the K-concatenated projection operands (the slab pair hi + lo comes out of the projection epilogue)
void launch_split_concat3(const float* src, int64_t ld_src, int64_t rows, int cols, const float* scale, void* dst, int64_t ld_dst,
                          int pattern, cudaStream_t st);

}  // namespace ks
