// b2_internal.cuh -- shared declarations of libb2gram.so (not part of the public C-ABI).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <type_traits>

#include "../../include/b2gram.h"

namespace b2 {

constexpr int kMaxD = B2_MAX_D;          // 128 features
constexpr int kMaxS = kMaxD + 2;         // 130: features, ones, y
constexpr int kKernelEventPairs = 64;
constexpr int kMaxRanks = 8;
constexpr size_t kXchgSlotDoubles = (size_t)kMaxS * kMaxS;                 // one rank's S
constexpr size_t kXchgDataDoubles = 2 * kMaxRanks * kXchgSlotDoubles;       // two epochs (parity) x ranks
constexpr size_t kXchgBytes = kXchgDataDoubles * sizeof(double) + 256;      // + flags[8] (u32) + ticket

// ---- tensor-core Gram kernel geometry (gram_tc.cu) --------------------------------------
constexpr int kTcRows = 64;              // rows of X per pipeline stage (4 MMA K-steps of 16)
constexpr int kTcM = 128;                // MMA M: feature index (zero padded)
constexpr int kTcEMax = 16;              // extra columns E = [1, y'_hi, y'_lo] per packed row: 3 * pack <= 16
// Width of the E block the MMAs cover: 8 columns hold up to pack = 2, 16 up to pack = 5 (kMaxPack).
inline int tc_e_width(int pack) { return pack >= 3 ? 16 : 8; }
// The per-CTA partial of the tensor-core Gram kernel holds, in fp64, exactly the accumulator entries the fold reads.
// Accumulator 0 is D1 = hi^T [hi | E] (RAWB: v^T-exact [x | E], lo added in), accumulator 1 is D2 = lo^T [hi | E]; row i
// is a feature (A side), column j < 128 a feature and j = 128 + e an E column (B side).  With `ew` E columns:
//   [0, kTcTri)                       D1, i <= j < 128: the upper triangle, packed column by column
//   [kTcTri, kTcTri + ew * 128)       D1, E columns
//   then (128 + ew) * 128             D2, every column (written only by hi + lo operands without RAWB)
// The entries a launch writes are the prefix [0, tc_part_elems(ew, d2)).
constexpr int kTcTri = kTcM * (kTcM + 1) / 2;   // 8256
__host__ __device__ constexpr int tc_part_index(int acc, int i, int j, int ew) {
  return acc == 0 ? (j < kTcM ? j * (j + 1) / 2 + i : kTcTri + (j - kTcM) * kTcM + i)
                  : kTcTri + ew * kTcM + j * kTcM + i;
}
__host__ __device__ constexpr int tc_part_elems(int ew, bool d2) {
  return kTcTri + ew * kTcM + (d2 ? (kTcM + ew) * kTcM : 0);
}
constexpr int kTcAccElems = tc_part_elems(kTcEMax, true);   // stride of one CTA's partial (28 736)
constexpr int kTcSums = 3;               // per-CTA CUDA-core sums: sum y', sum y'^2, rows used
// ctx->tc_part of a Gram launch on n_ctas CTAs: [n_ctas][kTcAccElems] fp64 accumulators, then [n_ctas][kTcSums] sums.
// The finalize locates the sums through its n_ctas, which must equal the Gram grid.  Allocated for n_ctas = sm_count.

// ---- scoring (b2_score, b2_metrics) and the refined fit (b2_fit_refined) ---------------------------------------------
constexpr int kNStats = 10;              // include/b2gram.h: b2_score stats_out layout (maxima at 4 and 9, sums elsewhere)
// the refined fit's model y = b0' + (x - m).beta and its residual passes
// one gradient: g_j = sum (x_j - m_j) e at j < kMaxD, g_1 = sum e at kMaxD, and sum e^2 at kMaxD + 1 (b2_residual_moments)
constexpr int kGradOut = kMaxD + 2;
// doubles of ctx->refine
constexpr int kRfBeta = 0;               // beta
constexpr int kRfB0 = kMaxD;             // b0'
constexpr int kRfMean = kMaxD + 1;       // m: S's column means (0 without an intercept)
constexpr int kRfPrevBeta = 2 * kMaxD + 1;   // beta and b0' before the last kept correction (where the guard returns)
constexpr int kRfPrevB0 = 3 * kMaxD + 1;
constexpr int kRfStep = 3 * kMaxD + 2;   // step of the last kept correction (+inf before the first)
constexpr int kRfGrad = 3 * kMaxD + 3;   // the reduced gradient of the current pass [kGradOut]
constexpr int kRfDoubles = kRfGrad + kGradOut;
// solve_out / solve_host slots of the refinement solve (beside coef [0, d), intercept kMaxD, info kMaxD + 1)
constexpr int kOutRefineStep = 2 * kMaxD + 3;
constexpr int kOutRefineGuard = 2 * kMaxD + 4;

// ---- the leave-one-out pass of b2_ridge_loo (ridge_loo.cu) and its eigendecomposition (solve_eigh_kernel) ----------
constexpr int kMaxAlphas = B2_MAX_ALPHAS;
// doubles of ctx->loo
constexpr int kLooQ = 0;                          // Q[i][k], row pitch kMaxD: column k is the eigenvector of eigenvalue k
constexpr int kLooLam = kMaxD * kMaxD;            // eigenvalues, ascending, >= 0
constexpr int kLooMean = kLooLam + kMaxD;         // m: S's column means (0 without an intercept)
constexpr int kLooC = kLooMean + kMaxD;           // c = Q^T r
constexpr int kLooMisc = kLooC + kMaxD;           // [0] ybar, [1] n, [2] h0, [3] 1: the Jacobi sweeps converged
constexpr int kLooAlpha = kLooMisc + 8;           // the alphas of the call [kMaxAlphas]
constexpr int kLooCw = kLooAlpha + kMaxAlphas;    // [kMaxD][kMaxAlphas] c_j / (lambda_j + alpha_a)
constexpr int kLooW = kLooCw + kMaxD * kMaxAlphas;   // [kMaxD][kMaxAlphas] 1 / (lambda_j + alpha_a)
constexpr int kLooSum = kLooW + kMaxD * kMaxAlphas;  // the reduced sums of e^2 per alpha [kMaxAlphas]
constexpr int kLooDoubles = kLooSum + kMaxAlphas;

// ---- the elastic-net paths of b2_solve_enet_path / b2_solve_enet_cv (solve.cu: solve_enet_kernel) --------------------
// Every pointer is into ctx->enet.  alphas: the call's alphas (grid != 0: the kernel writes sklearn's grid there, one row
// of n_alphas per l1_ratio); coef_init: nullptr or d starting coefficients; outputs per path (CTA) and alpha: coefs
// [n_alphas][d], intercepts, gaps (dual gap / n) and iters (as doubles); tol_out per path: tol * y_norm2 / n.
// Cross-validation (folds != nullptr): one path per (l1_ratio l, fold k), CTA l n_folds + k, on the sum of the other
// folds' statistics (folds: [n_folds][(d+2)^2]); mse [n_l1][n_alphas][n_folds] the held-out error from fold k's own.
struct EnetArgs {
  double l1_ratio, eps, tol;
  int n_alphas, grid, max_iter, positive, fit_intercept;
  double* alphas;
  const double* coef_init;
  double *coefs, *intercepts, *gaps, *iters, *tol_out;
  const double* folds = nullptr;
  const double* l1_ratios = nullptr;   // [n_l1]; nullptr: l1_ratio
  int n_folds = 1, n_l1 = 1;
  double* mse = nullptr;
};

// ---- BayesianRidge / ARDRegression (solve.cu: bayes_ridge_kernel, ard_kernel; DESIGN.md section 9) -------------------
// Every pointer is into ctx->enet.  anchor: nullptr or [w0 kMaxD | g0 kMaxD | s0 | sse0] (b2_residual_moments at w0);
// out: kBy* below; scores: max_iter + 1 doubles (written with compute_score); A: ard_kernel's copy of the centred Gram.
constexpr int kByCoef = 0;                       // [kMaxD] coef
constexpr int kByMisc = kMaxD;                   // [0] intercept [1] alpha [2] lambda (BayesianRidge) [3] n_iter [4] info
constexpr int kByLambda = kMaxD + 8;             // [kMaxD] ARD's lambda per feature
constexpr int kBySigma = 2 * kMaxD + 8;          // [d][d] sigma (row-major, pitch d)
constexpr int kByDoubles = kBySigma + kMaxD * kMaxD;
// operands of b2_score_std at ctx->enet: sigma [d][d] (pitch d), m, w, then [0] b + m.w, [1] noise_var
constexpr int kStdSigma = 0;
constexpr int kStdMean = kMaxD * kMaxD;
constexpr int kStdCoef = kStdMean + kMaxD;
constexpr int kStdMisc = kStdCoef + kMaxD;
constexpr int kStdDoubles = kStdMisc + 8;
struct BayesArgs {
  double a1, a2, l1, l2, alpha_init, lambda_init;   // a NaN init: scikit-learn's default
  double threshold_lambda, tol;
  int max_iter, compute_score, fit_intercept;
  const double* anchor;
  double *out, *scores, *A;
};

// ---- the generalised linear regressors (glm.cu; DESIGN.md section 10) -------------------------------------------------
// ctx->glm: the reduced sums [kGlmPart] of the last pass, then the operands at kGlmOp: w [kMaxD], the Newton step [kMaxD],
// [b, db, negative label, positive label].  The sums: [0] loss [1] const [2] sum y [3] rows kept [4] y out of range
// [5] h <= 0 [6] y not finite [7] (logistic passes) rows classified correctly, the
// gradient sum g x_j at kGlmGrad + j (sum g at kGlmGrad + d), the Hessian sum |h| z_i z_j (z = [x 1]) at kGlmHess +
// i kGlmHp + j, i <= j; a line search leaves the loss at step k in [k].  ctx->glm_part holds one kGlmPart per CTA, for
// up to two CTAs per SM.
constexpr int kGlmSteps = 21;            // sklearn's backtracking steps t = 1, 1/2, ..., 2^-20
constexpr int kGlmGrad = 8;
constexpr int kGlmHess = 144;
constexpr int kGlmHp = 144;              // pitch of the Hessian: D + 1 columns padded to 16
constexpr int kGlmPart = kGlmHess + kGlmHp * kGlmHp;
constexpr int kGlmOp = kGlmPart;
constexpr int kGlmOpW = 0, kGlmOpStep = kMaxD, kGlmOpMisc = 2 * kMaxD;
constexpr int kGlmDoubles = kGlmOp + 2 * kMaxD + 8;
enum GlmMode { kGlmGradient = 0, kGlmHessian = 1, kGlmLadder = 2 };   // what a pass computes
enum GlmFamily { kGlmTweedie = 0, kGlmBinomial = 1 };                 // the loss: half-Tweedie (link, power) or half-binomial
constexpr int kGlmCorrect = 7;
// b2_label_scan's counters (unsigned long long, in ctx->glm_part): the extremes as order-preserving keys of the fp32 value
enum LabelWord { kLabelKept = 0, kLabelNonFinite, kLabelNonIntegral, kLabelMin, kLabelMax, kLabelNMin, kLabelNMax,
                 kLabelWords };
// the order-preserving key of an fp32 label (monotone in v for finite v) and its inverse
__device__ __forceinline__ unsigned long long label_key(float v) {
  const uint32_t u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float label_of_key(unsigned long long k) {
  const uint32_t u = (uint32_t)k;
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// ---- the ridge classifier (classify.cu, solve.cu: solve_classes_kernel; DESIGN.md section 12) -------------------------
// doubles of ctx->cls: the centre c of the class sums, the sorted classes, the model W [kMaxClasses][kMaxD] and b, the
// solve's info (1-based failing pivot), the classify counts [kept, correct], the reduced class sums [K][d + 1] + 3 counts
constexpr int kMaxClasses = B2_MAX_CLASSES;
constexpr int kClsPart = kMaxClasses * (kMaxD + 1) + 8;   // one CTA's class sums (also the classify pass's two counts)
constexpr int kClsCenter = 0;
constexpr int kClsClasses = kMaxD;
constexpr int kClsCoef = kClsClasses + kMaxClasses;
constexpr int kClsIntercept = kClsCoef + kMaxClasses * kMaxD;
constexpr int kClsInfo = kClsIntercept + kMaxClasses;
constexpr int kClsCounts = kClsInfo + 8;
constexpr int kClsSums = kClsCounts + 8;
constexpr int kClsDoubles = kClsSums + kClsPart;
// the class of a kept row: the index of y in the sorted classes, -1 when y is none of them (NaN included)
__device__ __forceinline__ int class_of(const float* cls, int n_classes, float y) {
  int k = -1;
  for (int c = 0; c < n_classes; ++c) k = cls[c] == y ? c : k;
  return k;
}

// ---- the leave-one-out pass of b2_ridge_classifier_loo (ridge_loo.cu; DESIGN.md section 13) --------------------------
// doubles of ctx->loo_cls: the B operands of one call (built by its prep kernel from ctx->loo and the class sums at
// ctx->cls + kClsSums), ybar per target, and the reduced sums per alpha: sum e^2 over every target, rows whose first
// argmax of p = t - e is their class.  The per-CTA partials [grid][kLcPart] live in ctx->glm_part.
constexpr int kLcW = 0;                                    // [kMaxD][kMaxAlphas] 1 / (lambda_j + alpha_a)
constexpr int kLcCw = kLcW + kMaxD * kMaxAlphas;           // [kMaxD][T][8 ceil(A / 8)] C_jt / (lambda_j + alpha_a)
constexpr int kLcC = kLcCw + kMaxD * kMaxClasses * kMaxAlphas;   // [kMaxD][kMaxClasses] C = Q^T R
constexpr int kLcYbar = kLcC + kMaxD * kMaxClasses;        // [kMaxClasses] 2 n_k / n - 1 (0 without an intercept)
constexpr int kLcSum = kLcYbar + kMaxClasses;              // [2][kMaxAlphas] sum e^2, correct rows
constexpr int kLcPart = 2 * kMaxAlphas;
constexpr int kLcDoubles = kLcSum + kLcPart;

// ---- multinomial logistic regression (multinomial.cu; DESIGN.md section 14) ------------------------------------------
// doubles of ctx->mn_op: the sorted classes, the coefficients [K][kMaxD + 1] (row k = [w_k, b_k]) and the step beside
// them.  The reduced sums at ctx->mn_sum: the head [kMnHead] ([0] loss [1] kept [2] kept rows of no class [3] kept rows
// with y not finite [4] rows whose first argmax of eta is their class; a line search leaves the loss at step t in [t]),
// the gradient [K][d + 1], then (Hessian) the upper triangle of each class pair's block [P][dp][dp], dp = d + 1 padded
// to 16, pairs k <= l in row-major order.  Per-CTA partials in ctx->mn_part, [slice][the same layout], grown lazily.
constexpr int kMnHead = 32;
constexpr int kMnClasses = 0;
constexpr int kMnCoef = kMaxClasses;
constexpr int kMnStep = kMnCoef + kMaxClasses * (kMaxD + 1);
constexpr int kMnOpDoubles = kMnStep + kMaxClasses * (kMaxD + 1);

// ---- LinearDiscriminantAnalysis (discriminant.cu; DESIGN.md section 16) -------------------------------------------
// doubles of ctx->disc: the sorted classes, the class weights, the class means [kMaxClasses][kMaxD], then the reduced sums
// at kDaSums ([0] kept rows [1] kept rows of no class [2] kept rows with y not finite, then the upper triangle of the
// scatter at kDaHead + i kMaxD + j).  One CTA's partial in ctx->disc_part has the sums' layout, kDaPart doubles.
constexpr int kDaHead = 8;
constexpr int kDaPart = kDaHead + kMaxD * kMaxD;
constexpr int kDaClasses = 0;
constexpr int kDaWeights = kMaxClasses;
constexpr int kDaMeans = 2 * kMaxClasses;
constexpr int kDaSums = kDaMeans + kMaxClasses * kMaxD;
constexpr int kDaDoubles = kDaSums + kDaPart;

// ---- QuadraticDiscriminantAnalysis (qda.cu; DESIGN.md section 17) ---------------------------------------------------
// doubles of ctx->qda: the sorted classes, the class means [kMaxClasses][kMaxD], the offsets c_k and the transforms W_k
// ([K][d][d], pitch d) of the decision pass, then the reduced scatters [kMaxClasses][kMaxD][kMaxD] (upper triangle at
// i kMaxD + j) and the counts (rows per class [kMaxClasses], then kept rows, kept rows of no class, kept rows with y not
// finite).
constexpr int kQdClasses = 0;
constexpr int kQdMeans = kMaxClasses;
constexpr int kQdConst = kQdMeans + kMaxClasses * kMaxD;
constexpr int kQdW = kQdConst + kMaxClasses;
constexpr int kQdSums = kQdW + kMaxClasses * kMaxD * kMaxD;
constexpr int kQdCounts = kQdSums + kMaxClasses * kMaxD * kMaxD;
constexpr int kQdDoubles = kQdCounts + kMaxClasses + 8;
// rows of the class-order step: a span (its int32 indices fill ctx->qda_scratch, 64 MB), a chunk of its counts
constexpr int64_t kQdSpan = 1 << 24;
constexpr int kQdChunk = 8192;
constexpr int kQdMaxChunks = (int)(kQdSpan / kQdChunk);
constexpr size_t kQdScratchBytes = sizeof(int) * (size_t)kQdSpan;   // also the decisions of label-only calls
constexpr int kQdItemsPerSm = 2;                                    // work items of the scatter pass per SM
// ints of ctx->qda_hd: the decision pass's kept and correct rows (two unsigned long long), the span's work items and
// counts (written by order_scan_kernel), the chunk counts [kQdMaxChunks][kMaxClasses + 3] and the items [n][3]
// (class, begin, end) for qda_max_items
constexpr int kQdHdCorrect = 0;
constexpr int kQdHdNItems = 4;
constexpr int kQdHdCounts = 5;
constexpr int kQdHdStart = 8;                                        // [kMaxClasses + 1] class k's indices [start_k, start_k+1)
constexpr int kQdHdFirstItem = kQdHdStart + kMaxClasses + 1;         // [kMaxClasses + 1] class k's items [first_k, first_k+1)
constexpr int kQdHdCnt = 80;
constexpr int kQdHdItems = kQdHdCnt + kQdMaxChunks * (kMaxClasses + 3);
static_assert(kQdHdFirstItem + kMaxClasses + 1 <= kQdHdCnt, "qda header");
int qda_max_items(const b2_ctx* ctx);

// ---- cross-validation folds (folds.cu) ------------------------------------------------------------------------------
constexpr int kMaxFolds = 254;        // fold ids are bytes; 255 marks a dropped row
// first and last row of every fold of fold ids in device memory: range[2 k] = n - first, range[2 k + 1] = last + 1
// (both 0 for a fold without rows); range is zeroed by the launch
int launch_fold_ranges(b2_ctx* ctx, const uint8_t* fold_of_row, int64_t n, int n_folds, unsigned long long* range);
// S = the sum of the n_folds statistics of pitch (d+2)^2 in `folds`, added in fold order from 0
int launch_fold_sum(b2_ctx* ctx, const double* folds, int n_folds, int d, double* S);

// template width of the one-lane-per-row kernels (gram_narrow.cu, score.cu) for d <= 16 features: the next power of two
inline int narrow_dp(int d) { return d <= 1 ? 1 : d <= 2 ? 2 : d <= 4 ? 4 : d <= 8 ? 8 : 16; }

void set_error(const char* fmt, ...);

#define B2_CUDA(call)                                                                      \
  do {                                                                                     \
    cudaError_t e_ = (call);                                                               \
    if (e_ != cudaSuccess) {                                                               \
      b2::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
      return B2_E_CUDA;                                                                    \
    }                                                                                      \
  } while (0)

}  // namespace b2

struct b2_ctx {
  int device = 0;
  int sm_count = 0;
  size_t hbm_bytes = 0;
  char name[128] = {0};
  cudaStream_t stream = nullptr;       // compute stream (all kernels)
  cudaStream_t copy_stream = nullptr;  // H2D staging for B2_MEM_HOST
  cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;
  cudaEvent_t ev_k[b2::kKernelEventPairs][2];
  int k_pairs = 0;                     // pairs recorded since the last b2_last_kernel_ms
  int64_t launches = 0;                // kernels launched since ctx creation

  int kernel_mode = B2_KERNEL_AUTO;
  int drain_rows = 8192;
  int precision = B2_PRECISION_SPLIT;

  int d = 0;                           // feature count of the current statistic (0 = not reset)
  double* S = nullptr;                 // device, kMaxS*kMaxS (only (d+2)^2 used, row stride d+2)

  // tensor-core path scratch
  double* tc_part = nullptr;           // sm_count * (kTcAccElems + kTcSums): per-CTA fp64 partial Gram (col-major), y sums
  double* tc_red = nullptr;            // [kTcAccElems + 16]: reduced partials, y sums, b2_comm_barrier's slot at + 8
  float* shift = nullptr;              // gram_shift_bytes(): per-column shift c[kMaxD + 1] (c_y at kMaxD), sample scratch
  bool solve_attr_set = false;
  double* solve_host = nullptr;        // pinned mirror of solve_out (D2H without a staging copy)
  // tensor-map cache of the most recent tensor-core launch (a refit of resident rows re-uses the same maps)
  struct TmCache {
    const void* X = nullptr; const float* y = nullptr; const uint8_t* mask = nullptr;
    int64_t n = 0, ldx = 0; int d = 0, x_dtype = -1;
    int y_map_2d = 0, m_map_2d = 0;    // y / the mask read through a [n / k][k] view (gram_tc.cu: encode_vec)
    alignas(64) unsigned char tmX[128], tmY[128], tmM[128];
  } tm_cache;
  // SIMT path scratch
  double* simt_part = nullptr;         // [simt_ctas][kMaxS*kMaxS]
  int simt_ctas = 0;
  // scoring scratch
  double* score_part = nullptr;        // [score_ctas + 2][kNStats]: per-CTA partials, running totals (b2::score_totals)
  int score_ctas = 0;
  double* coef_dev = nullptr;          // [kMaxD + 1]
  // refined fit scratch
  double* grad_part = nullptr;         // [score_ctas][kGradOut] per-CTA gradient partials
  double* refine = nullptr;            // [kRfDoubles] beta, b0', m, the state before the last correction, step, gradient
  // ridge leave-one-out scratch
  double* loo = nullptr;               // [kLooDoubles] Q, lambda, m, c, ybar / n / h0, alphas, the B operands, the sums
  double* loo_part = nullptr;          // [sm_count][kMaxAlphas] per-CTA sums of e^2
  // elastic-net path: inputs and outputs of b2_solve_enet_path (b2::EnetArgs), grown to the largest call
  double* enet = nullptr;
  size_t enet_doubles = 0;
  // cross-validation: the fold statistics of b2_gram_folds / b2_solve_enet_cv ([n_folds][(d+2)^2]), grown to the
  // largest call, and the fold ranges of b2_gram_folds
  double* folds = nullptr;
  size_t folds_doubles = 0;
  int n_folds = 0;                     // folds held in `folds` (0: none)
  int folds_d = 0;                     // their d
  unsigned long long* fold_range = nullptr;   // [2 kMaxFolds]
  // generalised linear regressors: the sums and operands of b2_glm_* (b2::kGlm*), per-CTA partials [2 sm_count][kGlmPart];
  // allocated by the first call
  double* glm = nullptr;
  double* glm_part = nullptr;
  // the ridge classifier's operands and sums (b2::kCls*), allocated by the first call; its per-CTA partials in glm_part
  double* cls = nullptr;
  // the classifier's leave-one-out operands and sums (b2::kLc*, 2.1 MB), allocated by the first call
  double* loo_cls = nullptr;
  // multinomial logistic regression: the operands (b2::kMn*), the reduced sums and the per-CTA partials, each grown to the
  // largest call
  double* mn_op = nullptr;
  double* mn_sum = nullptr;
  size_t mn_sum_doubles = 0;
  double* mn_part = nullptr;
  size_t mn_part_doubles = 0;
  // LinearDiscriminantAnalysis: the operands and sums of b2_class_scatter (b2::kDa*) and the per-CTA partials
  // [sm_count][kDaPart], allocated by the first call
  double* disc = nullptr;
  double* disc_part = nullptr;
  // QuadraticDiscriminantAnalysis: operands and sums (b2::kQd*), the int header (b2::kQdHd*), the scratch of the class
  // order and of label-only decisions, all allocated by the first call; the scatter pass's per-item partials
  // [qda_max_items][kMaxD * kMaxD] by the first scatter call
  double* qda = nullptr;
  int* qda_hd = nullptr;
  void* qda_scratch = nullptr;
  double* qda_part = nullptr;
  double* coef_host = nullptr;         // pinned [2][kMaxD + 1]: upload slots of b2_score's coefficients
  cudaEvent_t ev_coef[2] = {nullptr, nullptr};
  int coef_slot = 0;
  long long* synth_count = nullptr;    // device counter of b2_synth_tranche (rows kept by the y >= 0 filter)
  // solve scratch
  double* solve_out = nullptr;         // [kMaxD + 2 + kMaxD]: coef, intercept, info, singular
  // host staging ring (B2_MEM_HOST)
  void* stage_x[2] = {nullptr, nullptr};
  float* stage_y[2] = {nullptr, nullptr};
  uint8_t* stage_m[2] = {nullptr, nullptr};
  size_t stage_bytes_x = 0;
  int64_t stage_rows = 0;
  cudaEvent_t ev_copied[2] = {nullptr, nullptr};
  cudaEvent_t ev_consumed[2] = {nullptr, nullptr};
  bool ev_consumed_valid[2] = {false, false};   // a kernel of an earlier call may still read stage buffer b
  // the per-row outputs of host rows (yhat, ystd, e^2, mu): two blocks of row_out_bytes each (at most stage_rows rows),
  // grown to the largest call
  char* row_out[2] = {nullptr, nullptr};
  size_t row_out_bytes = 0;
  void* bounce[2] = {nullptr, nullptr};         // pinned bounce blocks for pageable host rows (filled by host threads)
  cudaEvent_t ev_bounce[2] = {nullptr, nullptr};
  bool s_zero_pending = false;         // b2_gram_reset is lazy: the first kernel to write S overwrites it
  // NCCL
  void* comm = nullptr;
  int n_ranks = 1, rank = 0;
  // one-shot peer-memory all-reduce of S (p2p.cu): exchange buffer exported over CUDA IPC
  double* xchg = nullptr;              // [2 parities][kMaxRanks][kMaxS*kMaxS] slots, then flags / ticket words
  double* xchg_peer[8] = {nullptr};    // this rank's view of every rank's exchange buffer (own entry == xchg)
  bool p2p_ready = false;
  bool p2p_local = false;              // peers attached inside this process (b2_comm_p2p_attach_local): no IPC handles to close
  unsigned int xchg_epoch = 0;
  unsigned long long xchg_timeout_ns = 10000000000ull;   // bound of the wait for a peer's flag (b2_comm_set_timeout_ms)
  bool xchg_pending = false;           // an exchange was launched since the status word was last read
  unsigned int* xchg_status_host = nullptr;  // pinned mirror of the exchange status word
  // grid barrier / ticket words of the tensor-core finalize kernel (reduce + fold + peer scatter)
  unsigned int* tc_sync = nullptr;     // [0], [1] barrier arrivals, [2] ticket
  int fused_fits = 0;                  // b2_fit calls whose device rows ended on the tensor-core kernel (b2_ctx_stats)
  int sm_limit = 0;                    // > 0: persistent kernels use at most this many SMs (b2_ctx_set_sm_limit)
  bool sm_limit_auto = false;          // the limit was set by b2_comm_p2p_attach_local (contexts sharing a device)
};

namespace b2 {

// the kNStats running totals of the current b2_score / b2_metrics call (behind the per-CTA partials; b2_score_allreduce
// keeps its two maxima in the kNStats doubles after them)
inline double* score_totals(const b2_ctx* ctx) { return ctx->score_part + (size_t)ctx->score_ctas * kNStats; }

// ---- launch helpers (score.cu, gram_narrow.cu; gram_tc.cu selects its instantiation with with_rows / with_int) -------
// One launch with `smem` bytes of dynamic shared memory; the attribute is set before every launch.
template <typename... P, typename... A>
int launch_smem(void (*kernel)(P...), int grid, int threads, uint32_t smem, cudaStream_t stream, A... args) {
  B2_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  kernel<<<grid, threads, smem, stream>>>(args...);
  B2_CUDA(cudaGetLastError());
  return B2_OK;
}
// f(std::integral_constant<int, V>{}) for the first V of Vs equal to v, the last V when none is
template <int V, int... Vs, typename F>
int with_int(int v, F&& f) {
  if constexpr (sizeof...(Vs) == 0) return f(std::integral_constant<int, V>{});
  else return v == V ? f(std::integral_constant<int, V>{}) : with_int<Vs...>(v, f);
}
// f(X as const float* or const __nv_bfloat16*)
template <typename F>
int with_rows(int x_dtype, const void* X, F&& f) {
  if (x_dtype == B2_F32) return f(static_cast<const float*>(X));
  return f(static_cast<const __nv_bfloat16*>(X));
}
template <typename P>
using row_t = std::remove_const_t<std::remove_pointer_t<P>>;

// Which kernels read the rows [0, n) of one call.  Contiguous 16-byte aligned rows stream through a bulk-copy ring in
// whole tiles: one lane per row for d <= 16 (narrow, the mask aligned too), LPR lanes per row when a row is a multiple of
// 16 bytes (wide).  The rows after the last whole tile, and all rows of any other layout, go to the register-fed kernels
// (direct).  Scoring and the residual gradient share this plan, so a pass of the refined fit (and the leave-one-out pass
// of b2_ridge_loo) reads its rows the way b2_score does, in as many launches.
struct RowPlan {
  enum Kind { kDirect, kNarrow, kWide } kind = kDirect;
  int dp = 0;                   // narrow: the template width narrow_dp(d)
  int lpr = 0, sweeps = 0;      // wide: lanes per row, consumer sweeps per tile
  int n_tiles = 0, grid = 0;    // whole ring tiles and the ring's grid (n_tiles == 0: no ring launch)
  int64_t done = 0;             // rows [0, done) go through the ring
  bool direct = false;          // the register-fed kernels take the rows [done, n) (one launch when n == 0)
  int64_t rest = 0;
  int vec = 0, direct_grid = 0; // their 4-feature vector loads and grid
};

RowPlan plan_rows(const b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                  const uint8_t* mask);

// The rows [r0, r0 + rows) of a call: X (row pitch ldx), y and mask point at row r0 (y / mask null when the call has
// none); `first`: no earlier rows of the call have written its sums.
struct RowSpan {
  const void* X;
  const float* y;
  const uint8_t* mask;
  int64_t ldx, r0, rows;
  bool first;
};

// The rows [0, n) of a pass with a ring flavour that reads whole tiles of tile_rows rows: f(true, span) for the whole
// tiles when plan_rows streams the rows through a ring, then f(false, span) for the rest.  A part with no rows is
// skipped, except the direct part of an empty call that writes the sums first.
template <typename F>
int split_ring_rows(const b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                    const uint8_t* mask, int tile_rows, bool first, F&& f) {
  const bool ring_ok = plan_rows(ctx, X, x_dtype, n, d, ldx, y, mask).kind != RowPlan::kDirect;
  const int64_t ring_rows = ring_ok ? (n / tile_rows) * tile_rows : 0;
  const int es = x_dtype == B2_F32 ? 4 : 2;
  for (int part = 0; part < 2; ++part) {
    const bool ring = part == 0;
    const int64_t r0 = ring ? 0 : ring_rows, rows = ring ? ring_rows : n - ring_rows;
    if (rows == 0 && (ring || !first)) continue;
    const RowSpan s{static_cast<const char*>(X) + (size_t)r0 * ldx * es, y != nullptr ? y + r0 : nullptr,
                    mask != nullptr ? mask + r0 : nullptr, ldx, r0, rows, first};
    if (int r = f(ring, s)) return r;
    first = false;
  }
  return B2_OK;
}

// acc[e] = (first ? 0 : acc[e]) + part[0][e] + part[1][e] + ... over n_ctas per-CTA partials of pitch `stride`, in CTA
// order, so repeated calls are bit-identical.  The entries [0, n_lin), combined with fmax where bit e of max_mask is set;
// with d1 > 0 also the upper triangle i <= j < d1 at tri_off + i * tri_pitch + j.  One launch, counted with the pass
// whose partials it reduces (ctx->launches += 2).
int launch_ordered_reduce(b2_ctx* ctx, const double* part, int stride, int n_ctas, bool first, int n_lin,
                          unsigned max_mask, double* acc, int d1 = 0, int tri_off = 0, int tri_pitch = 0);

// ---- kernel launchers (each enqueues on ctx->stream and bumps ctx->launches) -----------------
// The Gram launchers are called by gram_dispatch (b2_api.cu) only.  assign: the kernel that writes S overwrites
// it instead of adding to it (the first writer after b2_gram_reset).  The tensor-core and narrow launchers cover the
// first gram_*_main_rows(n) rows and read the per-column shift c that launch_gram_shift sampled from all n rows.
size_t gram_shift_bytes();
int launch_gram_shift(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n, int d, int64_t ldx);
int launch_gram_simt(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n, int d,
                     int64_t ldx, const uint8_t* mask, int keep, bool assign);
bool gram_tc_supported(const void* X, int x_dtype, const float* y, int64_t n, int d, int64_t ldx,
                       const uint8_t* mask);
int64_t gram_tc_main_rows(int64_t n, int d, int64_t ldx, int* pack_out);
// scatter_epoch != 0: the finalize also stores S into every peer's exchange slot as exchange `scatter_epoch`
int launch_gram_tc(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n, int d,
                   int64_t ldx, const uint8_t* mask, int keep, bool assign, unsigned int scatter_epoch);
bool gram_narrow_supported(const void* X, int x_dtype, const float* y, int64_t n, int d, int64_t ldx,
                           const uint8_t* mask);
int64_t gram_narrow_main_rows(int64_t n, int d);
int launch_gram_narrow(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n, int d,
                       const uint8_t* mask, int keep, bool assign);
// gather_epoch != 0: the solve kernel first waits for the peer exchange `gather_epoch` and sums the slots into S
int launch_solve_cholesky(b2_ctx* ctx, double alpha, int fit_intercept, unsigned int gather_epoch = 0);
int launch_solve_eigvals(b2_ctx* ctx, double cond, int fit_intercept);
int launch_metrics(b2_ctx* ctx, const void* y, const void* yhat, int dtype, int64_t n, bool first);
int launch_solve_spectral(b2_ctx* ctx, double cond, int fit_intercept);
int launch_score(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx,
                 const float* y, const uint8_t* mask, int keep, float* yhat, bool first_block);
// residual gradient of the refined fit over the model in ctx->refine; `first_block` overwrites the gradient, otherwise
// the rows' sums are added to it
int launch_grad(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                const uint8_t* mask, int keep, bool first_block);
// the correction solve of one refinement pass: (A + alpha I) dbeta = g - alpha beta from the factor of S, then the
// update of ctx->refine; the result goes to ctx->solve_host
int launch_solve_refine(b2_ctx* ctx, double alpha, int fit_intercept);
// eigenvalues, orthonormal eigenvectors, m, ybar, n, h0 and c = Q^T r of the centred Gram of S into ctx->loo
int launch_solve_eigh(b2_ctx* ctx, int fit_intercept);
// the leave-one-out pass over the rows [0, n) for the n_alphas alphas at ctx->loo + kLooAlpha: the B operands (once per
// call, `first_block`), the pass (e^2 per row and alpha into cv when not null, NaN for rows not kept) and the ordered
// reduce of the per-CTA sums into ctx->loo + kLooSum (`first_block` overwrites, otherwise adds)
int launch_loo(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
               const uint8_t* mask, int keep, int n_alphas, double* cv, bool first_block);
// the classifier's leave-one-out pass over the rows [0, n) for the n_alphas alphas at ctx->loo + kLooAlpha, the
// eigendecomposition in ctx->loo and the classes and class sums in ctx->cls: the B operands (once per call,
// `first_block`), the pass (cv [row][T][n_alphas] when not null: e^2, or p = t - e with `accuracy`; NaN for rows not
// kept) and the ordered reduce of the per-CTA sums into ctx->loo_cls + kLcSum (`first_block` overwrites, else adds)
int launch_loo_classes(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                       const uint8_t* mask, int keep, int n_classes, int n_alphas, int fit_intercept, bool accuracy,
                       double* cv, bool first_block);
// the elastic-net path of the resident S (one launch; `args` points into ctx->enet)
int launch_solve_enet(b2_ctx* ctx, const EnetArgs& args);
// BayesianRidge's iteration in the eigenbasis of ctx->loo (launch_solve_eigh first); one launch
int launch_bayes_ridge(b2_ctx* ctx, const BayesArgs& args);
// ARDRegression's iteration on the resident S; one launch
int launch_ard(b2_ctx* ctx, const BayesArgs& args);
// ystd (and yhat when not null) of the rows [0, n): sqrt(max((x - m)^T sigma (x - m), 0) + noise_var) and x.w + b, from
// the operands at ctx->enet (kStd* in score_std.cu, written by the caller)
int launch_score_std(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, double* yhat, double* ystd);
// one pass of the GLM regressors or the logistic fits over the rows [0, n) at the operands of ctx->glm (mode: GlmMode;
// kGlmLadder takes the n_steps losses; family: GlmFamily, link and power for kGlmTweedie), then the ordered reduce of the
// per-CTA sums into ctx->glm (`first_block` overwrites, otherwise adds)
int launch_glm(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
               const uint8_t* mask, int keep, int mode, int family, int link, double power, int n_steps,
               bool first_block);
// mu of the rows [0, n): exp(x.w + b) (B2_GLM_LOG) or x.w + b, fp64
int launch_glm_predict(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, int link, double* mu);
// the logistic model of ctx->glm on the rows [0, n): eta (fp64), [1 - p, p] (fp64) and the label (fp32), each if not null
int launch_logistic_predict(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, double* decision,
                            double* proba, float* label);
// the kLabelWords counters of the kept rows of device y into st (two launches after two memsets)
int launch_label_scan(b2_ctx* ctx, const float* y, int64_t n, const uint8_t* mask, int keep, unsigned long long* st);
// the class sums of the rows [0, n) at the centre and classes of ctx->cls, then the ordered reduce of the per-CTA sums
// into ctx->cls + kClsSums (`first_block` overwrites, otherwise adds)
int launch_class_sums(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                      const uint8_t* mask, int keep, int n_classes, bool first_block);
// the model of ctx->cls on the rows [0, n): decision [n][n_targets] (fp64) and label (fp32), each if not null; with y,
// the kept and correct rows into ctx->cls + kClsCounts (`first_block` overwrites, otherwise adds)
int launch_classify(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                    const uint8_t* mask, int keep, int n_targets, double* decision, float* label, bool first_block);
// st[i], i <= max_values: the keys of the distinct finite kept y in ascending order, ~0 past the last (max_values + 1
// launches after one memset)
int launch_label_values(b2_ctx* ctx, const float* y, int64_t n, const uint8_t* mask, int keep, int max_values,
                        unsigned long long* st);
// one pass of multinomial logistic regression over the rows [0, n) at the classes, coefficients and step of ctx->mn_op
// (mode: GlmMode; kGlmLadder takes the n_steps losses), then one ordered reduce of every slice's partial into ctx->mn_sum
// (`first_block` overwrites, otherwise adds); ctx->mn_sum must hold multinomial_sum_doubles(d, n_classes, mode)
size_t multinomial_sum_doubles(int d, int n_classes, int mode);
int launch_multinomial(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                       const uint8_t* mask, int keep, int mode, int n_classes, int n_steps, bool first_block);
// sklearn.utils.extmath.softmax of each row of the device (n, k) fp64 array, in place (one launch)
int launch_softmax_rows(b2_ctx* ctx, double* values, int64_t n, int k);
// one pass of the linear SVMs (svm.cu) over the rows [0, n) at the operands of ctx->glm (loss: B2_SVM_*; hess: the
// Hessian change too), then the ordered reduce into ctx->glm in the GLM passes' layout (`first_block` overwrites,
// otherwise adds)
int launch_svm(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
               const uint8_t* mask, int keep, int loss, bool hess, bool first_block);
// the within-class scatter of the rows [0, n) at the classes, weights and means of ctx->disc, then the ordered reduce of
// the per-CTA sums into ctx->disc + kDaSums (`first_block` overwrites, otherwise adds)
int launch_class_scatter(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                         const uint8_t* mask, int keep, int n_classes, bool first_block);
// the per-class scatters of the rows [0, n) (n <= kQdSpan) at the classes and means of ctx->qda: the class order, the
// work items and the ordered reduce into ctx->qda + kQdSums and kQdCounts (`first_block` overwrites, otherwise adds)
int launch_class_scatters(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                          const uint8_t* mask, int keep, int n_classes, bool first_block);
// the QDA decisions of the rows [0, n) at the operands of ctx->qda into decision [n][n_classes] (device), then, each if
// not null, the labels, d_1 - d_0 (two classes) and, with y, the kept and correct rows added to ctx->qda_hd
int launch_qda_decision(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                        const uint8_t* mask, int keep, int n_classes, double* decision, float* label, double* diff);
// W and b of the ridge classifier from the resident S and the class sums at ctx->cls + kClsSums (one launch)
int launch_solve_classes(b2_ctx* ctx, double alpha, int fit_intercept, int n_classes);
int launch_p2p_allreduce(b2_ctx* ctx);
int launch_synth(b2_ctx* ctx, uint64_t seed, int64_t row_offset, int64_t n, int d, int64_t ldx,
                 int x_dtype, double alpha, double beta, double sigma, void* X, float* y);
int launch_synth_tranche(b2_ctx* ctx, uint64_t seed, int64_t n, double alpha, double beta, double sigma, float* X, float* y,
                         int64_t* n_kept_dev);

}  // namespace b2
