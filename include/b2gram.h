/*
 * b2gram.h -- C-ABI of libb2gram.so: the H100 (sm_90a) retrain hot path of
 * AlexIoannides/bodywork-mlops-demo, i.e. the least-squares / ridge fit that
 * mlops_simulation/stage_1_train_model.py performs through scikit-learn.
 *
 * This is the drop-in boundary: plain pointers and sizes, no C++/torch types.
 * The reference is pure Python, so the binding a maintainer adds is a ctypes stub
 * (see INTEGRATION.md); every entry point cites the reference call it replaces.
 *
 * Conventions
 *   - every function returns int: 0 = ok, <0 = error (B2_E_*); text via b2_last_error()
 *     (thread-local).  No exceptions cross the boundary.
 *   - the caller owns every buffer it passes; b2_ctx owns device scratch, streams, the
 *     fp64 sufficient statistic S and (optionally) one NCCL communicator.
 *   - one b2_ctx == one GPU; one process per GPU for multi-GPU (rows shard by rank, the
 *     only exchange is b2_gram_allreduce).  A ctx is not re-entrant.
 *   - there is NO CPU fallback: without a usable CUDA device every compute entry point
 *     fails with B2_E_CUDA.
 *
 * Sufficient statistic.  S = [X 1 y]^T [X 1 y], (D+2) x (D+2), row-major fp64, index
 * order: features 0..D-1, the ones column (D), y (D+1).  S[D][D] is the row count.
 */
#ifndef B2GRAM_H_
#define B2GRAM_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2_ABI_VERSION 2
#define B2_MAX_D 128

/* element type of X */
#define B2_F32 0
#define B2_BF16 1
#define B2_F64 2 /* b2_metrics, b2_upload_columns */

/* where a caller buffer lives */
#define B2_MEM_DEVICE 0 /* device pointer (HBM)                                   */
#define B2_MEM_HOST 1   /* host pointer (pinned preferred); streamed in row blocks */

/* kernel selection for b2_gram_accumulate */
#define B2_KERNEL_AUTO 0   /* d <= 16: NARROW; wider: TCGEN05; odd layouts / tiny blocks: SIMT */
#define B2_KERNEL_SIMT 1   /* fp64-accumulating CUDA-core kernel (any D <= 128)       */
#define B2_KERNEL_TCGEN05 2 /* TMA -> smem -> bf16 hi/lo split -> wgmma -> registers */
#define B2_KERNEL_NARROW 3  /* D <= 16: TMA bulk-copy pipeline -> fp32 FMA on CUDA cores */
/* tensor-core path requirements: 4 <= d <= 128, row bytes and row pitch multiples of 16, X / y / row_mask 16-byte
 * aligned, n_rows >= 64.  Contiguous rows with 17 <= d <= 64 are packed min(5, 128 / d) per 128-wide super-row.
 * narrow path requirements: d <= 16, contiguous rows (ldx == d), X / y / row_mask 16-byte aligned.
 * AUTO uses NARROW from 4096 rows and TCGEN05 from 2048 rows per call; smaller blocks (the reference's 1 440-row
 * daily tranche, stage_3_synthetic_data_generation.py:19) and every other layout take the exact fp64 SIMT kernel. */

/* operand precision of the tensor-core Gram kernel (b2_ctx_set_precision) */
#define B2_PRECISION_SPLIT 0 /* bf16 hi + lo operands (16 mantissa bits), default: coef error ~2e-6 at any n */
#define B2_PRECISION_BF16 1  /* single bf16 operand ("bf16-accum", BASELINE.json configs[1]): error ~2.4e-2/sqrt(n) */

/* error codes */
#define B2_OK 0
#define B2_E_ARG (-1)
#define B2_E_CUDA (-2)
#define B2_E_STATE (-3)
#define B2_E_SINGULAR (-4) /* Cholesky met a non-positive pivot (rank-deficient, alpha == 0) */
#define B2_E_COMM (-5) /* NCCL failure, or a peer did not deliver its partial statistic within the timeout */
#define B2_E_NCCL B2_E_COMM
#define B2_E_UNSUPPORTED (-6)

typedef struct b2_ctx b2_ctx;

/* ---- library / context ------------------------------------------------------------ */
int b2_abi_version(void);
const char* b2_last_error(void);
int b2_device_count(int* n_out);
int b2_ctx_create(int device, b2_ctx** out);
int b2_ctx_destroy(b2_ctx* ctx);
int b2_ctx_sync(b2_ctx* ctx);
/* name, SM count, HBM bytes of the ctx's device (name_cap bytes incl. NUL) */
int b2_ctx_info(b2_ctx* ctx, char* name, int name_cap, int* sm_count, size_t* hbm_bytes);
/* force a kernel family (B2_KERNEL_*); default AUTO */
int b2_ctx_set_kernel(b2_ctx* ctx, int kernel);
/* rows of fp32 tensor-core accumulation before the register accumulators are drained into fp64 (default 8192) */
int b2_ctx_set_drain_rows(b2_ctx* ctx, int rows);
/* the persistent Gram kernel uses at most n_sms SMs (0 = all): leaves room for other work on the device */
int b2_ctx_set_sm_limit(b2_ctx* ctx, int n_sms);
/* B2_PRECISION_*: operand precision of the tensor-core path (the CUDA-core kernel is always exact) */
int b2_ctx_set_precision(b2_ctx* ctx, int precision);

/* ---- caller-owned buffers (helpers; the Python shim has no other CUDA binding) ------------ */
int b2_dev_alloc(b2_ctx* ctx, size_t bytes, void** out);
int b2_dev_free(b2_ctx* ctx, void* p);
int b2_host_alloc(b2_ctx* ctx, size_t bytes, void** out); /* pinned */
int b2_host_free(b2_ctx* ctx, void* p);
int b2_copy_h2d(b2_ctx* ctx, void* dst, const void* src, size_t bytes); /* sync on return */
int b2_copy_d2h(b2_ctx* ctx, void* dst, const void* src, size_t bytes); /* sync on return */
int b2_copy_d2d(b2_ctx* ctx, void* dst, const void* src, size_t bytes); /* on the context's stream, asynchronous: bench.py
                                                                         times it as this box's own copy bandwidth */
int b2_dev_memset(b2_ctx* ctx, void* dst, int value, size_t bytes);
/* DataFrame columns -> row-major float32 rows in HBM.  reference: stage_1_train_model.py:95-96
 * (`X = data['X'].values.reshape(-1, 1)`): pandas hands every column over as its own strided array.  cols[j] = address of
 * row 0 of feature column j, strides[j] = bytes between consecutive rows of it, dtype = B2_F64 (pandas' default) or B2_F32;
 * X_dev: caller-owned device buffer of n_rows x d floats, row-major.  Host threads gather and convert into a pinned ring
 * while the previous block is on the wire; sync on return. */
int b2_upload_columns(b2_ctx* ctx, const void* const* cols, const int64_t* strides, int dtype, int64_t n_rows, int d,
                      float* X_dev);
/* The gather + conversion of b2_upload_columns alone, host to host (no device, no context): out[n_rows][d] float32, e.g. a
 * caller's own pinned block.  Multi-threaded like the upload. */
int b2_pack_columns(const void* const* cols, const int64_t* strides, int dtype, int64_t n_rows, int d, float* out);

/* ---- Gram accumulation: replaces LinearRegression.fit's pass over the rows -----------------
 * reference: stage_1_train_model.py:105-106 -> sklearn/linear_model/_base.py (centre + gelsd). */
int b2_gram_reset(b2_ctx* ctx, int d);
/* S += [X 1 y]^T [X 1 y] over the rows of this block (this rank's shard).
 *   X        n_rows x d, row-major, leading dimension ldx (elements), dtype x_dtype
 *   y        n_rows fp32
 *   row_mask NULL, or one byte per row: a row is used iff row_mask[r] == mask_keep.
 *            (lets train_test_split's shuffled 80/20 membership -- stage_1_train_model.py:98-103 --
 *            be applied without gathering rows)
 *   mem_kind where X / y / row_mask live (all three the same)                                */
int b2_gram_accumulate(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows,
                       int d, int64_t ldx, int mem_kind, const uint8_t* row_mask, int mask_keep);
/* sum S over the ranks of the communicator (one ncclAllReduce of (d+2)^2 doubles) */
int b2_gram_allreduce(b2_ctx* ctx);
/* copy S out / in (incremental-refit state).  S_out/S_in: (d+2)^2 doubles on the host */
int b2_gram_export(b2_ctx* ctx, double* S_out, int64_t* n_rows_out);
int b2_gram_import(b2_ctx* ctx, const double* S_in, int d);

/* ---- split: the row membership of train_test_split(X, y, test_size, random_state=seed) ---------------------------
 * reference: stage_1_train_model.py:98-103 -> sklearn ShuffleSplit: perm = RandomState(seed).permutation(n_rows);
 * test = perm[:n_test], train = the rest.  mask_out[r] = 0 for test rows, 1 for train rows (n_rows bytes, host) --
 * the row_mask b2_gram_accumulate / b2_fit (keep 1) and b2_score (keep 0) consume.  Host-side by nature (MT19937 +
 * Fisher-Yates are sequential); bit-exact with numpy's legacy generator, ~10x its speed at 10^8 rows. */
int b2_split_mask(int64_t n_rows, int64_t n_test, uint32_t seed, uint8_t* mask_out);

/* ---- the whole fit in one call: LinearRegression(fit_intercept).fit(X, y) / Ridge(alpha) ----------------------
 * reference: stage_1_train_model.py:105-106.  Equivalent to b2_gram_reset + b2_gram_accumulate + b2_gram_allreduce +
 * b2_solve with the same arguments, and runs the same Gram kernels; the solve kernel writes coef / intercept straight
 * to pinned host memory.  With a peer exchange attached and device-resident rows whose last Gram launch is the
 * tensor-core kernel, the exchange takes no launches of its own: the finalize kernel behind the Gram kernel stores S
 * into the peers' exchange slots and the solve kernel sums them. */
int b2_fit(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
           int mem_kind, const uint8_t* row_mask, int mask_keep, double alpha, int fit_intercept,
           double* coef, double* intercept);

/* b2_fit, then up to max_passes (0..16) residual passes over the same rows (see DESIGN section 2).  Each pass streams
 * the rows once for the fp64 gradient g = [X-m 1]^T (y - yhat) of the current solution and corrects it through the
 * factor of the approximate Gram, which takes a tensor-core fit to the fp64 least-squares solution of the stored rows.
 * tol >= 0: stop when the scale-free step max_j |dcoef_j| sigma_j / sigma_y <= tol.  A step larger than the one before
 * stops the passes and returns the state before the last kept correction.  passes_out: corrections kept; step_out: the
 * last step (0 when max_passes == 0).  max_passes == 0 is bit-identical to b2_fit.  S afterwards is b2_fit's S.
 * B2_E_UNSUPPORTED with more than one rank; B2_E_SINGULAR as b2_fit. */
int b2_fit_refined(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                   int mem_kind, const uint8_t* row_mask, int mask_keep, double alpha, int fit_intercept,
                   int max_passes, double tol, double* coef, double* intercept, int* passes_out, double* step_out);

/* ---- solve:replaces scipy.linalg.lstsq + _set_intercept ----------------------------------------
 * reference: sklearn/linear_model/_base.py (lstsq on centred data; intercept_ = y_mean - x_mean.coef_)
 * Single-SM fp64 LDL^T (square-root-free Cholesky) of (Xc^T Xc + alpha I).  coef: d doubles, intercept: 1 double
 * (host).  fit_intercept = 0 solves the uncentred problem.  Returns B2_E_SINGULAR on a non-positive pivot and
 * B2_E_COMM when the preceding peer-memory exchange timed out (S incomplete). */
int b2_solve(b2_ctx* ctx, double alpha, int fit_intercept, double* coef, double* intercept);
/* eigenvalues of the centred Gram (device Jacobi) -> singular_ (descending, d doubles) and rank_
 * (count of singular values > cond * max), plus the minimum-norm coefficients gelsd would return.
 * Any output pointer may be NULL. */
int b2_solve_spectral(b2_ctx* ctx, double cond, int fit_intercept, double* coef, double* intercept,
                      double* singular, int* rank);

/* singular_ (descending, d doubles) and rank_ only -- the attributes LinearRegression.fit stores beside coef_
 * (sklearn/linear_model/_base.py) -- as sqrt of the eigenvalues of the centred Gram: Householder tridiagonalisation +
 * Sturm multisection on one SM, no eigenvectors (b2_solve_spectral is only needed when rank < d). */
int b2_solve_eigvals(b2_ctx* ctx, double cond, int fit_intercept, double* singular, int* rank,
                     int64_t* n_rows_out /* rows in S; may be NULL */);

/* eigenvalues (ascending, d doubles) and eigenvectors (d x d row-major, column k belongs to eigenvalue k) of the
 * centred Gram (uncentred when fit_intercept == 0) of the resident S; either pointer may be NULL.  Two-sided cyclic
 * Jacobi on one SM: the eigenvectors are orthonormal to working precision for every eigenvalue, zero and clustered ones
 * included.  Negative rounding eigenvalues are returned as 0.  B2_E_SINGULAR if the sweeps have not converged within
 * their limit (30), which finite statistics at D <= 128 do not reach. */
int b2_solve_eigh(b2_ctx* ctx, int fit_intercept, double* eigvals, double* eigvecs);

/* ---- elastic net / lasso path: replaces sklearn.linear_model.enet_path(precompute=Gram) / ElasticNet / Lasso -------
 * reference: sklearn/linear_model/_coordinate_descent.py enet_path (alpha scaling, _alpha_grid) and _cd_fast.pyx
 * enet_coordinate_descent_gram (cyclic coordinate descent, dual gap, gap-safe screening, stopping rule), run on the
 * centred Gram Q = Xc^T Xc, q = Xc^T yc and ||yc||^2 of the resident S (uncentred without fit_intercept); one
 * single-SM launch for the whole path (DESIGN section 7).  Minimises, per alpha,
 *   1 / (2 n) ||yc - Xc w||^2 + alpha l1_ratio ||w||_1 + alpha (1 - l1_ratio) / 2 ||w||^2   (w >= 0 with positive)
 *   alphas      NULL: sklearn's grid geomspace(alpha_max, alpha_max eps, n_alphas), alpha_max = max |q| / (n l1_ratio)
 *               (max(0, max q) with positive); else n_alphas finite values >= 0, solved in the order given (host)
 *   coef_init   NULL (zeros) or d doubles: the start of the first alpha; each later alpha starts from the previous one
 *   outputs     (host) alphas_out n_alphas, coefs_out n_alphas x d (row-major), intercepts_out ybar - m.w,
 *               gaps_out the dual gap / n (sklearn's dual_gaps), n_iter_out sweeps (0: the start already met the gap),
 *               tol_out NULL or tol ||yc||^2 / n, the gap each alpha had to reach
 * A column whose centred diagonal is <= 1e-12 of its raw one is constant: coefficient 0, never updated.  Not reaching
 * the gap within max_iter sweeps is no error: n_iter_out == max_iter and gaps_out > tol_out.  The outputs are staged in
 * a device block of the context, grown to the largest call and freed with it.  B2_E_ARG: l1_ratio outside [0, 1], a
 * grid with l1_ratio == 0 or eps <= 0, an alpha < 0 or not finite, n_alphas < 1, max_iter < 1, tol < 0, a null output,
 * or a statistic without rows. */
int b2_solve_enet_path(b2_ctx* ctx, int fit_intercept, double l1_ratio, const double* alphas, int n_alphas, double eps,
                       int max_iter, double tol, int positive, const double* coef_init, double* alphas_out,
                       double* coefs_out, double* intercepts_out, double* gaps_out, int* n_iter_out, double* tol_out);

/* ---- cross-validated elastic net / lasso: replaces sklearn.linear_model.ElasticNetCV / LassoCV(precompute=True) --
 * reference: sklearn/linear_model/_coordinate_descent.py LinearModelCV.fit and _path_residuals (DESIGN section 8).
 * b2_gram_folds: the statistic S_k of every fold in one call.  Row r belongs to fold fold_of_row[r] (a value >= n_folds
 * drops the row; the ids live where X lives: device or host).  Fold k is the Gram dispatch of b2_gram_accumulate over
 * rows [first_k rounded down to a multiple of 16, last_k + 1) keeping the rows whose id is k: contiguous folds read each
 * row once and stay on the tensor-core / narrow kernels, shuffled folds cost up to n_folds passes.  The statistics stay
 * in a device block of the context (grown to the largest call); afterwards S = sum_k S_k, added in fold order, so
 * b2_solve_enet_path can refit from it.  fold_S_out: NULL or host n_folds x (d+2)^2.
 * B2_E_ARG: n_folds outside 2..254, a fold without rows, bad shapes; B2_E_UNSUPPORTED: more than one rank. */
int b2_gram_folds(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                  int mem_kind, const uint8_t* fold_of_row, int n_folds, double* fold_S_out);

/* b2_solve_enet_cv: every path of a cross-validation in one launch, one CTA per (l1_ratio l, fold k).  Path (l, k) is
 * b2_solve_enet_path's arithmetic on T_k = sum of the other folds' statistics (added in fold order) over the grid of the
 * summed statistic for l1_ratios[l] (alphas NULL; bit-identical to what b2_solve_enet_path writes for that S) or over
 * `alphas` in the order given, shared by every l1_ratio.  The held-out error of each solution (w, b) comes from S_k:
 *   mse = (vbar - b - mu.w)^2 + max(w~^T C w~, 0) / n_k,  w~ = [w; -1],
 * mu / vbar the fold's means of x / y, C the centred second moments of [x y].
 *   fold_S      NULL: the statistics of the last b2_gram_folds (same n_folds and d); else host n_folds x (d+2)^2 at the
 *               context's d, uploaded, and S becomes their sum
 *   outputs     (host) alphas_out [n_l1][n_alphas], mse_out [n_l1][n_alphas][n_folds] (sklearn's mse_path_),
 *               n_iter_out and gaps_out [n_l1][n_folds][n_alphas] (gap / n of T_k), coefs_out NULL or
 *               [n_l1][n_folds][n_alphas][d]
 * B2_E_ARG as b2_solve_enet_path, n_folds outside 2..254, n_l1 < 1, or a fold without rows; B2_E_STATE: no fold
 * statistics of this shape.  Repeated calls give identical results. */
int b2_solve_enet_cv(b2_ctx* ctx, const double* fold_S, int n_folds, int fit_intercept, const double* l1_ratios, int n_l1,
                     const double* alphas, int n_alphas, double eps, int max_iter, double tol, int positive,
                     double* alphas_out, double* mse_out, int* n_iter_out, double* gaps_out, double* coefs_out);

/* ---- ridge with the alpha chosen by leave-one-out error: replaces sklearn.linear_model.RidgeCV(alphas).fit ------
 * RidgeCV(alphas, fit_intercept).fit(X, y), cv=None: b2_fit's Gram of the kept rows, the eigendecomposition of its
 * centred Gram, then one fp64 pass over the same rows for the leave-one-out error of every alpha (DESIGN section 6).
 *   alphas    n_alphas (1..B2_MAX_ALPHAS) finite values > 0 (host)
 *   mse_out   n_alphas doubles (host): mean squared leave-one-out error per alpha (sklearn: best_score_ = -mse_out[best])
 *   cv_out    NULL, or n_rows x n_alphas doubles (row-major) where X lives (mem_kind): e^2 per row and alpha, NaN for
 *             rows not kept (sklearn: cv_results_ with store_cv_results=True, after dropping those rows)
 *   best_out  first index of the smallest mse (sklearn's tie rule); coef / intercept: the LDL^T solve at
 *             alphas[best] from the same S, bit-identical to b2_fit(alpha = alphas[best]) on the same rows and settings
 * Host rows with cv_out hold two device staging blocks of 262 144 x n_alphas doubles (134 MB at 64 alphas) in the
 * context, grown to the widest call and freed with it.
 * S afterwards is b2_fit's S.  B2_E_ARG: bad alphas / null outputs / no row kept; B2_E_UNSUPPORTED with > 1 rank;
 * B2_E_SINGULAR as b2_solve_eigh. */
#define B2_MAX_ALPHAS 64
int b2_ridge_loo(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                 int mem_kind, const uint8_t* row_mask, int mask_keep, const double* alphas, int n_alphas,
                 int fit_intercept, double* mse_out, double* cv_out, int* best_out, double* coef, double* intercept);

/* ---- BayesianRidge / ARDRegression: replaces sklearn.linear_model.BayesianRidge / ARDRegression .fit and
 * .predict(X, return_std=True) (DESIGN section 9).
 * b2_residual_moments: one fp64 pass over the kept rows at the model (coef, intercept), through the refined fit's
 * gradient kernels: out (host, d + 2 doubles) = sum (x_j - m_j) e, then sum e, then sum e^2, e = y - intercept - x.coef,
 * everything from the exactly converted stored values; m are the column means of the resident S (0 without
 * fit_intercept), which must have d features.  At the least-squares solution w0 of S (b2_fit, or b2_solve_spectral when
 * the factorisation refuses) with intercept ybar - m.w0 this is the anchor [w0 | out] of the solves below.  No rows (or
 * no kept row): out is d + 2 zeros.
 * B2_E_UNSUPPORTED with more than one rank; B2_E_STATE when the resident S has another d. */
int b2_residual_moments(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                        int mem_kind, const uint8_t* row_mask, int mask_keep, const double* coef, double intercept,
                        int fit_intercept, double* out);
/* b2_solve_bayes_ridge: BayesianRidge(...).fit on the resident S, restating scikit-learn 1.9's BayesianRidge.fit
 * (sklearn/linear_model/_bayes.py: _update_coef_, _log_marginal_likelihood, the MacKay updates of alpha_ / lambda_ and
 * the stopping test sum |coef_old - coef| < tol) in the eigenbasis of the centred Gram A = Xc^T Xc (b2_solve_eigh's
 * kernel, then one single-CTA kernel).
 *   hyper       [alpha_1, alpha_2, lambda_1, lambda_2, alpha_init, lambda_init]; a NaN init takes scikit-learn's default
 *               (1 / (y.var() + eps), 1)
 *   anchor      NULL, or [w0 (d) | g0 (d) | s0 | sse0] from b2_residual_moments at w0.  The residual sum of squares is
 *               sse(w) = sse0 - s0^2 / n - 2 (w - w0).g0 + (w - w0)^T A (w - w0) (the s0 term only with fit_intercept),
 *               exact for any w; NULL takes sse from S alone, ||yc||^2 - 2 w.r + w^T A w, whose error grows with
 *               ||yc||^2 / sse (statistics brought in by b2_gram_import)
 *   outputs     (host) coef d, intercept, alpha_out, lambda_out 1, n_iter_out; scores_out NULL or max_iter + 1 doubles
 *               (n_iter + 1 written, with compute_score: sklearn's scores_); sigma_out NULL or d x d (sklearn's sigma_)
 * Not converging within max_iter is no error (n_iter == max_iter).  B2_E_ARG: a hyper-parameter < 0 or not finite,
 * max_iter < 1, tol < 0, a null output, or a statistic without rows. */
int b2_solve_bayes_ridge(b2_ctx* ctx, int fit_intercept, const double* hyper, int max_iter, double tol,
                         const double* anchor, int compute_score, double* coef, double* intercept, double* alpha_out,
                         double* lambda_out, int* n_iter_out, double* scores_out, double* sigma_out);
/* b2_solve_ard: ARDRegression(...).fit on the resident S in one single-CTA launch, restating scikit-learn 1.9's
 * ARDRegression.fit (_update_sigma, update_coeff, the updates of lambda_ / alpha_, the prune lambda_ < threshold_lambda,
 * the score and the stopping test, in that order).  hyper = [alpha_1, alpha_2, lambda_1, lambda_2]; anchor as above;
 * lambda_out d doubles; scores_out NULL or max_iter doubles (n_iter
 * written); sigma_out NULL or d x d: sklearn's kept x kept sigma_ at the kept rows and columns, zeros
 * elsewhere (all zeros when every feature is pruned).  sigma is the exact inverse of diag(lambda) + alpha A on the kept
 * set; sklearn's pinvh drops eigenvalues below d eps lambda_max, so the two agree while that matrix has a condition
 * number below 1 / (d eps).  B2_E_SINGULAR on a non-positive pivot; B2_E_ARG as b2_solve_bayes_ridge, threshold_lambda
 * < 0, or fewer than 2 rows (sklearn's ensure_min_samples=2). */
int b2_solve_ard(b2_ctx* ctx, int fit_intercept, const double* hyper, double threshold_lambda, int max_iter, double tol,
                 const double* anchor, int compute_score, double* coef, double* intercept, double* alpha_out,
                 double* lambda_out, int* n_iter_out, double* scores_out, double* sigma_out);
/* b2_score_std: predict(X, return_std=True) of either model.  Per row, v = x - mean:
 *   ystd = sqrt(max(v^T sigma v, 0) + noise_var),  yhat = x.coef + intercept
 * mean (NULL: zeros; sklearn's X_offset_), sigma d x d, coef d: host; noise_var = 1 / alpha_.  yhat (may be NULL) and
 * ystd are n_rows fp64 where X lives (mem_kind); host rows hold two device staging blocks of 262 144 x 2 doubles in the
 * context.  One fp64 tensor-core pass over the rows; n_rows = 0 writes nothing.  B2_E_ARG: null sigma / coef / ystd,
 * noise_var < 0 or not finite. */
int b2_score_std(b2_ctx* ctx, const void* X, int x_dtype, int64_t n_rows, int d, int64_t ldx, int mem_kind,
                 const double* mean, const double* sigma, double noise_var, const double* coef, double intercept,
                 double* yhat, double* ystd);

/* ---- PoissonRegressor / GammaRegressor / TweedieRegressor (DESIGN.md section 10) --------------------------------
 * The row passes of scikit-learn's Newton solver (solver="newton-cholesky") for the half-Tweedie losses, with constants
 * dropped as sklearn drops them: per kept row eta = x.coef + intercept in fp64 from the stored value, then
 * sklearn's pointwise loss(y, eta), gradient g and Hessian h in eta.  Sums over the kept rows are unscaled (no 1 / n, no
 * penalty) and bit-identical between calls.  y: fp32 where X lives; row_mask / mask_keep as b2_score.
 * fit_intercept = 0 takes the intercept as 0.  B2_E_ARG: bad shapes, link not one of the two below, power not finite,
 * B2_GLM_IDENTITY with power != 0, null coef or outputs; B2_E_UNSUPPORTED with more than one rank.  n_rows = 0 (or no
 * kept row) is no error: every sum, the Hessian and the ladder are 0. */
#define B2_GLM_LOG 0       /* mu = exp(eta), HalfTweedieLoss(power); power 1 is HalfPoissonLoss, 2 HalfGammaLoss */
#define B2_GLM_IDENTITY 1  /* mu = eta, HalfTweedieLossIdentity, power 0 only (squared error) */
/* b2_glm_pass: one pass at (coef, intercept).  sums_out (host, d + 8 doubles): [0] sum loss [1] sum
 * constant_to_optimal_zero(y) [2] sum y [3] rows kept [4] rows with y outside the loss's interval (NaN included) [5] rows
 * with h <= 0 [6] rows with y not finite, [7, 7 + d) sum g x_j, [7 + d] sum g.  hess_out NULL (the pass skips the
 * Hessian) or (d+1) x (d+1) host doubles: sum |h| z z^T with z = [x 1], on the fp64 tensor core. */
int b2_glm_pass(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                int mem_kind, const uint8_t* row_mask, int mask_keep, int link, double power, const double* coef,
                double intercept, int fit_intercept, double* sums_out, double* hess_out);
/* b2_glm_line_search: the backtracking ladder of one Newton step in one pass: loss_out[k] = sum over kept rows of
 * loss(y, eta + 2^-k (x.step + step_intercept)) for k < n_steps (1..21; sklearn tries t = 1, 1/2, ..., 2^-20). */
int b2_glm_line_search(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                       int mem_kind, const uint8_t* row_mask, int mask_keep, int link, double power, const double* coef,
                       double intercept, const double* step, double step_intercept, int n_steps, double* loss_out);
/* b2_glm_predict: mu_out[i] = exp(eta_i) (B2_GLM_LOG) or eta_i, n_rows fp64 where X lives (mem_kind); host rows use two
 * device staging blocks of 262 144 doubles in the context. */
int b2_glm_predict(b2_ctx* ctx, const void* X, int x_dtype, int64_t n_rows, int d, int64_t ldx, int mem_kind, int link,
                   const double* coef, double intercept, double* mu_out);

/* ---- LogisticRegression, binary (DESIGN.md section 11) ----------------------------------------------------------
 * The row passes of scikit-learn's Newton solver for HalfBinomialLoss, the passes of b2_glm_pass on the half-binomial
 * loss: per kept row eta = x.coef + intercept in fp64, the target t = 1 where y == pos_label and 0 where y == neg_label,
 * and sklearn's closs_half_binomial / cgrad_hess_half_binomial branch by branch.  y: fp32 labels as stored (no binarised
 * copy); neg_label and pos_label are two distinct finite values exactly representable in fp32.  B2_E_ARG: bad shapes or
 * labels, null coef or outputs; B2_E_UNSUPPORTED with more than one rank. */
/* b2_logistic_pass: sums_out (host, d + 9 doubles): [0] sum loss [1] 0 [2] kept rows with y == pos_label [3] rows kept
 * [4] kept rows with y equal to neither label (NaN included) [5] rows with h <= 0 [6] rows with y not finite,
 * [7, 7 + d) sum g x_j, [7 + d] sum g, [8 + d] rows classified correctly: y == pos_label and eta > 0, or y == neg_label
 * and eta <= 0 (scikit-learn's predict rule).  hess_out as b2_glm_pass. */
int b2_logistic_pass(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                     int mem_kind, const uint8_t* row_mask, int mask_keep, double neg_label, double pos_label,
                     const double* coef, double intercept, int fit_intercept, double* sums_out, double* hess_out);
/* b2_logistic_line_search: loss_out[k] = sum over kept rows of the loss at eta + 2^-k (x.step + step_intercept), k <
 * n_steps (1..21), with the loss as sklearn's line search evaluates it (closs_grad_half_binomial). */
int b2_logistic_line_search(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d,
                            int64_t ldx, int mem_kind, const uint8_t* row_mask, int mask_keep, double neg_label,
                            double pos_label, const double* coef, double intercept, const double* step,
                            double step_intercept, int n_steps, double* loss_out);
/* b2_logistic_predict: per row, where X lives (mem_kind), each output optional (not all null): decision_out[i] = eta_i
 * (fp64), proba_out[2 i + c] = [1 - p_i, p_i] with p_i = 1 / (1 + exp(-eta_i)) (fp64), label_out[i] = pos_label if
 * eta_i > 0, else neg_label (fp32).  Host rows use device staging blocks in the context. */
int b2_logistic_predict(b2_ctx* ctx, const void* X, int x_dtype, int64_t n_rows, int d, int64_t ldx, int mem_kind,
                        const double* coef, double intercept, double neg_label, double pos_label, double* decision_out,
                        double* proba_out, float* label_out);
/* b2_label_scan: the labels of device fp32 y over the kept rows (row_mask / mask_keep as b2_score).  stats_out (host, 7
 * doubles): [0] kept rows [1] y not finite [2] finite y with y != rint(y) [3] min and [4] max of the finite kept y (NaN
 * when there is none) [5] kept rows equal to the min [6] kept rows equal to the max.  Counted with atomics: the result
 * does not depend on the order of the rows. */
int b2_label_scan(b2_ctx* ctx, const float* y, int64_t n_rows, const uint8_t* row_mask, int mask_keep,
                  double* stats_out);

/* ---- RidgeClassifier (DESIGN.md section 12) ----------------------------------------------------------------------
 * scikit-learn's RidgeClassifier solves (Xc^T Xc + alpha I) W = Xc^T Yc for the +-1 targets of LabelBinarizer: one target
 * (the second class) with two classes, one per class with more.  A fit is the Gram of the kept rows (b2_gram_reset +
 * b2_gram_accumulate), one b2_class_sums pass and one b2_solve_classes.  classes: n_classes (2..B2_MAX_CLASSES) finite
 * fp32 values in strictly ascending order (host); a row's class is the index of its fp32 y among them.  B2_E_ARG: bad
 * shapes, classes or null outputs; B2_E_UNSUPPORTED with more than one rank.  n_rows = 0 (or no kept row) is no error:
 * the sums and counts are 0, and b2_classify writes no row. */
#define B2_MAX_CLASSES 32
/* b2_class_sums: one fp64 pass over the kept rows (row_mask / mask_keep as b2_score; y fp32 where X lives).  sums_out
 * (host, n_classes x (d + 1)): [k][j] = sum over the kept rows of class k of x_j - center_j (j < d, x converted exactly),
 * [k][d] = their count; counts_out (host, 3): [0] kept rows [1] kept rows whose y is no class (NaN included) [2] kept rows
 * whose y is not finite.  center: NULL (zeros) or d doubles (host), the column means of S for a fit with an intercept.
 * Sums in a fixed order: repeated calls are bit-identical. */
int b2_class_sums(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                  int mem_kind, const uint8_t* row_mask, int mask_keep, const float* classes, int n_classes,
                  const double* center, double* sums_out, double* counts_out);
/* b2_class_scatter (LinearDiscriminantAnalysis, DESIGN.md section 16): the pooled within-class scatter of the kept
 * rows in one fp64 pass, scatter_out (host, d x d, both triangles, exactly symmetric) = sum over the kept rows of class
 * k of w_k (x - m_k)(x - m_k)^T, x converted exactly and u = x - m_k formed in fp64; the rows of no class add nothing.
 * classes and y as b2_class_sums; means (host, n_classes x d) the class means m_k; weights (host, n_classes; NULL: all 1)
 * the class weights w_k (1 for the scatter, p_k / n_k for the priors' covariance).  counts_out (host, 3): [0] kept rows
 * [1] kept rows whose y is no class (NaN included) [2] kept rows whose y is not finite.  On the fp64 tensor core, the
 * upper 16 x 16 blocks of the product; sums in a fixed order: repeated calls are bit-identical.  B2_E_ARG: bad shapes,
 * n_classes outside 2..B2_MAX_CLASSES, classes that are not finite and strictly ascending, null means or outputs,
 * non-finite means, weights that are negative or not finite; B2_E_UNSUPPORTED with more than one rank.  n_rows = 0 (or
 * no kept row) is no error: the scatter and counts are 0. */
int b2_class_scatter(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                     int mem_kind, const uint8_t* row_mask, int mask_keep, const float* classes, int n_classes,
                     const double* means, const double* weights, double* scatter_out, double* counts_out);
/* b2_class_scatters (QuadraticDiscriminantAnalysis, DESIGN.md section 17): every class's own scatter of the kept rows in
 * one fp64 pass that reads the rows once, in class order.  scatters_out (host, n_classes x d x d, both triangles, exactly
 * symmetric): block k = sum over the kept rows of class k of (x - m_k)(x - m_k)^T, x converted exactly and u = x - m_k
 * formed in fp64; a class without kept rows gets zeros, the rows of no class add nothing.  classes and y as
 * b2_class_sums; means (host, n_classes x d) the class means m_k.  class_counts_out (host, n_classes): the kept rows of
 * each class; counts_out (host, 3): [0] kept rows [1] kept rows whose y is no class (NaN included) [2] kept rows whose y
 * is not finite.  The work is cut by class so that skewed classes keep every SM busy; on the fp64 tensor core, the upper
 * 16 x 16 blocks of each product; sums in a fixed order: repeated calls are bit-identical.  Device scratch: 64 MB of
 * row indices plus qda_max_items x 128 KB of partials, held by the context.  B2_E_ARG: bad shapes, n_classes outside
 * 2..B2_MAX_CLASSES, classes that are not finite and strictly ascending, null means or outputs, non-finite means;
 * B2_E_UNSUPPORTED with more than one rank.  n_rows = 0 (or no kept row) is no error: the scatters and counts are 0. */
int b2_class_scatters(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                      int mem_kind, const uint8_t* row_mask, int mask_keep, const float* classes, int n_classes,
                      const double* means, double* scatters_out, double* class_counts_out, double* counts_out);
/* b2_qda_decision (QuadraticDiscriminantAnalysis, DESIGN.md section 17): per row and class in fp64,
 * d_k = -1/2 |(x - m_k) W_k|^2 + c_k, u = x - m_k formed in fp64 and u W_k on the fp64 tensor core.  means (host,
 * n_classes x d) m_k, transforms (host, n_classes x d x d, W_k row-major), offsets (host, n_classes) c_k.  Outputs where
 * the rows live, each optional (not all null): decision_out (n_rows x n_classes), label_out (fp32: classes[argmax_k
 * d_k], the first largest), diff_out (n_rows, two classes only: d_1 - d_0); counts_out (host, 2; needs y): [0] kept rows
 * [1] kept rows whose y equals their label.  Every row gets its decision and label: y and the mask only count.  Sums in
 * a fixed order: repeated calls are bit-identical.  B2_E_ARG: bad shapes, n_classes outside 2..B2_MAX_CLASSES, classes
 * that are not finite and strictly ascending, null means, transforms, offsets or outputs, non-finite means, transforms or
 * offsets, diff_out with more than two classes; B2_E_UNSUPPORTED with more than one rank. */
int b2_qda_decision(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                    int mem_kind, const uint8_t* row_mask, int mask_keep, const float* classes, int n_classes,
                    const double* means, const double* transforms, const double* offsets, double* decision_out,
                    float* label_out, double* diff_out, double* counts_out);
/* b2_solve_classes: the model of the resident S (every kept row of some class) and the class sums (host, n_classes x
 * (d + 1) as b2_class_sums returns them, at any center; NULL: the sums of the last b2_class_sums).  T = 1 for two
 * classes, else n_classes: coef_out (host, T x d) and intercept_out (host, T; ybar_t - mean.w_t, 0 without
 * fit_intercept).  Single-SM fp64 LDL^T with the T right-hand sides carried through the factorisation; B2_E_SINGULAR on a
 * non-positive pivot (the rule of b2_solve). */
int b2_solve_classes(b2_ctx* ctx, double alpha, int fit_intercept, const double* class_sums, int n_classes,
                     double* coef_out, double* intercept_out);
/* b2_classify: per row eta_t = x.coef_t + intercept_t in fp64, t < n_targets (1..B2_MAX_CLASSES); classes holds
 * max(2, n_targets) values.  Each output optional (not all null): decision_out[i][t] = eta_t (fp64, where X lives),
 * label_out[i] = classes[argmax_t eta_t] with the first largest winning, for n_targets = 1 classes[1] where eta > 0 and
 * classes[0] otherwise (fp32, where X lives); counts_out (host, 2; needs y): [0] kept rows [1] kept rows whose y equals
 * their label.  Host rows use device staging blocks in the context. */
int b2_classify(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                int mem_kind, const uint8_t* row_mask, int mask_keep, const double* coef, const double* intercept,
                int n_targets, const float* classes, double* decision_out, float* label_out, double* counts_out);
/* b2_label_values: the distinct finite values of device fp32 y over the kept rows in ascending order (-0.0 is 0.0):
 * values_out (host, max_values floats, 1 <= max_values <= B2_MAX_CLASSES) gets the first *n_values_out of them, *more_out
 * = 1 when there are more.  max_values + 1 launches of integer atomics on order-preserving keys: the result does not
 * depend on the order of the rows.  Run it after b2_label_scan has found y finite. */
int b2_label_values(b2_ctx* ctx, const float* y, int64_t n_rows, const uint8_t* row_mask, int mask_keep, int max_values,
                    float* values_out, int* n_values_out, int* more_out);

/* ---- LogisticRegression, multinomial (DESIGN.md section 14) -------------------------------------------------------
 * The row passes of scikit-learn's Newton solver for HalfMultinomialLoss with 3..B2_MAX_CLASSES classes.  Per kept row,
 * z = [x 1] and eta_k = z.coef_k in fp64 (x converted exactly), the softmax p_k = exp(eta_k - m) / s with m = max_k eta_k
 * and s the sum of the exponentials, the loss log(s) + m - eta_y and g_k = p_k - [y = k].  classes and y as
 * b2_class_sums (a row's class is the index of its fp32 y among the classes).  coef (host): n_classes x (d + 1) doubles,
 * row k = [w_k, b_k].  Sums in a fixed order: repeated calls are bit-identical.  B2_E_ARG: bad shapes, n_classes outside
 * 3..B2_MAX_CLASSES, classes that are not finite and strictly ascending, null outputs, n_steps outside 1..21;
 * B2_E_UNSUPPORTED with more than one rank.  n_rows = 0 (or no kept row) is no error: every sum is 0. */
/* b2_multinomial_pass: sums_out (host, 5 + n_classes (d + 1) doubles): [0] sum loss [1] kept rows [2] kept rows whose y
 * is no class (NaN included; their loss lacks the -eta_y term and their g the -1) [3] kept rows with y not finite [4] kept
 * rows whose first largest eta_k is their class, then G[k][j] = sum g_k z_j at 5 + k (d + 1) + j.  hess_out: NULL (no
 * Hessian), or (host) n_classes x n_classes x (d + 1) x (d + 1) doubles, block (k, l) = sum h_kl z z^T with h_kk =
 * p_k (1 - p_k) and h_kl = -p_k p_l (symmetric, and block (l, k) equals block (k, l)).  Without fit_intercept the
 * intercepts of coef are read as 0; the intercept column of the sums is always present.  One fp64 tensor-core CTA per
 * class pair and row slice. */
int b2_multinomial_pass(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                        int mem_kind, const uint8_t* row_mask, int mask_keep, const float* classes, int n_classes,
                        const double* coef, int fit_intercept, double* sums_out, double* hess_out);
/* b2_multinomial_line_search: loss_out[t] = sum over kept rows of the loss at eta + 2^-t z.step_k, t < n_steps (1..21);
 * step (host) as coef. */
int b2_multinomial_line_search(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d,
                               int64_t ldx, int mem_kind, const uint8_t* row_mask, int mask_keep, const float* classes,
                               int n_classes, const double* coef, const double* step, int n_steps, double* loss_out);
/* b2_softmax_rows: each row of the n_rows x n_cols fp64 array `values` (where mem_kind says) replaced by its softmax in
 * place, by the steps of sklearn.utils.extmath.softmax: v - max, exp, then / the sum (in column order, where numpy sums
 * 8-way unrolled and pairwise, so the two may differ by rounding).  Host values make
 * one round trip through a temporary device copy. */
int b2_softmax_rows(b2_ctx* ctx, double* values, int64_t n_rows, int n_cols, int mem_kind);

/* ---- LinearSVC / LinearSVR, primal (DESIGN.md section 15) ---------------------------------------------------------
 * The row pass of liblinear's trust-region Newton solver (TRON) for the L2-regularised squared hinge and squared
 * epsilon-insensitive losses, the GLM passes' row handling: per kept row z = [x 1] and eta = x.coef + intercept in fp64
 * (x converted exactly), at the trial point (coef, intercept) and, when coef_from is not NULL, at the accepted point
 * (coef_from, intercept_from), both by the same arithmetic in the same order.  A row is active at a point when
 *   B2_SVM_SQUARED_HINGE: m = 1 - t eta > 0, t = +1 where y == pos_label and -1 otherwise; loss m^2, g = eta - t;
 *   B2_SVM_SQUARED_EPSILON: |r| > eps with r = eta - y (eps = pos_label_or_epsilon); e = r - eps or r + eps, loss e^2,
 *   g = e.
 * Sums over the kept rows active at the trial point, unscaled (no C, no factor 2; z holds 1, not liblinear's bias
 * value), in a fixed order: repeated calls are bit-identical.  sums_out (host, d + 8 doubles): [0] sum loss [1] kept rows
 * [2] rows active at the trial point [3] rows entering the active set [4] rows leaving it [5] (squared hinge) kept rows
 * with y == pos_label [6] kept rows with y not finite, [7, 8 + d) sum g z.  dhess_out: NULL (no Hessian), or (host)
 * (d + 1) x (d + 1) doubles, sum sigma z z^T with sigma = active(trial) - active(from) in {-1, 0, 1}: the change of the
 * generalized Hessian between the two points, on the fp64 tensor core for the rows that changed side only.  coef_from =
 * NULL is the empty active set, so dhess_out is the Gram of the active rows.  fit_intercept = 0 takes both intercepts as
 * 0.  B2_E_ARG: bad shapes, an unknown loss, a non-finite pos_label, eps < 0 or not finite, null coef or sums_out;
 * B2_E_UNSUPPORTED with more than one rank.  n_rows = 0 (or no kept row) is no error: every sum is 0. */
#define B2_SVM_SQUARED_HINGE 0    /* LinearSVC(loss="squared_hinge"): liblinear's l2r_l2_svc_fun */
#define B2_SVM_SQUARED_EPSILON 1  /* LinearSVR(loss="squared_epsilon_insensitive"): liblinear's l2r_l2_svr_fun */
int b2_svm_pass(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                int mem_kind, const uint8_t* row_mask, int mask_keep, int loss, double pos_label_or_epsilon,
                const double* coef_from, double intercept_from, const double* coef, double intercept, int fit_intercept,
                double* sums_out, double* dhess_out);

/* ---- RidgeClassifierCV: replaces sklearn.linear_model.RidgeClassifierCV(alphas).fit with cv=None (DESIGN.md
 * section 13) ---------------------------------------------------------------------------------------------------------
 * The leave-one-out error of every class target and alpha: the Gram of the kept rows, b2_class_sums at its column means,
 * the eigendecomposition of the centred Gram (b2_solve_eigh), one fp64 pass over the same rows with the T targets
 * (T = 1 for two classes, else n_classes) t_k = +1 where the row's class is k (class 1 when T = 1) and -1 otherwise,
 * centred by ybar_k = 2 n_k / n - 1 with an intercept; then b2_solve_classes at alphas[best].  Per kept row, target and
 * alpha: e_k = ((t_k - ybar_k) - yhat_k) / (1 - h), p_k = t_k - e_k.  classes and y as b2_class_sums; as for
 * b2_solve_classes, the right-hand sides assume every kept row is of some class (counts_out[1] == 0).
 *   scoring      B2_LOO_SQUARED: best is the first smallest mse_out; B2_LOO_ACCURACY: the first largest correct_out
 *   mse_out      n_alphas (host): sum of e_k^2 over the kept rows and targets / (n T)
 *   correct_out  n_alphas (host): kept rows whose first argmax of p is the first argmax of t (every kept row when T = 1,
 *                as scikit-learn's accuracy scorer counts one column)
 *   cv_out       NULL, or n_rows x T x n_alphas doubles where X lives (mem_kind): e^2 (B2_LOO_SQUARED) or p
 *                (B2_LOO_ACCURACY), NaN for rows not kept.  Host rows hold two device staging blocks of at most 134 MB
 *                (fewer rows per block as T n_alphas grows) in the context.
 *   best_out     the chosen alpha's index; coef_out (T x d) and intercept_out (T): b2_solve_classes there
 *   counts_out   3 (host): the class-sum pass's kept rows, kept rows of no class, kept rows with y not finite
 * Sums in a fixed order: repeated calls are bit-identical.  B2_E_ARG: bad alphas, classes or scoring, null outputs, or
 * no kept row; B2_E_UNSUPPORTED with more than one rank; B2_E_SINGULAR from the eigendecomposition or the solve (every
 * output but coef_out / intercept_out is then written). */
#define B2_LOO_SQUARED 0
#define B2_LOO_ACCURACY 1
int b2_ridge_classifier_loo(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                            int mem_kind, const uint8_t* row_mask, int mask_keep, const float* classes, int n_classes,
                            const double* alphas, int n_alphas, int fit_intercept, int scoring, double* mse_out,
                            double* correct_out, double* cv_out, int* best_out, double* coef_out, double* intercept_out,
                            double* counts_out);

/* ---- scoring: replaces model.predict and model_metrics ------------------------------------------
 * reference: stage_1_train_model.py:107 / stage_2_serve_model.py:78 (X @ coef_ + intercept_)
 *            stage_1_train_model.py:79-90 (MAPE, r2_score, max_error)
 * yhat may be NULL (metrics only); y may be NULL (predict only; stats_out untouched).  n_rows == 0: no launch, yhat
 * untouched, stats_out (with y) ten zeros.
 * stats_out (host, 10 doubles):
 *   [0] sum |yhat-y|/max(|y|,eps_f64)  [1] sum (y-yhat)^2  [2] sum y  [3] sum y^2  [4] max |y-yhat|  [5] rows used
 *   [6] sum yhat  [7] sum yhat^2  [8] sum y*yhat  [9] max |yhat/y - 1|
 *   ([0]-[5]: stage_1's model_metrics; [6]-[9]: stage_4_test_model_scoring_service.py:89,101-105 -- APE,
 *    Pearson "r_squared", max APE.)
 * With a communicator, b2_score_allreduce combines the ten across ranks (sums; [4] and [9] by max). */
int b2_score(b2_ctx* ctx, const void* X, int x_dtype, int64_t n_rows, int d, int64_t ldx,
             int mem_kind, const double* coef, double intercept, const float* y,
             const uint8_t* row_mask, int mask_keep, float* yhat, double* stats_out);
int b2_score_allreduce(b2_ctx* ctx, double* stats_inout);
/* model_metrics(y_actual, y_predicted) (stage_1_train_model.py:79-90) on two vectors of dtype B2_F32 or B2_F64
 * (the reference works on float64 arrays): the same ten reductions as b2_score, divisions correctly rounded. */
int b2_metrics(b2_ctx* ctx, const void* y_actual, const void* y_predicted, int dtype, int64_t n_rows,
               int mem_kind, double* stats_out);

/* ---- synthetic rows on the device (benchmarks): stage_3_synthetic_data_generation.py:36-43 --------
 * X_ij ~ U(0,100), eps ~ N(0,1), y = alpha + beta * sum_j X_ij + sigma * eps   (Philox4x32-10,
 * counter = global row index + row_offset, so shards of one dataset can be drawn independently). */
int b2_synth(b2_ctx* ctx, uint64_t seed, int64_t row_offset, int64_t n_rows, int d, int64_t ldx,
             int x_dtype, double alpha, double beta, double sigma, void* X_dev, float* y_dev);

/* One reference tranche (D = 1) of day `day` >= 1, exactly as generate_dataset draws it
 * (stage_3_synthetic_data_generation.py:28-43): alpha(day) = 1 + 0.5 sin(2 pi 6 (day - 1) / 364), X ~ U(0,100),
 * y = alpha + beta X + sigma eps, rows with y < 0 dropped, order kept.  X_dev / y_dev hold n_rows floats; the
 * number of rows written comes back in *n_kept_out. */
int b2_synth_tranche(b2_ctx* ctx, uint64_t seed, int64_t n_rows, int day, double beta, double sigma,
                     float* X_dev, float* y_dev, int64_t* n_kept_out);

/* ---- multi-GPU (one process per GPU; NCCL is dlopen'ed on first use) ------------------------------ */
int b2_comm_unique_id(char* id_out /* 128 bytes */);
int b2_comm_init(b2_ctx* ctx, int n_ranks, int rank, const char* id /* 128 bytes */);
int b2_comm_destroy(b2_ctx* ctx);
int b2_comm_barrier(b2_ctx* ctx);
/* Optional one-shot peer-memory exchange for b2_gram_allreduce (2..8 ranks of one NVLink box): every rank exports
 * the CUDA-IPC handle of its exchange buffer (64 bytes), the caller gathers the handles of all ranks in rank
 * order and attaches them.  Once attached, b2_gram_allreduce stores S into every peer's buffer over NVLink and
 * sums the n slots in rank order (no NCCL launch; bit-identical S on every rank); NCCL stays the fallback. */
int b2_comm_p2p_export(b2_ctx* ctx, char* handle_out /* 64 bytes */);
int b2_comm_p2p_attach(b2_ctx* ctx, int n_ranks, int rank, const char* handles /* n_ranks x 64 bytes */);
int b2_comm_p2p_detach(b2_ctx* ctx); /* back to the NCCL all-reduce (all ranks must detach together) */
/* the same exchange between contexts of ONE process (several GPUs driven by one C client, or two contexts on one
 * GPU): peers[r] is rank r's context, peers[rank] == ctx.  Every context of the group calls it once. */
int b2_comm_p2p_attach_local(b2_ctx* ctx, int n_ranks, int rank, b2_ctx* const* peers);
/* how long a rank waits for a peer's partial statistic before the exchange fails with B2_E_COMM (default 10 000 ms) */
int b2_comm_set_timeout_ms(b2_ctx* ctx, int64_t ms);
/* ranks, this rank, and which exchange b2_gram_allreduce / b2_fit use (B2_EXCHANGE_*) */
#define B2_EXCHANGE_NONE 0
#define B2_EXCHANGE_NCCL 1
#define B2_EXCHANGE_PEER 2
int b2_comm_info(b2_ctx* ctx, int* n_ranks_out, int* rank_out, int* exchange_out);

/* ---- timing (CUDA events on the ctx stream) ---------------------------------------------------------
 * b2_timer_start/stop bracket any sequence of calls; *_ms is device time between the two events.
 * b2_last_kernel_ms: summed device time of the tensor-core Gram kernel launches (one CUDA-event pair each, at most
 * the 64 most recent) since the previous call to this function, and how many launches that sum covers. */
int b2_timer_start(b2_ctx* ctx);
int b2_timer_stop(b2_ctx* ctx, double* ms_out);
int b2_last_kernel_ms(b2_ctx* ctx, double* gram_ms_out, int* launches_out);
/* total number of kernels this ctx has launched since creation (bench.py's gpu_launches) */
int b2_launch_count(b2_ctx* ctx, int64_t* n_out);
/* out3[0] b2_fit calls whose device rows ended on the tensor-core kernel, [1] peer exchanges started, [2] kernels
 * launched */
int b2_ctx_stats(b2_ctx* ctx, int64_t* out3);

#ifdef __cplusplus
}
#endif
#endif /* B2GRAM_H_ */
