/*
 * dfb200.h -- C-ABI of libdfb200.so: the H100 (sm_90a) GP-BO inner loop behind Dragonfly's
 * Kernel / GP / gpb_acquisitions surfaces.
 *
 * The reference (dragonfly-opt 0.1.7) is pure Python + NumPy/SciPy and has NO C/FFI boundary on this
 * path (SURVEY.md 8b); the entry points below are what a ctypes binding placed at the reference's
 * three Python-level extension points would call.  Each one cites the reference function whose
 * numeric body it replaces (paths relative to the reference tree).  INTEGRATION.md shows the
 * reference-side ctypes stub.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch / C++ types.
 *   - every function returns int: 0 = ok; > 0 = LAPACK-style info (dfb_build_posterior: the 1-based
 *     index of the first non-positive pivot, i.e. np.linalg.LinAlgError in the reference -- the
 *     HOST then walks the reference's jitter ladder, general_utils.py:183-203); < 0 = argument or
 *     CUDA error, message in dfb_last_error().
 *   - all floating point data is IEEE fp64, row-major.
 *   - pointers named *_dev are device pointers on the handle's device (e.g. torch.Tensor.data_ptr());
 *     pointers with a `space` argument are host (DFB_HOST) or device (DFB_DEVICE) pointers; host
 *     buffers are copied inside the call on the handle's stream (pinned memory recommended).
 *   - the library allocates NO large device memory: the caller sizes a workspace with
 *     dfb_workspace_bytes() and hands it over with dfb_set_workspace().
 *   - a handle is not thread-safe; work is issued on the stream given to dfb_set_stream()
 *     (default: the legacy default stream) and calls that return host scalars synchronise it.
 *   - there is no CPU fallback: without a CUDA device dfb_create() fails.
 */
#ifndef DFB200_H_
#define DFB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DFB_VERSION 100

/* ---- memory spaces ------------------------------------------------------------------------- */
#define DFB_DEVICE 0
#define DFB_HOST   1

/* ---- kernel descriptor ------------------------------------------------------------------------
 * Canonical sum-of-products form of the kernels on the hot path (dragonfly/gp/kernel.py):
 *
 *     k(x, y) = post_scale * SUM_t ( ((pre_scale_t * b_{t,0}) * b_{t,1}) * ... )
 *
 * where every base factor b is an SE or half-integer Matern kernel on a subset of coordinates,
 * evaluated exactly in the reference's operation order:
 *     x~ = x[coords] / bandwidths                                   kernel.py:179-181, 255-257
 *     D2 = max(0, (|y~|^2 + |x~|^2) - 2 x~.y~)                      general_utils.py:58-70
 *     SE      b = scale * exp(-D2 / 2)                              kernel.py:171-177
 *     Matern  r = sqrt(D2); m = s8 * r; u = SUM_i coeffs[i] * m^(p-i);
 *             u *= gamma_ratio * exp(-s2 * r); b = scale * u        kernel.py:259-270, 292-299
 *             (scale here = hyperparams['scale'] * norm_constant, formed on the host)
 *   SEKernel / MaternKernel      : 1 term, 1 factor, pre_scale 1, post_scale 1
 *   AdditiveKernel               : G terms of 1 factor, post_scale = outer scale   kernel.py:484-494
 *   CoordinateProductKernel (MF) : 1 term of F factors, pre_scale = outer scale    kernel.py:573-584
 * A slot is one (coordinate, bandwidth) pair of one factor; the train and candidate matrices may
 * use different column indices for the same slot (Add-UCB scores d_j-column candidates against
 * columns g_j of the training matrix, gpb_acquisitions.py:160-168).
 *
 * esp_order = 0 selects the sum above.  esp_order = r > 0 selects the ESP kernel (Kandasamy & Yu
 * 2016; ESPKernel, kernel.py:671-744): every term is exactly one factor on one slot with
 * pre_scale 1, v_t is that factor's value, and
 *     k(x, y) = post_scale * e_r(v_1, ..., v_T)                     (1 <= r <= T = n_terms)
 * in the reference's operation order (Newton-Girard identities):
 *     p_i = ((0 + v_1^i) + v_2^i) + ... + v_T^i        i = 1..r   (^2 = v*v, ^i>=3 = pow(v, i))
 *     e_0 = 1;  e_m = ((0 + (+e_{m-1}) p_1) + (-e_{m-2}) p_2 + ... ((-1)^(m-1) e_0) p_m) / m
 * Its values may be slightly negative where the exact value is ~0 (cancellation), |k| <= k(x, x).
 *   ESPKernelSE / ESPKernelMatern : T terms of one 1-D factor (scale 1), post_scale = outer scale
 *
 * Two non-stationary factor kinds (k(x, x) depends on x) reuse the same fields:
 *     POLY      x~ = x[coords] * slot_bandwidth (a MULTIPLY: dim_scalings)             kernel.py:381-386
 *               b = scale * (x~.y~ + 1)^p          p = order (>= 0)
 *     EXPDECAY  z = x[coords] (raw), slot_bandwidth = the per-coordinate power p_q      kernel.py:415-426
 *               b = ((scale * k_1) * k_2 ...) + s2,   k_q = 1 / (1 + (z_q + z'_q))^p_q,   s2 = offset
 *   v^p follows NumPy's scalar-power fast paths: ^1 = v, ^2 = v * v, ^0.5 = sqrt(v), ^-1 = 1 / v, ^0 = 1,
 *   else pow(v, p).  Both kinds are evaluated by the descriptor interpreter only (no specialised K_* kernel).
 *   PolyKernel                   : 1 term, 1 factor (kernel_type 'poly')
 *   ExpDecayKernel               : 1 factor; the MF fidelity kernel of a CoordinateProductKernel
 * A descriptor is stationary when none of its factors is POLY or EXPDECAY; only then is kss meaningful.  The host
 * writes kss = NaN for non-stationary descriptors, and the library never runs the int8 screen or the bound pass of
 * dfb_score_argmax on them (their error model and variance floor rest on a constant k(x, x)).
 *
 * One factor kind compares categories (the categorical parts of Cartesian-product domains):
 *     HAMMING   z = x[coords] (raw: the host's non-negative integer code of each category, stored as fp64),
 *               slot_bandwidth = the per-coordinate weight w_q >= 0                    general_utils.py:113-146
 *               b = SUM_q w_q [z_q == z'_q]      each term exactly 0 or w_q, summed in NumPy's pairwise order
 *                                                (sequential below 8 terms, else 8 interleaved accumulators + tail)
 *   The factor's scale is 1 and is not read (HammingKernel has no scale).  k(x, x) = SUM_q w_q for every x, so a
 *   HAMMING factor keeps a descriptor stationary: kss = post_scale * ((pre_scale * k_0(x, x)) * k_1(x, x)) ...
 *   HammingKernel                : 1 factor; a categorical factor of a CartesianProductKernel (kernel.py:436-457)
 * HAMMING factors are evaluated by the descriptor interpreter and by dfb_lml_batch_mixed (the same comparison and sum
 * on the same staged codes); the bound pass, dfb_lml_batch and dfb_lml_gradients refuse them.
 */
#define DFB_MAX_FACTORS   48
#define DFB_MAX_TERMS     48
#define DFB_MAX_SLOTS     128
#define DFB_MAX_MATERN_P  3

#define DFB_BASE_SE        0
#define DFB_BASE_MATERN    1
#define DFB_BASE_POLY      2
#define DFB_BASE_EXPDECAY  3
#define DFB_BASE_HAMMING   4

typedef struct dfb_factor_desc {
  int32_t kind;          /* DFB_BASE_SE | DFB_BASE_MATERN | DFB_BASE_POLY | DFB_BASE_EXPDECAY | DFB_BASE_HAMMING */
  int32_t p;             /* Matern: nu = p + 1/2 (0 <= p <= DFB_MAX_MATERN_P);  POLY: order;  EXPDECAY, HAMMING: 0 */
  int32_t n_dims;        /* number of slots of this factor */
  int32_t slot_off;      /* first slot */
  double  scale;         /* SE, POLY, EXPDECAY: scale;  Matern: scale * norm_constant */
  double  s8;            /* sqrt(8 nu) */
  double  s2;            /* Matern: sqrt(2 nu);  EXPDECAY: offset */
  double  gamma_ratio;   /* Gamma(p+1) / Gamma(2p+1) */
  double  coeffs[DFB_MAX_MATERN_P + 1];  /* (p+i)! / (i! (p-i)!) */
} dfb_factor_desc;

typedef struct dfb_kernel_desc {
  int32_t n_terms;
  int32_t n_factors;
  int32_t n_slots;
  int32_t train_dim;     /* columns of the training matrix */
  int32_t cand_dim;      /* columns of the candidate matrix */
  int32_t esp_order;     /* 0: sum of products; r > 0: ESP kernel of order r (see above) */
  double  post_scale;
  double  kss;           /* k(x, x) for any x if the kernel is stationary, else NaN (see above) */
  int32_t term_first_factor[DFB_MAX_TERMS + 1];
  double  term_pre_scale[DFB_MAX_TERMS];
  dfb_factor_desc factors[DFB_MAX_FACTORS];
  int32_t slot_train_coord[DFB_MAX_SLOTS];
  int32_t slot_cand_coord[DFB_MAX_SLOTS];
  double  slot_bandwidth[DFB_MAX_SLOTS];   /* SE / Matern: bandwidth;  POLY: scaling;  EXPDECAY: power;  HAMMING: weight */
} dfb_kernel_desc;

/* ---- acquisition descriptor --------------------------------- dragonfly/opt/gpb_acquisitions.py */
#define DFB_ACQ_MEAN  0   /* score = mu                                   (uncert_form 'none')    */
#define DFB_ACQ_UCB   1   /* mu + beta * sigma                            :215-222, add_ucb :176  */
#define DFB_ACQ_EI    2   /* sigma (z Phi(z) + phi(z)), z=(mu-best)/sigma :247-260                */
#define DFB_ACQ_PI    3   /* Phi((mu - best)/sigma)                       :230-238                */
#define DFB_ACQ_TTEI  4   /* EI against a reference arm (ref_mean, ref_std) :269-279              */
#define DFB_ACQ_TS_MARGINAL 5   /* mu_i + sqrt(sigma^2_i) z_i, one normal z_i per candidate: dfb_score_argmax_ts only */

typedef struct dfb_acq_desc {
  int32_t kind;
  int32_t reserved;
  double  beta;        /* UCB: beta_th */
  double  best;        /* EI / PI: curr_max_val */
  double  ref_mean;    /* TTEI */
  double  ref_std;     /* TTEI */
} dfb_acq_desc;

/* ---- multi-objective scalarisation --------- dragonfly/opt/multiobjective_gpb_acquisitions.py */
#define DFB_MOO_MAX_OBJ 8
#define DFB_MOO_LIN_UCB 0   /* sum_k w_k mu_k + beta sqrt(sum_k w_k^2 sd_k^2)                     :79-91  */
#define DFB_MOO_TCH_UCB 1   /* min_k (mu_k + beta sqrt(sd_k) - ref_k) / w_k  (sqrt of the std, as written) :94-107 */
#define DFB_MOO_LIN_VAL 2   /* sum_k w_k v_k,  v = one posterior sample per objective (lin_ts)   :19-41  */
#define DFB_MOO_TCH_VAL 3   /* min_k (v_k - ref_k) / w_k                             (tch_ts)   :44-68  */

typedef struct dfb_moo_desc {
  int32_t kind;
  int32_t n_obj;                       /* 1 .. DFB_MOO_MAX_OBJ */
  double  beta;                        /* UCB kinds: beta_th = sqrt(0.2 d log(2 d t + 1)) (:73-75) */
  double  weight[DFB_MOO_MAX_OBJ];     /* anc_data.obj_weights */
  double  ref[DFB_MOO_MAX_OBJ];        /* anc_data.reference_point (Tchebychev kinds) */
} dfb_moo_desc;

/* ---- build flags ----------------------------------------------------------------------------- */
#define DFB_BUILD_FULL      0   /* L, W = L^-1, alpha, LML  (GP.build_posterior, gp_core.py:155-163) */
#define DFB_BUILD_LML_ONLY  1   /* L and LML only           (GPFitter._tuning_objective, :551-563)   */
#define DFB_BUILD_NO_ALPHA  2   /* L, W only; alpha is supplied with dfb_set_alpha (hallucinations)  */

typedef struct dfb_handle dfb_handle;

/* ---- life cycle ------------------------------------------------------------------------------ */
int         dfb_version(void);
const char* dfb_last_error(void);
int         dfb_create(dfb_handle** out, int device);
void        dfb_destroy(dfb_handle* h);
int         dfb_set_stream(dfb_handle* h, void* cuda_stream);
/* Bytes of device workspace needed for n_max training points, a kernel with n_slots slots and
 * scoring chunks of `chunk` candidates (chunk = 0: library default).  */
size_t      dfb_workspace_bytes(int64_t n_max, int32_t n_slots, int64_t chunk);
int         dfb_set_workspace(dfb_handle* h, void* workspace_dev, size_t bytes, int64_t n_max,
                              int64_t chunk);

/* ---- model ------------------------------------------------------------------------------------
 * dfb_set_kernel       : the GP's kernel (Kernel protocol, kernel.py:59-129), used for K(X, X).
 * dfb_set_test_kernel  : optional different descriptor for K(X*, X) and k(x*, x*) -- Add-UCB's
 *                        per-group kernel (gpb_acquisitions.py:160-176); NULL resets to the GP's.
 * dfb_set_train        : GP.set_data (gp_core.py:127-133): X (n x d) and y - mean_func(X).
 */
int dfb_set_kernel(dfb_handle* h, const dfb_kernel_desc* desc);
int dfb_set_test_kernel(dfb_handle* h, const dfb_kernel_desc* desc);
int dfb_set_train(dfb_handle* h, const double* X_dev, int64_t n, int32_t d,
                  const double* y_centred_dev);

/* GP.build_posterior (gp_core.py:155-163) + compute_log_marginal_likelihood (:222-227):
 * K = k(X,X); L = chol(K + (noise_var + jitter) I); alpha = L^-T L^-1 y_c; W = L^-1;
 * lml = -1/2 y_c^T alpha - sum log L_ii - n/2 log 2 pi.  Returns info > 0 when the matrix is not
 * positive definite (np.linalg.LinAlgError in stable_cholesky, general_utils.py:176-192).  */
int dfb_build_posterior(dfb_handle* h, double noise_var, double jitter, int32_t flags,
                        double* lml_out_host);
/* The LML of B hyper-parameter settings on the training set of dfb_set_train -- B x GPFitter._tuning_objective
 * (gp_core.py:565-574) in one launch, one CTA per item.  Pass the raw Y to dfb_set_train (mean 0): item b uses the
 * kernel descs[b] (esp_order == 0), noise_var[b] and y_c = Y - mean_const[b].  n <= 512.  lml_out[b] and info_out[b]
 * are what dfb_build_posterior(descs[b], noise_var[b], 0, DFB_BUILD_LML_ONLY) returns on the same data, bit for bit:
 * info_out[b] = 1 + index of the first non-positive pivot (lml_out[b] = NaN) or 0.  Does not touch the posterior.  One
 * host copy in, one launch, one copy out per batch that fits the scoring chunk buffer; larger B runs as several. */
int dfb_lml_batch(dfb_handle* h, const dfb_kernel_desc* descs, const double* noise_var, const double* mean_const,
                  int32_t B, double* lml_out, int32_t* info_out);
/* dfb_lml_batch for kernels with HAMMING factors as well (a CartesianProductKernel over Euclidean, integral, numeric and
 * categorical parts: CPGPFitter's tuning objective, cartesian_product_gp.py:379-391).  Same arguments, limits and
 * contract: every item is bit for bit dfb_build_posterior(descs[b], ..., DFB_BUILD_LML_ONLY) on the same data, whatever
 * else the batch holds.  A batch with a HAMMING factor runs a second instantiation of the batch kernel that compares
 * category codes; a batch without one runs dfb_lml_batch's kernel. */
int dfb_lml_batch_mixed(dfb_handle* h, const dfb_kernel_desc* descs, const double* noise_var, const double* mean_const,
                        int32_t B, double* lml_out, int32_t* info_out);
/* GP.add_data_multiple (gp_core.py:139-146) and the (N + q)-point factorisation of
 * eval_with_hallucinated_observations (gp_core.py:200-206) WITHOUT the reference's full rebuild: appends q
 * training points (X_new: q x d, y_centred_new: q) to a built posterior and re-derives only the last row block
 * of L, the last block column of L^-T / rows of W = L^-1, alpha and the LML (Cholesky row i depends on rows
 * <= i only).  Uses the kernel, noise_var and jitter of the last dfb_build_posterior.  Requires n + q to stay
 * within the posterior's padded size (multiple of 128), else returns < 0 and the caller rebuilds.
 * flags: DFB_BUILD_FULL or DFB_BUILD_NO_ALPHA, optionally | DFB_EXTEND_SAVE to snapshot what is overwritten so
 * that dfb_restore_posterior() puts the un-extended posterior back bit for bit (hallucinations are temporary).
 * Returns info > 0 if the extended matrix is not positive definite (with DFB_EXTEND_SAVE the old posterior is
 * restored first; without it the posterior is invalid and must be rebuilt).  */
#define DFB_EXTEND_SAVE 16
int dfb_extend_posterior(dfb_handle* h, const double* X_new_dev, int64_t q, const double* y_centred_new_dev,
                         int32_t flags, double* lml_out_host);
int dfb_restore_posterior(dfb_handle* h);
/* Gradients of the log marginal likelihood w.r.t. every hyper-parameter of a plain SE / Matern kernel, in one call:
 *     1/2 tr((alpha alpha^T - K^-1) dK/dparam)          GP.compute_grad_log_marginal_likelihood, gp_core.py:229-240
 * with dK/dparam = Kernel.gradient(param, X, X) (kernel.py:202-217 SE, 301-322 Matern) re-derived entry by entry
 * on the device (never materialised) and K^-1 = L^-T L^-1 from one triangular DMMA product.
 *   out_host[0]     'scale'
 *   out_host[1]     'noise_var' WITHOUT its factor noise_var: 1/2 (alpha.alpha - tr K^-1); the reference's value is
 *                   noise_var * out[1] (gp_core.py:232-233)
 *   out_host[2]     'noise_mean' = sum(alpha)                                                  gp_core.py:234-235
 *   out_host[3]     'same_dim_bandwidths'
 *   out_host[4 + j] 'dim_bandwidths', param_num = j  (j < d)
 * n_out >= 4 + d.  Needs a full posterior (DFB_BUILD_FULL).  Returns -3 for composite, ESP, POLY and EXPDECAY kernels (the
 * reference raises NotImplementedError there, kernel.py:123-125).  Uses the K_* chunk buffer as scratch. */
int dfb_lml_gradients(dfb_handle* h, double* out_host, int32_t n_out);

/* max(diag K) + noise_var of the current posterior -- the jitter ladder's scale (general_utils.py:183-189): kss + noise_var
 * for a stationary kernel, else the largest diagonal entry actually built (kept current by dfb_extend_posterior). */
int dfb_get_max_diag(dfb_handle* h, double* out_host);
/* Copies of gp.L (n x n lower), gp.alpha (n), gp.K_trtr_wo_noise (n x n); any may be NULL.
 * Read directly by _add_ucb (gpb_acquisitions.py:169-171) and gp_core.py:203.  */
int dfb_get_state(dfb_handle* h, double* L_dev, double* alpha_dev, double* K_dev);
/* Overrides alpha (n values; shorter vectors are zero-extended): eval_with_hallucinated_observations
 * takes the mean from the un-augmented GP and the variance from the augmented one
 * (gp_core.py:192-220).  */
int dfb_set_alpha(dfb_handle* h, const double* alpha_dev, int64_t n);

/* ---- prediction -------------------------------------------------------------------------------
 * GP.eval(X_test, 'none' | 'std') (gp_core.py:165-190): mu = mean_const + K_* alpha;
 * sd = sqrt(k(x*,x*) - |L^-1 k_*|^2) (no clamp: NaN for negative variances, like np.sqrt).
 * Never materialises the M x M covariance.  sd may be NULL (uncert_form 'none').  */
int dfb_eval(dfb_handle* h, const double* Xc, int64_t m, int32_t dc, int32_t space,
             double mean_const, double* mu, double* sd);
/* A certified upper bound mu_ub >= the mu of GP.eval(X_test, 'none') (gp_core.py:165-190, mean) -- at least the fp64
 * mu of dfb_eval by any of its K_* producers -- computed in single precision by the screen of dfb_score_argmax's bound
 * pass (option "prune").  +inf where the bound's analysis does not hold (coordinates beyond 2^60 after scaling), NaN
 * for rows with NaN.  Plain SE / Matern (p <= 2) kernels on <= 8 dims, no test kernel.  mu_ub_out in the space of
 * Xc.  */
int dfb_mu_upper_bound(dfb_handle* h, const double* Xc, int64_t m, int32_t dc, int32_t space, double mean_const,
                       double* mu_ub_out);
/* Optional second workspace for the block-exact joint posterior (covariance / Thompson sampling)
 * of up to `mb` candidates at a time (mb <= the scoring chunk).  */
size_t dfb_ts_workspace_bytes(int64_t n_max, int64_t mb);
int    dfb_set_ts_workspace(dfb_handle* h, void* workspace_dev, size_t bytes, int64_t mb);
/* Optional workspace for the JOINT posterior over up to m candidates at once (dfb_eval_covar, dfb_ts_draws for more
 * candidates than the TS workspace or the scoring chunk holds): about 8 Mpad^2 + 8 Mpad npad bytes plus 4 KB per
 * candidate (Mpad = m rounded up to 128, npad = n_max rounded up to 128; ~2.9 GB at m = 16384, n_max = 5000).
 * Caller-owned device memory, 256-byte aligned.  The covariance is factorised in place, so no second M x M matrix. */
size_t dfb_joint_workspace_bytes(int64_t n_max, int64_t m);
int    dfb_set_joint_workspace(dfb_handle* h, void* workspace_dev, size_t bytes, int64_t m);

/* GP.eval(X_test, 'covar') (gp_core.py:165-187): mu (m) and the full m x m posterior covariance
 * K** - V^T V, V = L^-1 K_*^T (device pointers).  Block form when the TS workspace holds m within one scoring
 * chunk, else the joint form when the joint workspace holds m; the leading q x q of a joint covariance is bit for bit
 * the block covariance of the first q candidates.  Used by draw_samples (gp_core.py:250-254). */
int dfb_eval_covar(dfb_handle* h, const double* Xc_dev, int64_t m, int32_t dc, double mean_const,
                   double* mu_dev, double* covar_dev);

/* The fused acquisition maximiser: the body of asy_ucb / asy_ei / asy_pi / _ttei / _add_ucb's
 * per-group objective + random_maximise's arg-max (oper_utils.py:70-80).  Scores every candidate
 * row and returns the FIRST index of the maximum with NaN counting as the maximum (np.argmax).
 * scores (m values, same space as Xc) may be NULL.  */
int dfb_score_argmax(dfb_handle* h, const dfb_acq_desc* acq, const double* Xc, int64_t m,
                     int32_t dc, int32_t space, double mean_const, double* scores,
                     double* best_score_host, int64_t* best_index_host);

/* Add-UCB's per-group objectives (_add_ucb, gpb_acquisitions.py:139-189) for the rows of several groups in one call,
 * as the sequential maximisers evaluate them (one point at a time, mean 0):
 *     score_r = fl(mu_r + fl(betas[g] * sd_r)),  g = group_host[r],
 * where (mu_r, sd_r) is what dfb_eval returns for row r alone, mean_const 0, with descs[g] bound by
 * dfb_set_test_kernel and option "score_impl" 0 or 2 (dfb_eval in fp64).  The contraction here is always fp64: with
 * "score_impl" 1, dfb_eval's int8 sigma may differ from it within its error bound.  Row r holds group g's
 * descs[g].cand_dim coordinates in the first columns of a host row-major matrix with ldx columns,
 * 1 <= ldx <= DFB_MAX_SLOTS.  Each group's K_* rows come from the K_* producer dfb_eval picks for its descriptor;
 * then up to 32 rows, of any groups, share one row-streaming contraction over W (the tile contraction when the workspace
 * cannot hold the streaming partials, as in dfb_eval), so m rows take ceil(m / 32) such passes.  A row's score does
 * not depend on the other rows of the call.  At most DFB_MAX_GROUPS groups, whose descriptors together use at most
 * DFB_MAX_SLOTS slots and DFB_MAX_FACTORS factors.  A test kernel bound with dfb_set_test_kernel stays bound.  Host
 * memory in and out; scores_host holds m values.  */
#define DFB_MAX_GROUPS 48
int dfb_score_groups(dfb_handle* h, const dfb_kernel_desc* descs, const double* betas, int32_t n_groups,
                     const double* X_host, int64_t m, int32_t ldx, const int32_t* group_host, double* scores_host);

/* Thompson sampling on Cartesian-product domains (asy_ts, gpb_acquisitions.py:119-127, with the `rand` maximiser of
 * _rand_maximise_vectorised_objective_in_cp_domain, exd_utils.py:247-274): the reference calls gp.draw_samples(1, [x])
 * (gp_core.py:250-254; draw_gaussian_samples, general_utils.py:224-232) once per candidate -- a 1 x 1 covariance, its
 * Cholesky factor sqrt(sigma^2) and one normal -- and takes np.argmax of the values.  Each candidate's draw is
 * independent of the others, so this is dfb_score_argmax with the acquisition DFB_ACQ_TS_MARGINAL:
 *     score_i = fl(fl(sqrt(sigma^2_i) * z_i) + mu_i)          (no FMA contraction)
 * z (m values, in the space of Xc) holds the caller's normals (np.random.normal(size=m) for seeded parity).  z = NULL:
 * the kernel generates them, z_i = element (0, row0 + i) of dfb_fill_rng(seed, ..., DFB_RNG_NORMAL), so a candidate's
 * normal depends on (seed, its global row) only.  The int8 screen applies with UCB's allowance, |z_i| in place of
 * |beta|; the bound pass (option "prune") does not run for this kind.  *n_nonpos_host (may be NULL) receives the
 * number of candidates whose fp64 sigma^2 is not > 0, NaN included: the reference's stable_cholesky raises there
 * (general_utils.py:183-203).  Their scores follow the usual NaN rules.  scores, best_score_host and best_index_host
 * as for dfb_score_argmax.  */
int dfb_score_argmax_ts(dfb_handle* h, const double* Xc, int64_t m, int32_t dc, int32_t space, double mean_const,
                        const double* z, uint64_t seed, int64_t row0, double* scores, double* best_score_host,
                        int64_t* best_index_host, int64_t* n_nonpos_host);

/* The multi-objective acquisitions' scalarisation + random_maximise's arg-max (np.argmax order) over m
 * candidates that n_obj GPs have already scored with dfb_eval on the device: a_dev[k] = mu_k (UCB kinds) or the
 * sampled values v_k (VAL kinds), b_dev[k] = sd_k (UCB kinds; NULL otherwise).  a_dev / b_dev are HOST arrays of
 * n_obj device pointers (each m doubles); scores_dev (m) may be NULL.  The handle supplies stream and scratch
 * only (any handle with a workspace on the same device).  */
int dfb_moo_score_argmax(dfb_handle* h, const dfb_moo_desc* desc, const double* const* a_dev,
                         const double* const* b_dev, int64_t m, double* scores_dev,
                         double* best_score_host, int64_t* best_index_host);

/* The multi-objective Thompson sampling acquisitions on Cartesian-product domains (mo_lin_asy_ts / mo_tch_asy_ts,
 * multiobjective_gpb_acquisitions.py:19-68, with the `rand` maximiser of
 * _rand_maximise_vectorised_objective_in_cp_domain, exd_utils.py:247-274): the reference calls every objective's
 * gp.draw_samples(1, [x]) once per candidate, so candidate i gets one marginal posterior draw per objective k,
 *     v_ik = fl(fl(sd_ik * z_ik) + mu_ik)          (no FMA contraction)
 * which desc->kind (DFB_MOO_LIN_VAL or DFB_MOO_TCH_VAL only) then scalarises as dfb_moo_score_argmax does, followed by
 * the arg-max in np.argmax order.  mu_dev / sd_dev: HOST arrays of n_obj device pointers (each m doubles, dfb_eval's mu
 * and sd).  z_dev (device, m x n_obj row-major, may be NULL): the caller's normals, in the order the reference consumes
 * them -- candidate-major, objective-minor, i.e. np.random.normal(size=(m, n_obj)).  z_dev = NULL: the kernel generates
 * them, z_ik = element (k, row0 + i) of dfb_fill_rng(seed, ..., DFB_RNG_NORMAL); for n_obj = 1 that is the normal
 * dfb_score_argmax_ts uses for the same (seed, row).  *n_nonpos_host (may be NULL) receives the number of candidates
 * with any objective's sd not > 0, NaN included (sigma^2 not > 0: the reference's stable_cholesky raises there).
 * scores_dev (m) may be NULL.  The handle supplies stream and scratch only, as for dfb_moo_score_argmax.  */
int dfb_moo_score_argmax_ts(dfb_handle* h, const dfb_moo_desc* desc, const double* const* mu_dev,
                            const double* const* sd_dev, int64_t m, const double* z_dev, uint64_t seed,
                            int64_t row0, double* scores_dev, double* best_score_host,
                            int64_t* best_index_host, int64_t* n_nonpos_host);

/* Thompson sampling at scale (BASELINE config 5: 256 draws x 10^6 candidates).  The reference draws its normals
 * with np.random.normal on the host (general_utils.py:230), which dfb_ts_draws reproduces when the caller supplies
 * them; at 10^6 x 256 that is 2 GB of host RNG and copies per call.  dfb_fill_rng generates them on the device
 * with a counter-based generator (Philox4x32-10 + Box-Muller, fp64): element (s, a) of the S x m output depends
 * only on (seed, col0 + a, s) -- the same candidate gets the same normals whatever the block or rank layout.
 * what: DFB_RNG_NORMAL or DFB_RNG_UNIFORM (53-bit uniforms in (0, 1), e.g. random_sample's U, oper_utils.py:62).
 * dfb_ts_argmax folds one block of draws (S x m, row stride ld) into running per-draw (value, index) pairs in
 * np.argmax order (sample.argmax() of asy_ts, gpb_acquisitions.py:127); reset != 0 starts a new arg-max.  */
#define DFB_RNG_NORMAL  0
#define DFB_RNG_UNIFORM 1
int dfb_fill_rng(dfb_handle* h, uint64_t seed, int64_t col0, int32_t S, int64_t m, int32_t what, double* out_dev);
int dfb_ts_argmax(dfb_handle* h, const double* samples_dev, int64_t ld, int32_t S, int64_t m, int64_t idx_base,
                  int32_t reset, double* best_dev, int64_t* index_dev);
/* random_sample + map_to_bounds (oper_utils.py:59-67, general_utils.py:25-27) on the device: rows row0 .. row0+m-1 of
 * the candidate matrix, row-major m x d, coordinate s of global row a = lo[s] + u * (hi[s] - lo[s]) with u the
 * DFB_RNG_UNIFORM element (s, a) of dfb_fill_rng for the same seed.  A row depends on (seed, its global index) only:
 * every rank generates just its shard, nobody holds the M x d matrix on the host, and the winning row is
 * regenerated from its index.  (np.random's MT19937 stream cannot be reproduced this way: the operators keep the
 * reference's host generation for seeded parity and use this in their throughput mode.)  lo / hi: HOST arrays of d.  */
int dfb_fill_candidates(dfb_handle* h, uint64_t seed, int64_t row0, int64_t m, int32_t d, const double* lo_host,
                        const double* hi_host, double* out_dev);
/* dfb_fill_candidates for the flattened rows of a Cartesian-product domain (sample_from_cp_domain_without_constraints,
 * cp_domain_utils.py:448-489), column s by kinds_host[s], from the same uniform u as dfb_fill_candidates:
 *   DFB_CAND_REAL        lo[s] + u * (hi[s] - lo[s]), bit for bit what dfb_fill_candidates writes
 *   DFB_CAND_INTEGER     that value truncated toward zero (.astype(int), oper_utils.py:337-340)
 *   DFB_CAND_CATEGORICAL a category code uniform on [0, n_levels_host[s]) (lo / hi unread), n_levels >= 1
 * Rows depend on (seed, global row index) only, as with dfb_fill_candidates.  n_levels_host may be NULL when no column
 * is categorical.  */
#define DFB_CAND_REAL        0
#define DFB_CAND_INTEGER     1
#define DFB_CAND_CATEGORICAL 2
int dfb_fill_mixed_candidates(dfb_handle* h, uint64_t seed, int64_t row0, int64_t m, int32_t d, const int32_t* kinds_host,
                              const double* lo_host, const double* hi_host, const int64_t* n_levels_host, double* out_dev);

/* Domain constraints of a Cartesian-product domain as a certified stack program (dragonfly_b200/constraints.py
 * compiles it; tests/constraint_ref.py is its NumPy oracle).  Each stack entry is a value and a radius bounding the
 * distance to NumPy's value of the same expression (radius +inf: unknown); boolean entries hold 0 (false), 1 (true) or
 * 2 (undecided).  Ops, with arg / arg2 / val:
 *   COL c; CONST val; LOOKUP column arg, entries [arg2, arg2 + val) of tab_key / tab_val (first equal key; none: unknown)
 *   ADD SUB MUL DIV (arg 1: integer operands, unknown unless |result| < 2^53), NEG, ABS, SQRT, EXP, LOG,
 *   POW exponent arg in 0..8 (arg2 1: integer), MIN MAX (Python's builtin, first operand kept on ties),
 *   NPSUM n / NORM n (pop n entries: np.sum / np.linalg.norm of them), LT LE GT GE EQ NE, AND OR NOT (three-valued),
 *   ACCEPT (pop a boolean and fold it into the row's status: any 0 rejects, else any 2 leaves it undecided).
 * Every arithmetic step is round-to-nearest without contraction, radii are formed in the same order by the oracle. */
#define DFB_CONS_MAX_OPS   128
#define DFB_CONS_MAX_STACK 16
#define DFB_CONS_MAX_TAB   64
#define DFB_CONS_MAX_VEC   16
#define DFB_CONS_OP_COL     0
#define DFB_CONS_OP_CONST   1
#define DFB_CONS_OP_LOOKUP  2
#define DFB_CONS_OP_ADD     3
#define DFB_CONS_OP_SUB     4
#define DFB_CONS_OP_MUL     5
#define DFB_CONS_OP_DIV     6
#define DFB_CONS_OP_NEG     7
#define DFB_CONS_OP_ABS     8
#define DFB_CONS_OP_SQRT    9
#define DFB_CONS_OP_EXP     10
#define DFB_CONS_OP_LOG     11
#define DFB_CONS_OP_POW     12
#define DFB_CONS_OP_MIN     13
#define DFB_CONS_OP_MAX     14
#define DFB_CONS_OP_NPSUM   15
#define DFB_CONS_OP_NORM    16
#define DFB_CONS_OP_LT      17
#define DFB_CONS_OP_LE      18
#define DFB_CONS_OP_GT      19
#define DFB_CONS_OP_GE      20
#define DFB_CONS_OP_EQ      21
#define DFB_CONS_OP_NE      22
#define DFB_CONS_OP_AND     23
#define DFB_CONS_OP_OR      24
#define DFB_CONS_OP_NOT     25
#define DFB_CONS_OP_ACCEPT  26
#define DFB_CONS_N_OPS    27
#define DFB_CONS_REJECT    0
#define DFB_CONS_ACCEPT    1
#define DFB_CONS_UNDECIDED 2
typedef struct {
  int32_t n_ops, n_tab, n_cols, reserved;
  int32_t op[DFB_CONS_MAX_OPS];
  int32_t arg[DFB_CONS_MAX_OPS];
  int32_t arg2[DFB_CONS_MAX_OPS];
  double  val[DFB_CONS_MAX_OPS];
  double  tab_key[DFB_CONS_MAX_TAB];
  double  tab_val[DFB_CONS_MAX_TAB];
} dfb_cons_prog;
/* One status byte per row of rows_dev (m x n_cols, row stride ld) in status_dev (DFB_CONS_*), and in counts_host the
 * number of rows of each status.  The program is validated here: op codes, columns < n_cols <= ld, stack depth within
 * DFB_CONS_MAX_STACK with one entry left per ACCEPT, table ranges, exponents and vector lengths. */
int dfb_constraint_status(dfb_handle* h, const dfb_cons_prog* prog, const double* rows_dev, int64_t m, int64_t ld,
                          uint8_t* status_dev, int64_t* counts_host);
/* Order-preserving compaction: the rows i of rows_dev (m x d, stride ld) with status_dev[i] == keep are written to
 * out_rows_dev (count x d, contiguous) in row order, idx_base + i to out_idx_dev, and their number to *count_host.  */
int dfb_compact_rows(dfb_handle* h, const double* rows_dev, int64_t m, int32_t d, int64_t ld, const uint8_t* status_dev,
                     int32_t keep, int64_t idx_base, double* out_rows_dev, int64_t* out_idx_dev, int64_t* count_host);

/* The GA acquisition maximiser of a Cartesian-product domain, resident on the device (the reference's CPGAOptimiser,
 * cp_ga_optimiser.py / ga_optimiser.py, driven by Philox instead of MT19937).  Rows are in the level form of
 * dfb_fill_mixed_candidates (categorical columns hold level indices); lut maps them to the column values the kernel
 * descriptor scores (Hamming codes, or the levels of a prod_discrete_numeric part).  Parts:
 *   DFB_GA_PART_REAL / _INTEGER  every column c: x + (hi - lo) / 10 * z, clipped to [lo, hi] (integer: then rounded half to
 *                                even), z = element (c, row) of dfb_fill_rng(seed, ..., DFB_RNG_NORMAL)
 *   DFB_GA_PART_CATEGORICAL      one coordinate q = c0 + floor(u1 (c1 - c0)) changes to a uniformly chosen OTHER level
 *                                floor(u2 (L_q - 1)) (skipping the current one); u1, u2 = DFB_RNG_UNIFORM elements
 *                                (1 + c0, row) and (1 + d + c0, row).  Every coordinate needs L_q >= 2.
 *   DFB_GA_PART_NUMERIC          every coordinate c: np.random.choice(levels, p = 0.8 w / sum(w) + 0.2 / L) with
 *                                w_l = exp(-|level_l - x|), levels at lut[val_off[c] ..], u = element (1 + c, row)
 * Parents of the 5 rows of an epoch starting at row r0: row r0 + j takes the inverse CDF of
 * exp((v_i - mean) / (2 (std + 1e-4))) over every value so far at u = element (0, r0 + j), uniform when a term or the sum
 * is not finite.  */
#define DFB_GA_MAX_COLS  32
#define DFB_GA_MAX_PARTS 16
#define DFB_GA_MAX_LUT   256
#define DFB_GA_PART_REAL        0
#define DFB_GA_PART_INTEGER     1
#define DFB_GA_PART_CATEGORICAL 2
#define DFB_GA_PART_NUMERIC     3
typedef struct {
  int32_t d, n_parts;
  int32_t kind[DFB_GA_MAX_COLS];        /* DFB_CAND_* */
  int32_t n_levels[DFB_GA_MAX_COLS];    /* categorical columns */
  int32_t lut_off[DFB_GA_MAX_COLS];     /* categorical columns: column value of level l = lut[lut_off + l] */
  int32_t val_off[DFB_GA_MAX_COLS];     /* DFB_GA_PART_NUMERIC columns: level l's number = lut[val_off + l] */
  int32_t part_kind[DFB_GA_MAX_PARTS];  /* DFB_GA_PART_* */
  int32_t part_c0[DFB_GA_MAX_PARTS], part_c1[DFB_GA_MAX_PARTS];   /* columns [c0, c1) */
  double  lo[DFB_GA_MAX_COLS], hi[DFB_GA_MAX_COLS];
  double  lut[DFB_GA_MAX_LUT];
} dfb_ga_desc;
/* The whole search on the handle's stream, one synchronisation at the end: rows 0 .. n_init-1 from
 * dfb_fill_mixed_candidates(seed, 0, n_init), then epochs of 5 mutated rows (ga_epoch_kernel) until n_total rows, every
 * row scored with acq (UCB / EI / PI / TTEI, fp64) into vals_dev[row].  Returns the first largest value (NaN never wins),
 * its row index and its level row.  rows_dev: n_total x d, vals_dev: n_total, coded_dev: max(n_init, 5) x d, all device
 * memory owned by the caller.  */
int dfb_ga_maximise(dfb_handle* h, const dfb_acq_desc* acq, double mean_const, const dfb_ga_desc* desc, uint64_t seed,
                    int64_t n_init, int64_t n_total, double* rows_dev, double* vals_dev, double* coded_dev,
                    double* best_value_host, int64_t* best_index_host, double* best_row_host);

/* Kernel.__call__(X1, X2) (kernel.py:72-83): the n1 x n2 Gram matrix, device pointers. */
int dfb_kernel_matrix(dfb_handle* h, const dfb_kernel_desc* desc, const double* X1_dev, int64_t n1,
                      int32_t d1, const double* X2_dev, int64_t n2, int32_t d2, double* K_dev);

/* Thompson sampling (asy_ts, gpb_acquisitions.py:119-127; GP.draw_samples, gp_core.py:250-254;
 * draw_gaussian_samples, general_utils.py:224-232): samples = (L_post U)^T + mu with
 * L_post = chol(K** - V^T V + jitter I) for ONE block of m <= mb candidates (TS workspace, S <= 256 per call), or
 * jointly over all m candidates when only the joint workspace holds them (dfb_set_joint_workspace; any S, one
 * factorisation per call, the product in passes of 256 draws).  Ut_dev is U^T, the S x m matrix of standard normals
 * (drawn on the host with np.random.normal for parity), samples_dev is S x m, mu_dev (m) may be NULL.  max_diag_host
 * receives max(diag covariance), the scale of stable_cholesky's jitter ladder.  Returns info > 0 if the covariance
 * is not PD at this jitter (the host then walks the ladder, general_utils.py:183-203; each attempt forms the
 * covariance again).  */
int dfb_ts_draws(dfb_handle* h, const double* Xc_dev, int64_t m, int32_t dc, double mean_const,
                 const double* Ut_dev, int32_t S, double jitter, double* samples_dev, double* mu_dev,
                 double* max_diag_host);

/* Counters for bench.py: number of kernels this handle has launched. */
int64_t dfb_launch_count(dfb_handle* h);
/* Diagnostics (tests/test_gpu_i8_exact.py), not on the product path: runs the int8 scoring contraction (gemm_i8.cuh)
 * on caller-owned digit planes in its pair-interleaved layout, three planes each: A = n_rb * 128 rows of W digits,
 * B = n_cb * BN rows of K_* digits (BN = 64 with radix256 = 1, 32 with radix-128 digits), both with K = n_rb * 128
 * columns.  partial_dev receives the n_rb x (n_cb * BN) partial sums, leading dimension ld_partial >= n_cb * BN;
 * rowscale_dev holds n_rb * 128 row scales; abort_count_dev may be NULL (else the launch writes nothing while
 * *abort_count_dev > 4096, the shortlist capacity).  Tile grouping as option "i8_c2_group".  Synchronises. */
int dfb_debug_score_i8(dfb_handle* h, int32_t radix256, const void* a_planes_dev, const void* b_planes_dev, int32_t n_rb,
                       int32_t n_cb, const double* rowscale_dev, double colscale, const int32_t* abort_count_dev,
                       double* partial_dev, int64_t ld_partial);
/* Diagnostics: device-to-device copy of one internal buffer of the current state; bytes must equal its size (query
 * "npad" and "chunk"): "W" (fp64 L^-1, npad^2), "Wi8" (its three digit planes, 6 npad^2 bytes), "rowscale" (npad
 * doubles), "Ki8" (the three K_* digit planes of the chunk buffer, 6 chunk npad bytes), "Ks" (fp64 K_* rows,
 * chunk x npad, written only when the digits are not emitted by the K_* kernel), "partial" ((npad / 128) x chunk),
 * "T" (the factorised tall matrix [L ; L^-T ; (L^-1 y_c)^T], (2 npad + 128) x npad: its padding, the y row), "alpha"
 * (npad doubles, padding included), "kssv" (k(x*, x*) of the last scored chunk, chunk doubles), "prune_ub" (query
 * "keep_cap" doubles: the bounds acq(mu_ub, sqrt(k**)) of the first screen launch of the last bound pass, one per row
 * of its first step, +inf for a PI row without one), "seed_idx" (query "seed_cap" int64: the global indices of the
 * last bound pass's seeds in row order, query "last_seed_rows" of them), "list_idx" (4096 int64), "list_s8" and
 * "list_err" (4096 doubles each): the shortlist of the last int8 pass or dfb_debug_acq -- global index, int8 score and
 * allowance (-1: always kept) of its first min(count, 4096) entries in append order.  With a Thompson-
 * sampling workspace (dfb_set_ts_workspace; mbp = its mb rounded up to 128, and q = the last block's m rounded up to
 * 128, whose data sits at the start of each buffer with leading dimension q): "ts_Cov" (mbp^2 doubles: the padded
 * posterior covariance of the last dfb_eval_covar / dfb_ts_draws block, q x q; dfb_ts_draws writes its lower tiles
 * only) and "ts_T" ((2 mbp + 128) mbp doubles: the tall matrix dfb_ts_draws factorised, (2 q + 128) x q, whose top is
 * the factor of Cov + jitter I); without a TS workspace these two names are an error.  With a joint workspace
 * (Mpad = its m rounded up to 128, q = the last joint call's m rounded up to 128, ld q): "js_Cov" (Mpad^2 doubles:
 * after dfb_eval_covar the q x q covariance, after dfb_ts_draws its Cholesky factor in the lower tiles, zero above the
 * diagonal inside the diagonal tiles, the covariance's K** part in the upper tiles).
 * Synchronises. */
int dfb_debug_copy(dfb_handle* h, const char* name, void* dst_dev, int64_t bytes);
/* Diagnostics (tests/test_gpu_prune_f32.py): the largest relative error of ex2.approx.ftz.f32 (which = 0) over every
 * float in [-126, 0], or of rsqrt.approx.ftz.f32 (which = 1) over every float in [2^-120, 2^126), against fp64
 * references -- the inputs the bound pass of dfb_score_argmax gives them.  Synchronises. */
int dfb_debug_approx_error(dfb_handle* h, int32_t which, double* out_host);
/* Diagnostics (tests/test_gpu_chol_diag.py), not on the product path: copies the 128 x 128 block at blk_dev (leading
 * dimension ld >= 128) to out_blk_dev (leading dimension 128) and factorises the copy in place with the diagonal-block
 * elimination of the batched LML builds (which = 0) or with the posterior build's chol_diag_kernel (which = 1): L in
 * the lower triangle, zeros above, d_j on the diagonal, L^-1 (lower) in out_dinv_dev (128 x 128).  *info_host: 0, or
 * the 1-based index of the first pivot that is not > 0, in which case nothing but the copy is written.  Synchronises. */
int dfb_debug_chol_diag(dfb_handle* h, int32_t which, const double* blk_dev, int64_t ld, double* out_blk_dev,
                        double* out_dinv_dev, int32_t* info_host);
/* Diagnostics (tests/test_gpu_acq_exact.py), not on the product path: the acquisition epilogue of dfb_score_argmax's
 * int8 pass on caller vectors, chunk by chunk of the handle's chunk size.  Per chunk: the acquisition kernel (acq->kind
 * UCB, EI, PI, TTEI or DFB_ACQ_TS_MARGINAL) with sd_i = sqrt(kss_i - ((partial[0][i] + partial[1][i]) + ...)) over
 * nrb rows of partial_dev (leading dimension ld_partial >= m; nrb = 0: sd_i = sqrt(kss_i)), the block arg-max and,
 * when b2 > 0, the running best_lb = max(best_lb, s_i - E_i) with the allowance E_i of the error model (b2, sens;
 * sens < 0: the sensitivity dfb_score_argmax uses for acq->kind; TS: sens = |z_i| whatever is passed); the merge into the running (score, index, best_lb); then the shortlist of the chunk against that
 * best_lb with slack pad (read back with dfb_debug_copy "list_idx", "list_s8", "list_err").  z_dev (TS, m values) may
 * be NULL: then z_i = element (0, i) of dfb_fill_rng(seed, ...).  best_lb is the initial value of the running bound.
 * sd_dev and scores_dev (m each) receive sd and the scores; a chunk after the shortlist overflowed (count > 4096)
 * writes nothing, as in dfb_score_argmax.  Returns the running (score, index), best_lb and the shortlist count.
 * Synchronises. */
int dfb_debug_acq(dfb_handle* h, const dfb_acq_desc* acq, const double* mu_dev, const double* partial_dev,
                  int64_t ld_partial, int32_t nrb, const double* kss_dev, int64_t m, const double* z_dev, uint64_t seed,
                  double b2, double sens, double pad, double best_lb, double* sd_dev, double* scores_dev,
                  double* best_score_host, int64_t* best_index_host, double* best_lb_host, int32_t* count_host);
/* Diagnostics: the self-check of dfb_score_argmax's int8 pass on caller vectors of count entries -- int8 scores s8,
 * allowances err (< 0: not checked) and exact scores s64.  out_host[0] = the violations it counts, out_host[1] = the
 * largest |s8 - s64| / err, scaled by 1e6 and capped at 1e9 (query "last_selfcheck_ratio" before scaling).
 * Synchronises. */
int dfb_debug_selfcheck(dfb_handle* h, const double* s8_dev, const double* err_dev, const double* s64_dev, int32_t count,
                        int32_t* out_host);

/* Tuning switches.
 *  "gemm_impl"  : 0 = cp.async-ring DMMA kernel, 1 = TMA + mbarrier warp-specialised DMMA kernel for the
 *                 fp64 scoring contraction (env DFB200_GEMM=v1|tma at dfb_create; default tma).
 *  "score_impl" : how |L^-1 k_*|^2 is contracted (env DFB200_SCORE=fp64|i8|auto at dfb_create; default auto;
 *                 readable back through dfb_query "score_impl").  ONE switch -- score_impl = 0 -- puts every call
 *                 on the pure fp64 DMMA path:
 *                 0 = fp64 DMMA everywhere (no reduced-precision arithmetic anywhere);
 *                 1 = int8-slice wgmma path everywhere, sigma vectors included (exact digit expansion of both fp64
 *                     operands, exact int32 accumulation; a-priori bound: query "i8_sigma2_bound"), except for
 *                     non-stationary kernels (POLY / EXPDECAY factors), which always score in fp64;
 *                 2 = auto: dfb_eval stays fp64; dfb_score_argmax screens with the int8 path, re-scores in fp64
 *                     every candidate whose int8 score -- widened by the error allowance that follows from the
 *                     bound -- could reach the fp64 maximum, returns the fp64 arg-max (index and score) of those,
 *                     and finally checks the int8 scores of that shortlist against the fp64 ones: a candidate
 *                     outside its allowance voids the screen and the call is redone in fp64 (queries
 *                     "last_selfcheck_violations", "last_selfcheck_ratio").  The bound (api.cu: i8_sigma2_bound) is
 *                     a sqrt(n) rounding-error model validated by a sweep (tools/sweep_i8_bound.py: 480
 *                     configurations), not a worst-case bound.  The screen is skipped when the
 *                     bound exceeds 5e-9 ABSOLUTE (half the 1e-8 sigma^2 contract, whatever the kernel scale;
 *                     query "i8_bound_limit") or n < 1024.
 *  "i8_radix"   : digit scheme of the int8 path (gemm_i8.cuh, one wgmma kernel; switching re-slices W): 1 = five
 *                 radix-256 digits, 15 products; 0 = six radix-128 digits, 21 products (about 12x more accurate);
 *                 -1 (default) = radix 256 whenever its a-priori bound is below 5e-9 (absolute) for the training
 *                 kernel, else radix 128.
 *  "i8_fuse"    : 1 (default) = the K_* kernel emits the int8 digit planes directly, 0 = via an fp64 K_* buffer.
 *  "i8_unguarded": diagnostics only (tools/sweep_i8_bound.py): 1 = run the int8 path even when its a-priori bound exceeds
 *                 the limit, so that the bound can be compared with the measured error where it would refuse.
 *  "lookahead"  : 1 (default) = look-ahead schedule of the blocked factorisation (next panel's column updated first,
 *                 chol_diag + panel solve of step k+1 overlap the bulk trailing update of step k on a second stream;
 *                 bit-identical results), 0 = one stream, step after step.
 *  "small_eval" : 1 (default) = dfb_eval of <= 32 points computes |L^-1 k_*|^2 by streaming the rows of W once (one
 *                 warp per row, HBM-bound) instead of spending 128-wide DMMA tiles on them; 0 = tile kernels always.
 *  "kstar_seg"  : 1 (default) = second-generation K_* kernels (kstar_seg_kernel: training-stationary, digits from one FMA) for
 *                 plain SE / Matern on <= 8 dims; 0 = the round-1 kernels in the reference's operation order.
 *  "kstar_rows64": 1 (default) = the fp64 K_* rows of the fp64 scoring paths come from kstar_seg_kernel's row form too.
 *  "i8_c2_group": candidate tiles per group of the int8 kernel's tile order (tiles of 64 candidates with radix-256
 *                 digits, 32 with radix-128); 0 (default) = 8.  The kernel runs in clusters of two CTAs on adjacent
 *                 tiles that share one load of the W digits, so an odd group is rounded up by one tile; query
 *                 "last_c2_group" gives the group in effect.
 *  "prune"      : 1 (default) = dfb_score_argmax's int8 path contracts only the candidates whose acquisition can reach
 *                 the arg-max.  Every candidate gets a certified upper bound mu_ub of its mean (single precision,
 *                 dfb_mu_upper_bound) and so an upper bound ub = acq(mu_ub, sqrt(k(x*, x*))) of its score (sigma^2 <=
 *                 k(x*, x*)).  The candidates with the largest ub (the seeds, option "prune_seed_rows") are scored
 *                 first and give a certain lower bound of the fp64 maximum; every other candidate is dropped when its
 *                 ub lies below it, and the survivors are scored as usual.  Index and score are those of the full
 *                 pass, bit for bit.  Applies to EI, PI and UCB with beta >= 0, plain SE / Matern (p <= 2) kernels on <= 8 dims, no
 *                 test kernel, m > chunk, no score vector, and when the posterior's variance
 *                 floor k** s / (n k** + s) (s = noise + jitter) exceeds the int8 error bound.  0 = contract every
 *                 candidate.
 *  "prune_seed_rows": K, 1..4096 (default 256): the seeds of option "prune" are the rows with the K largest bounds ub
 *                 among the first screen launch's rows (up to 2^20 device rows, or one staging batch of host rows):
 *                 every row above a threshold and the exact ties at it in row order, K to 2K rows in all (fewer when
 *                 there are fewer rows).  Any seed set gives the same result; K only sets how many rows are
 *                 contracted before the screen.
 *  "kstar_fast" : 1 (default) = plain SE / Matern kernels on <= 8 dims get specialised K_* kernels; 0 = they go through
 *                 the descriptor interpreter (kstar_kernel).  Which K_* kernel runs: kernels.cu, route_kstar.
 *  "tma_cb_group": scheduling knob of the fp64 TMA contraction. */
int dfb_set_option(dfb_handle* h, const char* name, int64_t value);
/* Diagnostics: "i8_sigma2_bound", "i8_bound_limit", "i8_ready", "i8_radix256", "score_impl",
 * "last_used_i8", "last_shortlist" (-1 = overflow -> fp64 pass), "last_selfcheck_violations" (> 0: the int8 screen
 * was voided and the call redone in fp64), "last_selfcheck_ratio" (max |s_int8 - s_fp64| / allowance over the last
 * shortlist; the model's margin is its inverse), "chunk", "npad", "last_c2_group"; "i8_impl" is always 2 (bench.py
 * reports it); "last_survivors" (candidates of rows chunk.. that the bound pass of option "prune" contracted, as
 * seeds or as survivors of the screen; > 4 chunks = overflow, the screen was voided; 0 when it did not run),
 * "last_pruned_candidates" (candidates of rows chunk.. contracted in no pass; with "last_survivors" they add up to
 * m - chunk), "last_seed_rows" (the bound pass's seeds, all rows), "last_contracted_rows" (rows of all m the bound
 * pass's int8 scoring contracted: seeds + survivors; after an overflow, seeds + m), "keep_cap", "seed_cap". */
int dfb_query(dfb_handle* h, const char* name, double* out);

/* Per-kernel-class device timing with CUDA events on the handle's stream (bench.py's roofline):
 * class 0 = K_* build (+mu), 1 = the DMMA contraction |L^-1 k_*|^2, 2 = acquisition + arg-max,
 * 3 = posterior build (whole dfb_build_posterior), 4 = the bound pass of dfb_score_argmax (upper bound of mu + screen,
 * option "prune").  dfb_profile_read synchronises, returns the accumulated milliseconds, launches and work units
 * (candidates for 0-2 and 4, builds for 3) and resets.  Class 1 counts only the candidates actually contracted. */
#define DFB_PROF_KSTAR 0
#define DFB_PROF_GEMM  1
#define DFB_PROF_ACQ   2
#define DFB_PROF_BUILD 3
#define DFB_PROF_PRUNE 4
/* The stages of dfb_build_posterior alone (tools/build_breakdown.py; dfb_extend_posterior and the Thompson-sampling
 * blocks are not counted), each on the stream it runs on, one interval per launch or group of launches, units =
 * intervals: 5 = K(X, X) and the tall matrix's initialisation, 6 = the diagonal-block Cholesky of every step, 7 = the
 * panel solves and the look-ahead's next-column updates (the critical path), 8 = the remaining trailing updates (the
 * bulk stream; all trailing updates in the single-stream schedule), 9 = the tail (W, alpha, the LML sums), 10 = the
 * scoring state of the new posterior (the int8 digit planes of W when they are made, the fp64 TMA maps). */
#define DFB_PROF_BUILD_KXX   5
#define DFB_PROF_BUILD_CHOL  6
#define DFB_PROF_BUILD_CHAIN 7
#define DFB_PROF_BUILD_REST  8
#define DFB_PROF_BUILD_TAIL  9
#define DFB_PROF_BUILD_I8    10
/* The stages of a joint dfb_ts_draws (more candidates than one block; tools/bench_ts_joint.py), one interval per call
 * on the handle's stream, units = intervals: 11 = the covariance (K_*, V^T, K**, Sigma = K** - V^T V), 12 = the
 * factor-only factorisation of Sigma + jitter I, 13 = the L U product passes with mu and the copy-out. */
#define DFB_PROF_TS_COV      11
#define DFB_PROF_TS_FACTOR   12
#define DFB_PROF_TS_PRODUCT  13
int dfb_profile_enable(dfb_handle* h, int on);
int dfb_profile_read(dfb_handle* h, int cls, double* ms_total, int64_t* launches, double* units);

/* Live roofline denominators for bench.py, measured on `device` in the calling process (best of 3 short launches):
 * DFB_PEAK_I8 -> issue rate of wgmma.m64n256k32.s32.s8.s8 from shared memory in int8 TOP/s (2 per MAC), the peak the
 * int8-slice contraction is quoted against; DFB_PEAK_DMMA_F64 -> fp64 DMMA.8x8x4 issue rate in TFLOP/s.
 * Not on the product path; replaces nothing in the reference.  */
#define DFB_PEAK_I8         0
#define DFB_PEAK_DMMA_F64   1
int dfb_measure_peak(int device, int what, double* out_host);

#ifdef __cplusplus
}
#endif
#endif  /* DFB200_H_ */
