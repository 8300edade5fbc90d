/*
 * vzgp.h -- C ABI of libvzgp.so: the H100 (sm_90a) GP-Bandit hot path.
 *
 * The reference (google/vizier @ b0651861) has NO native/FFI layer: its
 * GP-bandit arithmetic is reached through JAX/TFP Python calls.  Each entry
 * point below replaces one of those Python call sites (cited as
 * file:line in the reference); the Python host (vizier_b200/) binds them
 * with ctypes, and INTEGRATION.md shows the stub a Vizier maintainer would
 * add to vizier/_src/algorithms/designers/gp_bandit.py.
 *
 * Conventions
 *  - extern "C", plain pointers and sizes; no C++/torch types.
 *  - Every function returns int: 0 = ok, <0 = argument/CUDA error (message via
 *    vzgp_last_error()), >0 = numeric event documented per function.  Nothing
 *    throws.
 *  - All matrices are row-major fp64.  "device" pointers are caller-owned CUDA
 *    device memory (e.g. torch.Tensor.data_ptr()); "host" pointers are ordinary
 *    host memory.  Small hyper-parameter vectors are always host memory.
 *  - A handle owns workspaces and the fitted model (X, L, L^-1, alpha).  A
 *    handle is bound to one device and one stream and must not be used from
 *    two threads at once; different handles are independent (the Vizier
 *    service runs different studies concurrently, vizier_service.py:297).
 *  - Work is enqueued on the handle's stream.  Functions that return values
 *    to HOST memory synchronise the stream before returning; the others do
 *    not.
 *  - Categorical features (int32, Hamming term of the kernel) are accepted by
 *    every entry point through (Z, Dk); pass NULL / 0 when absent.
 */
#ifndef VZGP_H_
#define VZGP_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vzgp_handle vzgp_handle;

/* Status codes (<0). */
#define VZGP_OK 0
#define VZGP_ERR_ARG (-1)
#define VZGP_ERR_CUDA (-2)
#define VZGP_ERR_STATE (-3)  /* e.g. scoring before fit */
#define VZGP_ERR_UNSUPPORTED (-4)

/* Hyper-parameters of VizierGaussianProcess (tuned_gp_models.py:161-271).
 * All host memory. */
typedef struct vzgp_params {
  double signal_variance;             /* sigma_f^2  in [1e-3, 10]   */
  double observation_noise_variance;  /* sigma_n^2  in [1e-10, 1]   */
  const double* continuous_length_scale_squared;  /* [Dc], in [1e-2, 1e2] */
  const double* categorical_length_scale_squared; /* [Dk] or NULL         */
  /* The `linear_coef` variant (tuned_gp_models.py:203-245); linear_coef = 0 switches it off.  The kernel
   * gains (coef*slope)^2 * sum_d (x_d/l_d - coef*shift)(x'_d/l_d - coef*shift) over the continuous features
   * and the GP the constant mean coef*mean_constant.  With it the gradient vectors have 3 more entries, in
   * jaxopt's sorted-key order: [cat ls2 | cont ls2 | linear_shift, linear_slope_amplitude, mean_fn | noise |
   * signal].  Such models run the general launch sequences (no captured graph, no fused small-study or
   * persistent Eagle kernels, explicit K* for the scoring). */
  double linear_coef;
  double linear_slope_amplitude;  /* in [1e-3, 10] */
  double linear_shift;            /* unbounded */
  double mean_constant;           /* unbounded */
} vzgp_params;

/* Acquisition + trust-region parameters (acquisitions.py:213-225, :152-174,
 * :691-820).  trust_radius > 0.5 disables the region exactly like the
 * reference (:160-166); pass use_trust_region = 0 for trust_region=None. */
typedef struct vzgp_acq {
  double ucb_coefficient;       /* 1.8 by default (acquisitions.py:217) */
  int use_trust_region;
  double trust_radius;          /* TrustRegion.trust_radius, computed by the host */
  const uint8_t* tr_dim_mask;   /* host [Dc]: 1 = dimension takes part; NULL = all */
  int tr_rows;                  /* trusted points = first tr_rows rows of the model's X; 0 = all valid rows */
  int tr_strict;                /* 0: inside if dist <= radius (acquisitions.py:160-166);
                                   1: inside if dist <  radius (gp_ucb_pe.py:236-241) */
} vzgp_acq;

/* Acquisition function of the single-model, ensemble and stack scoring calls (acquisitions.py:213-274,
 * :368-492), evaluated on the posterior mean mu and stddev sd of each candidate before the trust region:
 *   UCB  mu + coefficient * sd              (the default: vzgp_acq.ucb_coefficient)
 *   LCB  mu - coefficient * sd
 *   EI   imp * Phi(imp / sd) + sd * phi(imp / sd),  imp = mu - best_label - exploration  (TFP default 0.01)
 *   PI   Phi((mu - best_label - exploration) / sd)                                     (exploration 0)
 * With sd = 0 (a clamped variance) EI = max(imp, 0) and PI = (imp > 0).
 * use_threshold (AcquisitionTrustRegion): where the `thresholding` value t is not >= threshold the score is
 * bad_acq_value - t, elsewhere the `main` acquisition.  The caller resolves a NaN threshold and apply_tr_after by
 * passing use_threshold = 0. */
typedef enum vzgp_acq_kind { VZGP_ACQ_UCB = 0, VZGP_ACQ_LCB = 1, VZGP_ACQ_EI = 2, VZGP_ACQ_PI = 3 } vzgp_acq_kind;
typedef struct vzgp_acq_term {
  int kind;               /* vzgp_acq_kind */
  double coefficient;     /* UCB / LCB */
  double best_label;      /* EI / PI: finite */
  double exploration;     /* EI / PI */
} vzgp_acq_term;
typedef struct vzgp_acq_fn {
  vzgp_acq_term main;
  int use_threshold;      /* AcquisitionTrustRegion: 0 = main only */
  vzgp_acq_term thresholding;
  double threshold, bad_acq_value;
} vzgp_acq_fn;

/* Sets the acquisition function of every later call on h that takes a vzgp_acq (vzgp_score and its host / top-k
 * variants, vzgp_suggest_host, vzgp_random_search, vzgp_eagle_run and the host-stepped loop's scoring); fn = NULL
 * restores UCB with vzgp_acq.ucb_coefficient (the default).  Multi-handle calls (ensemble, stack) use the setting
 * of hs[0].  GP-UCB-PE (single- and multi-metric), set-PE and multi-metric calls ignore it.  Unknown kinds and a non-finite best_label for EI
 * or PI are rejected with VZGP_ERR_ARG. */
int vzgp_set_acquisition(vzgp_handle* h, const vzgp_acq_fn* fn);

/* GP-UCB-PE acquisition (vizier/_src/algorithms/designers/gp_ucb_pe.py:282-492) built from two
 * fitted models: A = completed trials (mean, stddev), B = completed + pending trials
 * (stddev_from_all; its labels are irrelevant).
 *   mode 0 (UCBScoreFunction, :344-381): mean_A + ucb_coefficient * stddev_B
 *   mode 1 (PEScoreFunction,  :434-492): stddev_B + penalty_coefficient *
 *                                         min(mean_A + explore_coefficient*stddev_A - threshold, 0)
 * followed by the strict trust region of :221-242 measured against the first tr_rows rows of B. */
typedef struct vzgp_pe_params {
  int mode;
  double ucb_coefficient;       /* 1.8  (mode 0) */
  double explore_coefficient;   /* 0.5  (mode 1) */
  double penalty_coefficient;   /* 10.0 (mode 1) */
  double threshold;             /* _compute_ucb_threshold (:175-218), computed by the host */
  int use_trust_region;
  double trust_radius;
  const uint8_t* tr_dim_mask;   /* host [Dc] or NULL */
  int tr_rows;                  /* 0 = all rows of B */
} vzgp_pe_params;

const char* vzgp_last_error(void);       /* thread-local message of the last failure */
int vzgp_version(void);                  /* ABI version, currently 3 (1: without the linear_* fields of vzgp_params;
                                            2: without vzgp_eagle_config.n_parallel) */
int vzgp_device_count(void);

/* device: CUDA ordinal.  stream: a cudaStream_t cast to void*, or NULL for a
 * private non-blocking stream created (and destroyed) by the handle. */
int vzgp_create(int device, void* stream, vzgp_handle** out);
int vzgp_destroy(vzgp_handle* h);
int vzgp_synchronize(vzgp_handle* h);
/* Number of kernels this library has launched through `h` so far. */
int64_t vzgp_launch_count(const vzgp_handle* h);

/* Tuning knobs.  "dataflow_ctas": worker CTAs the dataflow factorisation launches (0 = every resident slot;
 * callers that run several handles concurrently, like the ARD restarts, give each an equal share).
 * "score_i8": 1 = large candidate pools (>= one 64-candidate tile per SM, 128 <= padded N <= 4096, no linear
 * kernel) are scored by the wgmma integer-split kernel, 0 = always the FP64 DMMA kernel, -1 = the process
 * default (environment VZGP_SCORE_I8, default 0).
 * "small_tiles": pools of at most this many 64-candidate tiles take the small-pool kernels (0 = never), -1 = the
 * process default (environment VZGP_SMALL_TILES, default 8). */
int vzgp_set_int(vzgp_handle* h, const char* key, int value);

/* Route the last scoring call on a handle took (vzgp_get_int key "score_route"; -1 before the first one).
 * Every scoring entry point - vzgp_score, the host and top-k variants, GP-UCB-PE, ensemble, stack and
 * multi-metric - records it on each handle it scores with. */
typedef enum vzgp_score_route {
  VZGP_ROUTE_SMALL = 0,    /* <= small_tiles tiles: k_cross_small, k_var_small, k_small_finalize */
  VZGP_ROUTE_SPLIT = 1,    /* 2 * tiles <= SMs: k_score, score_nsplit CTAs per tile, then k_score_finalize */
  VZGP_ROUTE_CLUSTER = 2,  /* every other pool: k_score in 2-CTA clusters */
  VZGP_ROUTE_I8 = 3,       /* "score_i8" on and eligible: k_score_i8 */
  VZGP_ROUTE_GENERAL = 4   /* linear_coef models: explicit K* and W, k_general_finalize; every vzgp_score_qsets call */
} vzgp_score_route;

/* Route the last NLL + gradient evaluation on a handle took (vzgp_get_int key "nll_route"; -1 before the first).
 * vzgp_nll_grad, vzgp_nll_grad_multi and vzgp_nll_grad_batch record it on every handle they evaluate with. */
typedef enum vzgp_nll_route {
  VZGP_NLL_SMALL = 0,      /* N <= 64, one metric, no linear_coef: k_nll_grad_small (retry loop inside the kernel) */
  VZGP_NLL_GRAPH = 1,      /* the replayed single-evaluation CUDA graph, no pivot flagged */
  VZGP_NLL_EAGER = 2,      /* eager launches with the host retry loop: a pivot flagged in a graph, linear_coef or
                              VZGP_NLL_GRAPH=0; also a restart of vzgp_nll_grad_batch that fell back */
  VZGP_NLL_BATCH = 3       /* vzgp_nll_grad_batch, no pivot flagged for this restart */
} vzgp_nll_route;

/* Factorisation route of the last fit, NLL evaluation, vzgp_cholesky_retry or vzgp_factor_inverse on a handle
 * (vzgp_get_int key "factor_route"; -1 before the first).  A retry ladder records its last attempt. */
typedef enum vzgp_factor_route {
  VZGP_FACTOR_PANEL = 0,   /* 64-wide panel kernels (potrf_blocked; k_nll_grad_small factors its 64 x 64 block in
                              the same way) */
  VZGP_FACTOR_DATAFLOW = 1 /* k_chol_dataflow: factor, L^-1, L^-T (and K_y^-1 for the NLL) in one launch */
} vzgp_factor_route;

/* Counters.  "launches" (= vzgp_launch_count), "score_i8_launches": launches of the integer-split scoring kernel.
 * "sm_count": multiprocessors of the handle's device.  Of the last scoring call: "score_route" (vzgp_score_route),
 * "score_nsplit" (CTAs per 64-candidate tile: > 1 on the split route only, 1 on the cluster and i8 routes, 0
 * otherwise), "score_grid" (CTAs of the k_score / k_score_i8 launch, 0 on the other routes).  Of the last NLL
 * evaluation and factorisation: "nll_route" (vzgp_nll_route), "factor_route" (vzgp_factor_route). */
int vzgp_get_int(const vzgp_handle* h, const char* key, int64_t* value);

/* ---- stage-wise entry points (parity tests call these one by one) -------- */

/* K = K_theta(X,X) + diag_add*I, both triangles, K is [N x ldk] device.
 * Rows/cols >= n_valid are replaced by identity (padded observations,
 * stochastic_process_model.py:962-964).  Replaces the tfd.GaussianProcess
 * covariance build at tuned_gp_models.py:307-313. */
int vzgp_kernel_matrix(vzgp_handle* h, const double* X, const int32_t* Z, int N, int Dc, int Dk,
                       int n_valid, const vzgp_params* p, double diag_add, double* K, int ldk);

/* Ks[m, n] = k_theta(Xs[m], X[n]), Ks is [M x ldks] device.  Replaces the
 * kernel.matrix(x*, X) inside prior.posterior_predictive,
 * stochastic_process_model.py:830-832. */
int vzgp_cross_kernel(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const double* X,
                      const int32_t* Z, int N, int Dc, int Dk, const vzgp_params* p, double* Ks,
                      int ldks);

/* L = chol(A) with TFP retrying_cholesky semantics (tuned_gp_models.py:272-280):
 * on failure add jitter0, 10*jitter0, ... to the diagonal, at most max_iters
 * times.  A [N x lda] device (lower triangle read, not modified); L [N x ldl]
 * device (upper triangle zeroed).  Returns the number of retries (>= 0); if
 * the last attempt still fails returns max_iters+1 and L holds NaNs.
 * *shift_out (host, optional) receives the diagonal shift finally used. */
int vzgp_cholesky_retry(vzgp_handle* h, const double* A, int N, int lda, double jitter0,
                        int max_iters, double* L, int ldl, double* shift_out);

/* The factorisation stage of the fit on its own (no jitter retry): L = chol(A), Linv = L^-1 and, if Kinv !=
 * NULL, the lower triangle of A^-1 = L^-T L^-1.  A [N x lda] device (lower triangle read); L, Linv, Kinv
 * [N x ld] device.  N > 64 runs the dataflow kernel (csrc/dataflow.cu: one launch for all three), N <= 64
 * or VZGP_DATAFLOW=0 the panel kernels.  Returns 1 on a non-positive pivot (outputs hold NaN).
 * Replaces potrf / triangular_solve inside stochastic_process_model.py:940-997. */
int vzgp_factor_inverse(vzgp_handle* h, const double* A, int N, int lda, double* L, double* Linv, double* Kinv,
                        int ld);

/* Linv = L^-1 for lower-triangular L (both [N x ld] device, upper zeroed). */
int vzgp_tri_inverse(vzgp_handle* h, const double* L, int N, int ldl, double* Linv, int ldi);

/* ---- model: fit, loss, score --------------------------------------------- */

/* precompute_predictive (stochastic_process_model.py:968-997): builds K_y,
 * factors it (retrying), forms L^-1 and alpha = K_y^-1 y, and keeps X, L,
 * L^-1, alpha in the handle.  X [N x Dc], Z [N x Dk], y [N] device.  Returns
 * the number of Cholesky retries (>=0). */
int vzgp_fit(vzgp_handle* h, const double* X, const int32_t* Z, const double* y, int N, int Dc,
             int Dk, int n_valid, const vzgp_params* p);

/* Multi-metric problems: the independent multi-task GP of tuned_gp_models.py:282-288 (tfpke.Independent)
 * is n_metrics GPs sharing one kernel, one set of hyper-parameters and hence one factor; only alpha differs.
 * Y is metric-major [n_metrics x N] device (metric m contiguous at Y + m*N); n_metrics <= 8.
 * vzgp_fit / vzgp_nll_grad are the n_metrics = 1 cases.  The loss is the sum of the per-metric negative
 * log-likelihoods (+ the regularisers once): grad uses G = M K_y^-1 - sum_m alpha_m alpha_m^T. */
int vzgp_fit_multi(vzgp_handle* h, const double* X, const int32_t* Z, const double* Y, int N, int Dc,
                   int Dk, int n_valid, int n_metrics, const vzgp_params* p);
int vzgp_nll_grad_multi(vzgp_handle* h, const double* X, const int32_t* Z, const double* Y, int N, int Dc,
                        int Dk, int n_valid, int n_metrics, const vzgp_params* p, double* loss_out,
                        double* grad_out);

/* R evaluations of vzgp_nll_grad_multi - the restarts of one ARD fit, same data, different hyper-parameters -
 * in ONE graph launch: hs[r] (distinct handles and streams on one device) holds the workspaces of restart r,
 * the R launch sequences run as parallel branches of one CUDA graph, results come back through pinned host
 * memory after a single synchronisation.  ps [R] parameter structs (host), active [R] (0 = skip the update
 * and the outputs of that restart; NULL = all), loss_out [R], grad_out [R x (Dk+Dc+2)], status_out [R]
 * (Cholesky retries of the restarts that needed the jitter loop; those fall back to the single-evaluation
 * path).  N > 64.  This is what the lock-step L-BFGS-B driver (vizier_b200/ard.py) calls once per round, in
 * place of the reference's sequential restarts (jaxopt_wrappers.py:139-152). */
int vzgp_nll_grad_batch(vzgp_handle* const* hs, int R, const double* X, const int32_t* Z, const double* Y, int N,
                        int Dc, int Dk, int n_valid, int n_metrics, const vzgp_params* ps, const uint8_t* active,
                        double* loss_out, double* grad_out, int* status_out);

/* Hyper-volume scalarised UCB, the acquisition VizierGPBandit uses for multi-objective problems
 * (gp_bandit.py:214-242; acquisitions.py:571-625; scalarization.py:85-111):
 *   u_m = mu_m + ucb_coefficient * sigma            (sigma is shared by the metrics of the independent GP)
 *   score = mean_s max( (min_m max(u_m - reference_point[m], 0) / weights[s][m]) ^ n_metrics, max_scalarized[s] )
 * weights [n_scalarizations x n_metrics] (rows of unit L2 norm, positive), reference_point [n_metrics]
 * (acquisitions.py:132-149), max_scalarized [n_scalarizations] or NULL - all HOST.  No trust region
 * (gp_bandit.py:241). */
typedef struct vzgp_scalarization {
  int n_metrics;
  int n_scalarizations;          /* <= 4096; the reference default is 1000 */
  const double* weights;
  const double* reference_point;
  const double* max_scalarized;
  double ucb_coefficient;
} vzgp_scalarization;

/* Multi-metric GP-UCB-PE (gp_ucb_pe.py:344-381, :434-492) with model A fitted by vzgp_fit_multi (n_metrics metrics
 * sharing sigma_A) and model B on completed + pending trials (its labels are irrelevant: a single-metric fit on zero
 * labels will do):
 *   mode 0: u_m = mu_A,m + ucb_coefficient * sigma_B, then the hyper-volume scalarisation of `scalarization` exactly
 *           as vzgp_score_multi (floored at max_scalarized when given, mean over the rows; its ucb_coefficient is
 *           ignored)
 *   mode 1: sigma_B + agg_m( penalty_coefficient * min(mu_A,m + explore_coefficient * sigma_A - thresholds[m], 0) )
 *           with agg = mean (AVERAGE), max (UNION) or min (INTERSECTION) (MultimetricPromisingRegionPenaltyType,
 *           gp_ucb_pe.py:63-78)
 * followed by the strict trust region of :221-242 over the first tr_rows rows of B, as in vzgp_pe_params. */
typedef enum vzgp_region_penalty {
  VZGP_REGION_AVERAGE = 0,
  VZGP_REGION_UNION = 1,
  VZGP_REGION_INTERSECTION = 2
} vzgp_region_penalty;
typedef struct vzgp_pe_multi_params {
  int mode;
  double ucb_coefficient;       /* 1.8  (mode 0) */
  double explore_coefficient;   /* 0.5  (mode 1) */
  double penalty_coefficient;   /* 10.0 (mode 1) */
  int use_trust_region;
  double trust_radius;
  const uint8_t* tr_dim_mask;   /* host [Dc] or NULL */
  int tr_rows;                  /* 0 = all rows of B */
  int n_metrics;                /* must equal model A's */
  const double* thresholds;     /* host [n_metrics] (mode 1): _compute_ucb_threshold per metric (:175-218) */
  int region_penalty;           /* vzgp_region_penalty (mode 1) */
  const vzgp_scalarization* scalarization;   /* mode 0 */
} vzgp_pe_multi_params;

/* Scores M device candidates: score [M] required; mu [n_metrics x M] metric-major, sigma (model A) and sigma_all
 * (model B) [M] optional; all device.  Mode 0 uploads the scalarisation tables (synchronises once), then
 * asynchronous. */
int vzgp_score_pe_multi(vzgp_handle* hA, vzgp_handle* hB, const double* Xs, const int32_t* Zs, int M,
                        const vzgp_pe_multi_params* pe, double* score, double* mu, double* sigma, double* sigma_all);

/* Copy the fitted factor / alpha out (device destinations). */
int vzgp_get_cholesky(vzgp_handle* h, double* L, int ldl);
int vzgp_get_alpha(vzgp_handle* h, double* alpha);

/* loss_with_aux + its gradient (stochastic_process_model.py:940-966, called
 * through jaxopt at jaxopt_wrappers.py:139-152): loss = -log N(y;0,K_y) +
 * regularisers; grad in the order [categorical ls2 (Dk), continuous ls2 (Dc),
 * noise variance, signal variance] (jaxopt's sorted-key flattening).
 * loss_out [1], grad_out [Dk+Dc+2] are HOST.  Returns Cholesky retries.
 * The handle's fitted model is NOT valid afterwards (call vzgp_fit with the chosen parameters).
 * Execution: N <= 64 is one single-CTA kernel; larger N replays a CUDA graph of the launch sequence that
 * is captured on the first call with a given (X, Z, y, N, Dc, Dk, n_valid) and re-parameterised per
 * call - keep the buffers alive and unchanged in shape across an optimisation run to benefit. */
int vzgp_nll_grad(vzgp_handle* h, const double* X, const int32_t* Z, const double* y, int N, int Dc,
                  int Dk, int n_valid, const vzgp_params* p, double* loss_out, double* grad_out);

/* BayesianScoringFunction.score / score_with_aux (acquisitions.py:177-207)
 * on the fitted model: mu = K* alpha, var = sf2 - ||L^-1 K*^T||^2 + sn2
 * (clamped at 0), score = UCB then trust region.  Xs [M x Dc], Zs [M x Dk]
 * device.  score [M] device (required); mu, sigma, linf [M] device, each
 * optional (NULL).  Asynchronous on the handle's stream.  The number of candidates
 * whose variance round-off went negative and was clamped (the reference would
 * yield NaN there) accumulates in the handle; read it with vzgp_clamped_count. */
int vzgp_score(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_acq* acq,
               double* score, double* mu, double* sigma, double* linf);

/* Multi-metric counterpart of vzgp_score on a model fitted with vzgp_fit_multi: score [M] (required), mu
 * [n_metrics x M] metric-major and sigma [M] optional; all device.  Uploads the scalarisation tables
 * (synchronises once), then asynchronous. */
int vzgp_score_multi(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_scalarization* sc,
                     double* score, double* mu, double* sigma);

/* Synchronises, returns the clamp counter accumulated since the last call and resets it. */
int vzgp_clamped_count(vzgp_handle* h, int64_t* count_out);

/* Same as vzgp_score but with HOST buffers: copies Xs to the device, scores,
 * copies the requested outputs back (this is the call bench.py's e2e times). */
int vzgp_score_host(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M,
                    const vzgp_acq* acq, double* score, double* mu, double* sigma, double* linf);

/* Joint posterior over M query points (Predictor.predict/sample, gp_bandit.py:562-627;
 * acquisitions.sample_from_predictive): mean [M] and covariance [M x ldc] (device outputs),
 * cov = K** - (K* Linv^T)(K* Linv^T)^T (+ sn2 on the diagonal if add_noise, the TFP
 * posterior_predictive default).  Asynchronous on the handle's stream. */
int vzgp_posterior(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, int add_noise,
                   double* mean, double* cov, int ldc);

/* The same for a model fitted with vzgp_fit_multi: mean is [n_metrics x M] metric-major; the covariance is
 * shared by the metrics. */
int vzgp_posterior_multi(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, int add_noise,
                         double* mean, double* cov, int ldc);

/* Top-`count` of score[0..M) (device), descending, ties -> lowest index, NaN
 * treated as -inf (vectorized_base.py:580,598).  idx_out [count] int64 and
 * val_out [count] are HOST. */
int vzgp_topk(vzgp_handle* h, const double* score, int64_t M, int count, int64_t* idx_out,
              double* val_out);

/* vzgp_score + vzgp_topk + gather of the winning rows in one call and one host synchronisation
 * (the per-shard step of a multi-GPU suggest).  Xs device [M x Dc]; score_dev optional device
 * [M] buffer that receives all scores (NULL: internal).  best_x [count x Dc], best_score [count],
 * best_index [count] (optional) are HOST outputs, best first. */
int vzgp_score_topk(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_acq* acq,
                    int count, double* score_dev, double* best_x, double* best_score, int64_t* best_index);

/* Uniform ensemble of E models (UniformEnsemblePredictive.predict_with_aux,
 * stochastic_process_model.py:846-868: equal-weight MixtureSameFamily; used when
 * VizierGPBandit(ensemble_size > 1) keeps the E best ARD restarts, gp_models.py:200-223).
 * All members must be fitted on the same trials and share device and stream.
 * mean = avg mu_e;  var = avg(sigma_e^2 + mu_e^2) - mean^2;  score = UCB (+ trust region) of those.
 * mu / sigma / linf are optional device outputs [M]. */
int vzgp_score_ensemble(vzgp_handle* const* hs, int E, const double* Xs, const int32_t* Zs, int M,
                        const vzgp_acq* acq, double* score, double* mu, double* sigma, double* linf);

/* Candidate-pool shards over several GPUs (SURVEY 8e; the reference is single-process, its
 * counterpart is the arg-partition over ONE pool, vectorized_base.py:575-587).
 * vzgp_score_topk_pack: score this rank's shard, select its top `count` and write them to the DEVICE
 * buffer payload_dev[count][Dc+2] as rows [score, index_base + local index, features] (fp64; indices
 * below 2^53 are exact).  Missing winners (M < count) are [-inf, -1, 0...].  No host synchronisation:
 * the caller all-gathers the payloads (NCCL, on the handle's stream) and calls
 * vzgp_merge_topk: rows_dev[n_rows][width] -> out_dev[count][width]: larger score first, NaN as -inf,
 * ties -> lower global index (every rank computes the identical result).  If host_out != NULL the
 * merged rows are also copied there asynchronously on the handle's stream (pinned memory; valid
 * after vzgp_synchronize or an event). */
int vzgp_score_topk_pack(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_acq* acq,
                         int count, int64_t index_base, double* score_dev, double* payload_dev);
int vzgp_merge_topk(vzgp_handle* h, const double* rows_dev, int n_rows, int width, int count,
                    double* out_dev, double* host_out);

/* ---- global top-k over candidate-pool shards (one process per GPU) -------------------------------
 * SURVEY 8b/8e: the pool shards over the GPUs of one box; after vzgp_score_topk_pack every rank holds
 * count rows [score, global index, features] and needs the global top-`count` (the reference's
 * counterpart is the arg-partition over ONE pool, vectorized_base.py:575-587).  A vzgp_exchange owns a
 * small device buffer that every peer maps (CUDA IPC across processes; plain pointers inside one
 * process).  vzgp_allgather_topk(use_nccl = 0) is ONE kernel launch on the handle's stream: push the rows
 * into every peer's buffer over NVLink, publish a sequence flag (st.release.sys), wait for all peers'
 * flags (ld.acquire.sys, bounded by a timeout), merge deterministically (every rank computes the identical
 * result).  use_nccl = 1 is the checked fallback: ncclAllGather (libnccl.so.2 through dlopen, communicator
 * created by vzgp_exchange_nccl_init) + the merge kernel.  No host synchronisation either way; host_out
 * (pinned, optional) receives the merged rows by an asynchronous copy.  All ranks must call in lock-step. */
typedef struct vzgp_exchange vzgp_exchange;
int vzgp_exchange_create(vzgp_handle* h, int rank, int world, int count, int width, vzgp_exchange** out);
int vzgp_exchange_destroy(vzgp_exchange* x);
/* 64-byte cudaIpcMemHandle_t of this rank's buffer; all-gather them (any transport) and pass the
 * [world][64] array, in rank order, to vzgp_exchange_open on every rank. */
int vzgp_exchange_ipc_handle(vzgp_exchange* x, void* handle_out64);
int vzgp_exchange_open(vzgp_exchange* x, const void* handles);
/* Same-process alternative: base pointers (vzgp_exchange_base) of every rank, in rank order. */
void* vzgp_exchange_base(vzgp_exchange* x);
int vzgp_exchange_set_peers(vzgp_exchange* x, void* const* bases);
/* NCCL fallback: rank 0 draws a 128-byte ncclUniqueId, everybody calls _nccl_init with it (collective). */
int vzgp_nccl_unique_id(void* id_out128);
int vzgp_exchange_nccl_init(vzgp_exchange* x, const void* id128);
int vzgp_allgather_topk(vzgp_handle* h, vzgp_exchange* x, const double* payload_dev, double* out_dev,
                        double* host_out, int use_nccl);
/* Synchronises the stream; *status_out = 1 if a fused exchange timed out waiting for a peer
 * (VZGP_EXCHANGE_TIMEOUT_MS, default 10 s; the merged rows of that step are [-inf, -1, 0...]). */
int vzgp_exchange_status(vzgp_handle* h, vzgp_exchange* x, int* status_out);

/* One sharded suggest from HOST memory in one call (what bench.py's e2e times at every N): Xs [M x Dc]
 * host candidates of this rank's shard (pinned memory recommended) -> device (copies pipelined against
 * the scoring, as in vzgp_score_host) -> fused score -> device top-`count` -> rows [score, index_base +
 * local index, features] -> vzgp_allgather_topk over `x` (NULL: this rank alone) -> best_rows
 * [count x (Dc+2)] HOST, identical on every rank; score_host (optional, HOST [M]) receives all of this
 * shard's scores.  Synchronous.  Replaces the body of VectorizedOptimizer.__call__ for the random-pool
 * strategy on caller-provided candidates (vectorized_base.py:431-495, :575-587). */
int vzgp_suggest_host(vzgp_handle* h, vzgp_exchange* x, int use_nccl, const double* Xs, int M, const vzgp_acq* acq,
                      int count, int64_t index_base, double* score_host, double* best_rows);

/* ---- acquisition optimisers (device-resident loops) ---------------------- */

/* EagleStrategyConfig (eagle_strategy.py:111-167), continuous features. */
typedef struct vzgp_eagle_config {
  double visibility, gravity, negative_gravity;
  double perturbation, perturbation_lower_bound, penalize_factor;
  double normalization_scale, prior_trials_pool_pct;
  int pool_size;        /* P, multiple of batch_size */
  int batch_size;       /* B */
  int max_evaluations;  /* steps = (max_evaluations-1)/B + 1 */
  /* categorical mutation (eagle_strategy.py:149-151) */
  double categorical_perturbation_factor;       /* 1.0  */
  double pure_categorical_perturbation_factor;  /* 30.0 (no continuous feature) */
  double prob_same_category_without_perturbation; /* 0.98 */
  int mutate_normalization_type;  /* 0 = MEAN (default), 1 = RANDOM (eagle_strategy.py:858-885; the
                                     GP-UCB-PE default, gp_ucb_pe.py:678-692) */
  int n_parallel;       /* 0 / 1: a fly is one point.  q > 1 (host-stepped loop only, continuous features, q*Dc <= 64):
                           a fly is a SET of q points [q x Dc] scored together (set acquisitions, gp_ucb_pe.py:510-594;
                           vectorized_base.py:331-377): distances and moves over all q*Dc coordinates, forces normalised by
                           Dc, Laplace perturbations normalised over the q members of each coordinate
                           (eagle_strategy.py:1013-1046). */
} vzgp_eagle_config;

/* VectorizedOptimizer.__call__ with VectorizedEagleStrategy
 * (vectorized_base.py:324-542; eagle_strategy.py:527-1247) scoring against
 * the fitted model.  prior [n_prior x Dc] / prior_z [n_prior x Dk] device (may
 * be NULL/0) are the observed trials in creation order.  cat_sizes (host, [Dk])
 * = number of categories of each categorical feature (<= 64).  best_x
 * [count x Dc], best_z [count x Dk], best_score [count] are HOST outputs, best
 * first.  Randomness: Philox4x32-10 keyed by `seed`.
 * Execution: the whole loop runs on the device - one persistent single-CTA kernel (N <= 64 trials,
 * batch <= 64), one cooperative persistent grid (batch <= 512), otherwise a replayed CUDA graph of the
 * per-step launches; the forms agree to rounding (sums over the pool are grouped differently). */
int vzgp_eagle_run(vzgp_handle* h, const vzgp_eagle_config* cfg, const vzgp_acq* acq,
                   const double* prior, const int32_t* prior_z, int n_prior, const int32_t* cat_sizes,
                   int count, uint64_t seed, double* best_x, int32_t* best_z, double* best_score);
/* The same loop with the multi-metric scalarised UCB as the scoring function (model fitted with
 * vzgp_fit_multi). */
int vzgp_eagle_run_multi(vzgp_handle* h, const vzgp_eagle_config* cfg, const vzgp_scalarization* sc,
                         const double* prior, const int32_t* prior_z, int n_prior, const int32_t* cat_sizes,
                         int count, uint64_t seed, double* best_x, int32_t* best_z, double* best_score);
/* The same loop against a uniform ensemble (see vzgp_score_ensemble). */
int vzgp_eagle_run_ensemble(vzgp_handle* const* hs, int E, const vzgp_eagle_config* cfg, const vzgp_acq* acq,
                            const double* prior, const int32_t* prior_z, int n_prior, const int32_t* cat_sizes,
                            int count, uint64_t seed, double* best_x, int32_t* best_z, double* best_score);

/* GP-UCB-PE scoring of M device candidates with models hA / hB (same device and stream).
 * score [M] required; mu, sigma (model A) and sigma_all (model B) optional; all device. */
int vzgp_score_pe(vzgp_handle* hA, vzgp_handle* hB, const double* Xs, const int32_t* Zs, int M,
                  const vzgp_pe_params* pe, double* score, double* mu, double* sigma, double* sigma_all);

/* Transfer learning: a stack of residual GPs (StackedResidualGP, gp/gp_models.py:91-140, :245-300; VizierGPBandit.
 * set_priors, gp_bandit.py:289-318).  hs[0] is fitted on the first prior study, every further hs[e] on the residuals
 * y - (sum of the means of the levels below) of the next study, hs[E-1] on the current study.  Combined prediction
 * (gp/transfer_learning.py:62-152): mean = sum_e mean_e;  stddev: s = sd_0, then s = sd_e^alphas[e] * s^(1 - alphas[e])
 * for e = 1 .. E-1 (alphas[0] unused; the caller derives them from the levels' degrees of freedom).  UCB / trust
 * region as in vzgp_score, the trust region measured against the trials of hs[E-1].  All levels share device, stream
 * and feature dimensions. */
int vzgp_score_stack(vzgp_handle* const* hs, int E, const double* alphas, const double* Xs, const int32_t* Zs, int M,
                     const vzgp_acq* acq, double* score, double* mu, double* sigma, double* linf);
int vzgp_eagle_run_stack(vzgp_handle* const* hs, int E, const double* alphas, const vzgp_eagle_config* cfg,
                         const vzgp_acq* acq, const double* prior, const int32_t* prior_z, int n_prior,
                         const int32_t* cat_sizes, int count, uint64_t seed, double* best_x, int32_t* best_z,
                         double* best_score);

/* Set-PE acquisition of GP-UCB-PE batches (SetPEScoreFunction, gp_ucb_pe.py:510-594): Xs holds n_sets sets of q points
 * ([n_sets * q x Dc] device, continuous features, q <= 16).  score[s] = logdet of the q x q joint predictive covariance
 * under model B (completed + pending trials) + penalty * sum_i min(mean_A + explore * stddev_A - threshold, 0)
 * (+ the set trust-region term, :245-269); -inf when the covariance block is not positive definite (:495-507).
 * mu / sigma (model A) and sigma_all (sqrt of the diagonal of B's covariance), each [n_sets * q], are optional. */
int vzgp_score_set_pe(vzgp_handle* hA, vzgp_handle* hB, const double* Xs, int n_sets, int q, const vzgp_pe_params* pe,
                      double* score, double* mu, double* sigma, double* sigma_all);

/* Parallel (q-) acquisitions (acquisitions.py:495-568): Monte Carlo estimates over the joint posterior predictive of
 * a set of q points.  Per set, with mean mu [q] and covariance Sigma [q x q] (observation noise on the diagonal),
 * L = Cholesky of Sigma (unshifted, then shifts 1e-4 * 10^k, k < 5; a set whose factor still fails scores NaN) and
 * S draws f_s = mu + L z_s:
 *   QEI   mean_s max_j max(f_sj - best_label - 0.01, 0)
 *   QPI   mean_s [max_j f_sj - best_label > 0]
 *   QUCB  mean_s max_j (mu_j + coefficient * |f_sj - mu_j|)
 * A non-finite best_label (no observation) makes QEI and QPI score mean_s max_j f_sj.  Ensembles (E members) are
 * the uniform mixture: each (set, sample) draws one member and samples all q points from it; QUCB's mu is the
 * mixture mean.  Draws depend on the set's position p = set index mod period (common random numbers across the
 * batches of an optimiser run): z for (p, s, j) from Philox stream 12, elements 2e and 2e + 1 with e = (p S + s) q + j
 * (Box-Muller), the member from stream 13, element p S + s.  With the trust region on and trust_radius <= 0.5, each
 * point farther than the radius (L-inf, over tr_dim_mask) from the first tr_rows trials adds -1e4 - distance
 * (gp_ucb_pe.py:245-269). */
typedef enum vzgp_qacq_kind { VZGP_QACQ_QEI = 0, VZGP_QACQ_QPI = 1, VZGP_QACQ_QUCB = 2 } vzgp_qacq_kind;
typedef struct vzgp_qacq {
  int kind;                     /* vzgp_qacq_kind */
  double best_label;            /* QEI / QPI */
  double coefficient;           /* QUCB */
  int num_samples;              /* S, 1 .. 8192 */
  int period;                   /* positions repeat every `period` sets; <= 0: n_sets */
  int use_trust_region;
  double trust_radius;
  const uint8_t* tr_dim_mask;   /* host [Dc] or NULL (all dimensions) */
  int tr_rows;                  /* 0 = all valid trials */
  double* cov_out;              /* optional device [E][n_sets][q][q]: the covariance blocks */
} vzgp_qacq;

/* Scores n_sets sets of q points (Xs [n_sets * q x Dc], Zs [n_sets * q x Dk], device) under the E models hs (E = 1: a
 * single model; members must be fitted on the same trials and share device and stream).  1 <= q <= 16, E <= 16.
 * Device outputs: score [n_sets]; optional mu (mixture mean), sigma (mixture stddev) and linf (L-inf distance to the
 * trusted trials), each [n_sets * q].  K* and W = K* L^-T go through the general route in chunks of whole sets. */
int vzgp_score_qsets(vzgp_handle* const* hs, int E, const double* Xs, const int32_t* Zs, int n_sets, int q,
                     const vzgp_qacq* qa, uint64_t seed, double* score, double* mu, double* sigma, double* linf);
/* The Monte Carlo stage alone on given moments: mean [E][n_sets * q], cov [E][n_sets][q][q] (device).  The trust
 * region fields are ignored. */
int vzgp_qacq_from_moments(vzgp_handle* h, int n_sets, int q, int E, const double* mean, const double* cov,
                           const vzgp_qacq* qa, uint64_t seed, double* score);

/* Host-stepped form of the same optimiser: identical device-resident state and kernels, but the CALLER scores every
 * batch - for acquisitions libvzgp cannot evaluate by itself, e.g. one with a user-supplied `prior_acquisition` term
 * (gp_ucb_pe.py:286-381, :589-592; the reference calls `acquisition_optimizer(scoring_fn.score, ...)` with an arbitrary
 * callable, vectorized_base.py:431-495).  begin -> [write n_prior prior rewards to *prior_rewards_dev, seed] ->
 * repeat { ask: batch features [B x Dc] / [B x Dk] on the device and where to put the B rewards; tell } -> end
 * (winners to the host; synchronises).  Everything else is asynchronous on the handle's stream. */
int vzgp_eagle_begin(vzgp_handle* h, const vzgp_eagle_config* cfg, const int32_t* cat_sizes, int count, uint64_t seed,
                     int n_prior, double** prior_rewards_dev);
int vzgp_eagle_seed(vzgp_handle* h, const double* prior, const int32_t* prior_z);
int vzgp_eagle_ask(vzgp_handle* h, const double** batch_x_dev, const int32_t** batch_z_dev, double** batch_rewards_dev);
int vzgp_eagle_tell(vzgp_handle* h);
int vzgp_eagle_end(vzgp_handle* h, double* best_x, int32_t* best_z, double* best_score);

/* vzgp_eagle_run with the GP-UCB-PE acquisition as the scoring function (gp_ucb_pe.py:1006-1155). */
int vzgp_eagle_run_pe(vzgp_handle* hA, vzgp_handle* hB, const vzgp_eagle_config* cfg,
                      const vzgp_pe_params* pe, const double* prior, const int32_t* prior_z, int n_prior,
                      const int32_t* cat_sizes, int count, uint64_t seed, double* best_x, int32_t* best_z,
                      double* best_score);
/* The same with the multi-metric GP-UCB-PE acquisition (vzgp_score_pe_multi); always the replayed-graph form of
 * the loop. */
int vzgp_eagle_run_pe_multi(vzgp_handle* hA, vzgp_handle* hB, const vzgp_eagle_config* cfg,
                            const vzgp_pe_multi_params* pe, const double* prior, const int32_t* prior_z, int n_prior,
                            const int32_t* cat_sizes, int count, uint64_t seed, double* best_x, int32_t* best_z,
                            double* best_score);

/* RandomVectorizedStrategy with batch = max_evaluations = M
 * (random_vectorized_optimizer.py:32-123): generates M uniform candidates on
 * the device (Philox), scores them, returns the top `count` (HOST outputs).
 * index_base offsets the Philox element counter so ranks can generate
 * disjoint shards of one global pool: candidate g = index_base + m. */
int vzgp_random_search(vzgp_handle* h, int64_t M, int64_t index_base, const vzgp_acq* acq,
                       const int32_t* cat_sizes, int count, uint64_t seed, double* best_x,
                       int32_t* best_z, double* best_score, int64_t* best_index);

/* Fill X [M x Dc] (device) with the same Philox uniforms vzgp_random_search
 * uses (stream STREAM_RANDOM_POOL), for parity tests and the benchmark. */
int vzgp_random_pool(vzgp_handle* h, int64_t M, int Dc, int64_t index_base, uint64_t seed,
                     double* X);
/* Categorical counterpart: Z [M x Dk] int32 device, uniform over [0, cat_sizes[k]). */
int vzgp_random_pool_cat(vzgp_handle* h, int64_t M, int Dk, const int32_t* cat_sizes,
                         int64_t index_base, uint64_t seed, int32_t* Z);

#ifdef __cplusplus
}
#endif
#endif /* VZGP_H_ */
