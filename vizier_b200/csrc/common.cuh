// Shared declarations for libvzgp: handle, error plumbing, small device helpers.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/vzgp.h"
#include "acq_fn.cuh"

namespace vzgp {

constexpr int kBlk = 64;       // padding / factorisation block size
constexpr int kMaxDk = 32;     // categorical feature dims held in KernelParams; wider models take the tiled kernels
constexpr int kMaxDkWide = 1024;   // categorical feature dims of any model
constexpr int kCatTile = 32;       // categorical features the tiled (wide) kernels stage in shared memory at a time
constexpr int kMaxMetrics = 8; // metrics of the independent multi-task GP (one factor, several alpha)
constexpr size_t kMaxDynSmem = 227 * 1024;   // dynamic shared memory of one sm_90 CTA
constexpr int kNllBufs = 15;   // handle buffers a captured NLL graph points into

void set_error(const char* fmt, ...);
// Raises (never lowers: other threads may be about to launch larger) `kernel`'s dynamic shared-memory limit.
int raise_dyn_smem(const void* kernel, size_t bytes);

#define VZ_CUDA(expr)                                                              \
  do {                                                                             \
    cudaError_t _e = (expr);                                                       \
    if (_e != cudaSuccess) {                                                       \
      ::vzgp::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,              \
                        cudaGetErrorString(_e));                                   \
      return VZGP_ERR_CUDA;                                                        \
    }                                                                              \
  } while (0)

#define VZ_CHECK_LAUNCH()                                                          \
  do {                                                                             \
    cudaError_t _e = cudaGetLastError();                                           \
    if (_e != cudaSuccess) {                                                       \
      ::vzgp::set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__,          \
                        cudaGetErrorString(_e));                                   \
      return VZGP_ERR_CUDA;                                                        \
    }                                                                              \
  } while (0)

#define VZ_ARG(cond, msg)                                                          \
  do {                                                                             \
    if (!(cond)) {                                                                 \
      ::vzgp::set_error("%s:%d: bad argument: %s (%s)", __FILE__, __LINE__, msg,   \
                        #cond);                                                    \
      return VZGP_ERR_ARG;                                                         \
    }                                                                              \
  } while (0)

#define VZ_TRY(expr)                                                               \
  do {                                                                             \
    int _s = (expr);                                                               \
    if (_s < 0) return _s;                                                         \
  } while (0)

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }
inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Growable device buffer owned by a handle.
struct DevBuf {
  void* ptr = nullptr;
  size_t bytes = 0;
  int reserve(size_t n) {
    if (n <= bytes) return 0;
    if (ptr) cudaFree(ptr);
    ptr = nullptr;
    bytes = 0;
    cudaError_t e = cudaMalloc(&ptr, n);
    if (e != cudaSuccess) {
      set_error("cudaMalloc(%zu) failed: %s", n, cudaGetErrorString(e));
      return VZGP_ERR_CUDA;
    }
    bytes = n;
    return 0;
  }
  void release() {
    if (ptr) cudaFree(ptr);
    ptr = nullptr;
    bytes = 0;
  }
  template <typename T>
  T* as() const { return reinterpret_cast<T*>(ptr); }
};

// Layout of a handle's XT buffer (offsets in doubles): three [dc][np] planes of transposed trials - scaled by
// 1/ls, unscaled, and centred then scaled (k_score's fast instance) - then the [np] squared norms of the third
// plane and the [dc] centre it was taken about.  The writers (k_transpose_scale, k_centre_trials), the readers and
// the allocation all take their offsets from here.
__host__ __device__ constexpr size_t xt_plane(int p, int dc, int np) { return (size_t)p * dc * np; }
__host__ __device__ constexpr size_t xt_norms(int dc, int np) { return xt_plane(3, dc, np); }
__host__ __device__ constexpr size_t xt_centre(int dc, int np) { return xt_norms(dc, np) + np; }
__host__ __device__ constexpr size_t xt_doubles(int dc, int np) { return xt_centre(dc, np) + dc; }

// Kernel hyper-parameters in the form the kernels consume (device constant-ish,
// passed by value in kernel arguments; <= 4 KB parameter space is fine).
struct KernelParams {
  int dc;
  int dk;
  double sf2;
  double inv_ls2_c[kMaxDc];
  double inv_ls_c[kMaxDc];   // sqrt(inv_ls2_c): the reference's FeatureScaled divides by the length scale
  double inv_ls2_k[kMaxDk];      // dk <= kMaxDk
  const double* inv_ls2_k_wide;  // dk > kMaxDk: device array [dk] owned by a handle (fill_kernel_params); else null
  // linear_coef variant: k += lin_a * sum_d (x_d inv_ls_c[d] - lin_b)(x'_d inv_ls_c[d] - lin_b)
  int use_linear;
  double lin_a, lin_b;
};

// Hyper-volume scalarised UCB parameters (multi.cu); the weight tables live in handle->scal.
struct ScalArgs {
  int n_metrics = 0, n_scal = 0, has_max = 0;
  double coef = 1.8;
  double ref[kMaxMetrics] = {};
};

}  // namespace vzgp

constexpr int kNllBufsDecl = vzgp::kNllBufs;
struct vzgp_handle {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  int sm_count = 132;
  int64_t launches = 0;

  // Fitted model (all padded to np = round_up(n, 64); pad rows are identity/zero).
  bool fitted = false;
  int n = 0, np = 0, dc = 0, dk = 0, n_valid = 0, n_metrics = 1;
  vzgp::KernelParams kp;
  double sn2 = 0.0;
  double mean_const = 0.0;   // constant prior mean (linear_coef variant), 0 otherwise
  vzgp::DevBuf X;      // [np x dc]
  vzgp::DevBuf XT;     // transposed trials, norms and centre: xt_plane / xt_norms / xt_centre (the third plane,
                       // the norms and the centre are written by fits only)
  vzgp::DevBuf Z;      // [np x dk] int32
  vzgp::DevBuf L;      // [np x np]
  vzgp::DevBuf Linv;   // [np x np]
  vzgp::DevBuf LinvT;  // [np x np] L^-T (upper), produced by the dataflow factorisation (dataflow.cu)
  vzgp::DevBuf alpha;  // [n_metrics][np]
  vzgp::DevBuf ypad;   // [n_metrics][4][np]: y, w = Linv y, r, tmp
  // Models with more than kMaxDk categorical features: the inverse categorical length scales [kMaxDkWide] that kp
  // points to (allocated once, so captured graphs keep one address), and the same for the calls that must not
  // overwrite the fitted model's (stand-alone kernel matrices, the N <= 64 NLL kernel, the separable task Gram).
  // cat_sizes: the category counts of the random candidate pools (launch_random_fill_cat).
  vzgp::DevBuf wk, wk_scratch, cat_sizes;

  // Workspaces.
  vzgp::DevBuf Kws;     // [np x np] kernel matrix / temporaries
  vzgp::DevBuf Tws;     // [np x np] second temporary
  vzgp::DevBuf Kinv;    // [np x np]
  vzgp::DevBuf scratch; // per-CTA K* tiles for the score kernel
  void* scratch_window = nullptr;  // base of the L2 persisting window currently installed
  vzgp::DevBuf small;   // flags, partial reductions
  vzgp::DevBuf xs_dev;  // staging for *_host entry points
  vzgp::DevBuf out_dev;
  vzgp::DevBuf eagle;   // eagle state
  void* eagle_step = nullptr;   // EagleStepState (c_abi.cu) of a host-stepped optimiser run
  vzgp::DevBuf pe_tmp;  // GP-UCB-PE: per-candidate pieces of the two models
  vzgp::DevBuf pe_multi_tmp;  // multi-metric GP-UCB-PE (multi.cu): mu_A [n_metrics][M], sigma_A, sigma_B, L-inf, dummies
  vzgp::DevBuf gen;     // general scoring path: explicit K* and W chunks
  vzgp::DevBuf qmom;    // q-acquisitions (score_q.cu): per-member set means and covariance blocks, L-inf distances
  vzgp::DevBuf scal;    // multi-metric: [S][M] inverse scalarisation weights, then [S] best observed values
  vzgp::ScalArgs scal_args;
  // Separable multi-task GP (c_abi.cu, multi.cu): the first member handle keeps the eigenvectors Q of the task
  // covariance (row-major [sep_m][kMaxMetrics]) and the rotated labels; sep_m = 0 on every other handle.
  int sep_m = 0;
  double sep_q[vzgp::kMaxMetrics * vzgp::kMaxMetrics] = {};
  vzgp::DevBuf sep_y;   // [M][N] eigen-task labels Y Q;  NLL batches: also the task Gram workspace
  void* pinned = nullptr;
  size_t pinned_bytes = 0;
  cudaStream_t copy_stream = nullptr;   // H2D staging of vzgp_score_host, overlapped with scoring
  cudaEvent_t copy_ev[4] = {nullptr, nullptr, nullptr, nullptr};

  // CUDA graph of one NLL + gradient evaluation (c_abi.cu): the ARD loop re-evaluates the same shapes
  // and buffers hundreds of times with new hyper-parameters; only three kernel nodes take them.
  cudaGraph_t nll_graph = nullptr;
  cudaGraphExec_t nll_exec = nullptr;
  cudaGraphNode_t nll_nodes[3] = {nullptr, nullptr, nullptr};   // kernel matrix, transpose+scale, gradient tiles
  const void* nll_key[3] = {nullptr, nullptr, nullptr};          // X, Z, y
  int nll_key_dims[5] = {0, 0, 0, 0, 0};                         // N, dc, dk, n_valid, n_metrics
  const void* nll_bufs[kNllBufsDecl] = {};                                 // handle buffers the graph points into (a growth reallocates them)
  int nll_launches = 0;
  int nll_factor_route = 0;   // factor route of the captured sequence (fixed by np and VZGP_DATAFLOW)
  void* batch = nullptr;   // BatchGraph (c_abi.cu): this handle leads a batch of concurrent evaluations

  // Route of the last NLL + gradient evaluation on this handle (vzgp_nll_route) and of its last factorisation
  // (vzgp_factor_route); -1 before the first.  Tests read them through vzgp_get_int.
  int nll_route = -1, factor_route = -1;

  // Dataflow factorisation (dataflow.cu): task list for the current nb, flags, chain partial sums.
  vzgp::DevBuf df_tasks[2], df_flags, df_S;     // task lists without / with the K_y^-1 tasks
  int df_nb[2] = {0, 0}, df_ntasks[2] = {0, 0}, df_ncrit[2] = {0, 0};
  int df_ctas = 0;                              // worker CTAs per launch (0: all slots); vzgp_set_int

  // Integer-split scoring on the int8 tensor cores (score_i8.cu): digit planes of Linv, their row scales, K* digit scratch.
  int score_i8 = -1;                            // -1: environment VZGP_SCORE_I8 (default off), 0 / 1: vzgp_set_int
  bool i8_ready = false;                        // the digit planes describe the current Linv
  int64_t i8_launches = 0;
  vzgp::DevBuf i8_planes, i8_scale, i8_kdig;

  // Candidate scoring (score.cu): pools of at most small_tiles 64-candidate tiles take the small-pool kernels
  // (-1: environment VZGP_SMALL_TILES, default 8).  The last launch_score on this handle records the route it
  // took (vzgp_score_route), the CTAs sharing one tile (split route) and the grid of k_score / k_score_i8; tests
  // read them through vzgp_get_int to check which kernel a case exercised.
  int small_tiles = -1;
  int score_route = -1, score_nsplit = 0, score_grid = 0;

  // Form of the last Eagle loop on this handle (vzgp_eagle_route); -1 before the first.  A cooperative launch that was
  // refused records the graph form that ran instead.  Tests read it through vzgp_get_int.
  int eagle_route = -1;
  // ContinuousFeaturePerturbationType of the Eagle loops started on this handle (vzgp_set_int "eagle_perturbation"):
  // 0 = ADDITIVE, 1 = MULTIPLICATIVE.  Copied into EagleDev when a loop starts.
  int eagle_perturbation = 0;

  // Acquisition function set by vzgp_set_acquisition (c_abi.cu); without one the calls score UCB with their
  // vzgp_acq.ucb_coefficient.  Read at every call: no launch state is built from it.
  bool has_acq_fn = false;
  vzgp::AcqFn acq_fn;

  // MaxValueEntropySearch (mes.cu): the max-value samples, allocated once at kMaxMesSamples so that launches and
  // captured graphs see one address, the fit's scratch (trial moments), and the model they were drawn for: every
  // change of the fitted model bumps model_gen, and samples with mes_gen != model_gen are stale.
  vzgp::DevBuf mes, mes_tmp;
  int64_t model_gen = 0, mes_gen = -1;

  // Cumulative hypervolume (pareto.cu): per-CTA partial sums [CTAs][n] of the last call.
  vzgp::DevBuf pareto;

  // Fused Adam ARD (ard_adam.cu): initial points, bounds, final parameters, losses, loss trace and status of the last
  // vzgp_ard_adam_small call.
  vzgp::DevBuf ard;
};
