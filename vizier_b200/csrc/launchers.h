// Internal prototypes of the per-file launch helpers (all return 0 or a negative vzgp status).
#pragma once
#include <tuple>
#include <type_traits>

#include "acq_fn.cuh"
#include "common.cuh"

namespace vzgp {

int fill_kernel_params(const vzgp_params* p, int dc, int dk, KernelParams* kp);
int launch_kernel_matrix(vzgp_handle* h, const double* X, const int32_t* Z, int n, int n_valid,
                         const KernelParams& kp, double diag_add, double* K, int ldk);
int launch_cross_kernel(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const double* X,
                        const int32_t* Z, int n, int n_valid, const KernelParams& kp, double* Ks,
                        int ldks);
int potrf_blocked(vzgp_handle* h, double* L, int ld, double* Linv, int ldi, int np, int* flag);
int trtri_doubling(vzgp_handle* h, const double* L, int ld, double* Linv, int ldi, double* T, int ldt,
                   int np);
// The captured NLL graph (c_abi.cu, nll_graph_eval) re-parameterises three kernel nodes per evaluation by
// ARGUMENT POSITION.  The positions live here, next to the prototypes, and each kernel's translation unit
// static_asserts them against its real signature (KernelArgs), so a signature change cannot silently write
// the hyper-parameters into the wrong slot.
constexpr int kKernelMatrixArgs = 8, kKernelMatrixKpArg = 4, kKernelMatrixDiagArg = 5;
constexpr int kTransposeScaleArgs = 5, kTransposeScaleKpArg = 3;
constexpr int kNllGradTilesArgs = 13, kNllGradTilesKpArg = 4;
template <class F> struct KernelArgs;
template <class... A> struct KernelArgs<void (*)(A...)> {
  static constexpr int count = (int)sizeof...(A);
  template <int I> using arg = typename std::tuple_element<I, std::tuple<A...>>::type;
};
// Host-side entry addresses of the three kernels whose arguments carry the hyper-parameters (graph node lookup).
const void* kernel_matrix_func();
const void* transpose_scale_func();
const void* nll_grad_tiles_func();
constexpr int kLauumSplit = 4;   // K_y^-1 is produced as this many partial planes [z][np][ldk] (linalg.cu)
int lauum_plane_rows(int np);
int launch_sum_planes(vzgp_handle* h, double* Kinv, int np, int kc);
int launch_lauum(vzgp_handle* h, const double* Linv, int ldi, double* Kinv, int ldk, int np);
int launch_copy_lower_shift(vzgp_handle* h, const double* A, int lda, int n_src, int np, double shift,
                            double* L, int ldl);
int launch_diag_inv(vzgp_handle* h, const double* L, int ld, double* Linv, int ldi, int np);
int launch_gemv_rows(vzgp_handle* h, const double* M, int ld, int np, const double* v, double* out,
                     int lower_only, int ncols = 0);
int launch_gemv_lower_T(vzgp_handle* h, const double* M, int ld, int np, const double* v, double* out);
int launch_residual(vzgp_handle* h, const double* Ky, int ld, int np, const double* y, const double* a,
                    double* r);
int launch_axpy(vzgp_handle* h, int n, double a, const double* x, double* y);
int launch_add_scalar(vzgp_handle* h, int n, double a, double* y);
int launch_pad_vector(vzgp_handle* h, const double* src, int n, int n_valid, int np, double* dst, double offset = 0.0);
int launch_pad_rows(vzgp_handle* h, const double* src, int n, int d, int np, double* dst);
int launch_transpose_scale(vzgp_handle* h, const double* X, int np, int dc, const KernelParams& kp, double* XT);
int launch_pad_rows_i32(vzgp_handle* h, const int32_t* src, int n, int d, int np, int32_t* dst);
int launch_logdet_quad(vzgp_handle* h, const double* L, int ld, int n, int n_valid, const double* w, double* out,
                       int wstride = 0, int n_metrics = 1, const double* alpha = nullptr);

int launch_gemm_nt_tri(vzgp_handle* h, const double* A, int lda, int mp, const double* B, int ldb, int np,
                       double* C, int ldc);
int launch_cov_update(vzgp_handle* h, const double* W, int ldw, int kdim, int mp, double* C, int ldc,
                      double diag_add);

int launch_nll_grad_tiles(vzgp_handle* h, const double* X, const int32_t* Z, int np, int n_valid,
                          const KernelParams& kp, const double* Kinv, int ldk, const double* alpha,
                          double* partial, double* out, int plane_rows = 0, int n_metrics = 1);

// CUtensorMap (passed as void*) of an fp64 row-major matrix [rows x cols], row pitch ld elements, boxes of
// box_rows x 16 doubles with the 128-byte swizzle (score.cu).
int make_tensor_map_f64(void* map, const double* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows);

// Blocked Cholesky + both triangular inverses (+ K_y^-1) as ONE dataflow kernel (dataflow.cu): L (lower,
// holds the shifted matrix on entry), Linv = L^-1 (lower), LinvT = L^-T (upper), optional Kinv (lower
// tiles of L^-T L^-1).  Returns 1 if the dataflow path is unavailable for this call (caller falls back).
int chol_dataflow(vzgp_handle* h, double* L, double* Linv, double* LinvT, double* Kinv, int np, int* flag);
int chol_dataflow_prepare(vzgp_handle* h, int np, bool want_kinv);
int chol_dataflow_timed_out(vzgp_handle* h, int* out);

// The trust region of a scoring request (vzgp_acq, vzgp_pe_params, vzgp_pe_multi_params or vzgp_qacq), measured on
// the trials of `trials`: tr_rows clamped to its valid rows, tr_dim_mask expanded over its dimensions.
template <class P>
TrustRegion trust_region_of(const vzgp_handle* trials, const P& p, bool strict) {
  TrustRegion t;
  t.apply = p.use_trust_region ? 1 : 0;
  t.rows = (p.tr_rows > 0 && p.tr_rows < trials->n_valid) ? p.tr_rows : trials->n_valid;
  t.strict = strict ? 1 : 0;
  t.radius = p.trust_radius;
  for (int d = 0; d < kMaxDc; ++d) t.mask[d] = (d < trials->dc) ? (p.tr_dim_mask ? (p.tr_dim_mask[d] ? 1 : 0) : 1) : 0;
  return t;
}
// Whether the region can move a score, so the scoring call must compute the distances.
inline bool tr_needs_distance(const TrustRegion& t) { return t.apply && t.radius <= 0.5; }

// The posterior alone (UCB coefficient 0, no trust region), as the multi-model launchers score their members; `mask`
// and `rows` select the distance such a call reports through `linf`.
inline vzgp_acq posterior_request(const uint8_t* mask = nullptr, int rows = 0) {
  vzgp_acq a;
  a.ucb_coefficient = 0.0; a.use_trust_region = 0; a.trust_radius = 1.0; a.tr_dim_mask = mask;
  a.tr_rows = rows; a.tr_strict = 0;
  return a;
}

// The scoring launchers take the acquisition function as `fn`; nullptr means UCB with acq->ucb_coefficient (the
// per-member scorings inside the ensemble, stack and GP-UCB-PE launchers rely on that).
int launch_score(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_acq* acq,
                 double* score, double* mu, double* sigma, double* linf, const AcqFn* fn = nullptr);
// wgmma integer-split variant of the large-pool scoring kernel (score_i8.cu).
bool score_i8_eligible(const vzgp_handle* h, int M);
int launch_score_i8(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_acq* acq,
                    double* score, double* mu, double* sigma, double* linf, const AcqFn* fn = nullptr);
// CUtensorMap (void*) of a u8 tensor of `rank` <= 3 dims (innermost first), byte strides of dims 1.., 128-byte swizzle.
int make_tensor_map_u8(void* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                       const uint32_t* box, bool promote_256 = true);
int launch_score_pe(vzgp_handle* hA, vzgp_handle* hB, const double* Xs, const int32_t* Zs, int M,
                    const vzgp_pe_params* pe, double* score, double* mu, double* sigma, double* sigma_all);
int launch_score_stack(vzgp_handle* const* hs, int E, const double* alphas, const double* Xs, const int32_t* Zs, int M,
                       const vzgp_acq* acq, double* score, double* mu, double* sigma, double* linf,
                       const AcqFn* fn = nullptr);
int launch_set_pe_combine(vzgp_handle* h, int n_sets, int q, const vzgp_pe_params* pe, const double* cov, int ldc,
                          const double* mu_a, const double* sd_a, const double* linf, double* score, double* sd_all);
// General scoring path (score.cu): explicit K* and W = K* Linv^T of at most kGeneralChunk candidates at a time, in the
// handle's `gen` buffers ([kGeneralChunk x np] each, rows padded to 64; Xp / Zp the padded candidates).
constexpr int kGeneralChunk = 4096;
struct GeneralChunk {
  double* Ks;
  double* W;
  double* Xp;
  int32_t* Zp;
};
int general_chunk_buffers(vzgp_handle* h, GeneralChunk* c);
int launch_general_chunk(vzgp_handle* h, const double* Xs, const int32_t* Zs, int mc, const GeneralChunk& c);
// Parallel (q-) acquisitions (score_q.cu).
int launch_score_qsets(vzgp_handle* const* hs, int E, const double* Xs, const int32_t* Zs, int n_sets, int q,
                       const vzgp_qacq* qa, uint64_t seed, double* score, double* mu, double* sigma, double* linf);
int launch_qacq_mc(vzgp_handle* h, int n_sets, int q, int E, const double* mean, const double* cov, const double* linf,
                   const vzgp_qacq* qa, uint64_t seed, double* score, double* mu, double* sigma);
int prepare_scalarization(vzgp_handle* h, const vzgp_scalarization* sc);
int launch_score_multi(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, double* score, double* mu_out,
                       double* sigma_out);
int prepare_score_pe_multi(vzgp_handle* hA, const vzgp_pe_multi_params* pe);
int launch_score_pe_multi(vzgp_handle* hA, vzgp_handle* hB, const double* Xs, const int32_t* Zs, int M,
                          const vzgp_pe_multi_params* pe, double* score, double* mu, double* sigma, double* sigma_all);
int launch_random_fill(vzgp_handle* h, double* X, int64_t total, int64_t elem_base, uint64_t seed,
                       uint32_t stream, uint32_t iteration);
struct ArgMax {
  double v;
  long long i;
};
int launch_topk_device(vzgp_handle* h, const double* score, int64_t M, int count, long long* d_idx,
                       double* d_val, ArgMax* d_partial, int nblocks);
int launch_gather_rows(vzgp_handle* h, const double* X, int dc, const long long* idx, int count,
                       int64_t M, double* out);

int launch_nll_grad_small(vzgp_handle* h, const double* X, const int32_t* Z, const double* y, int N, int n_valid,
                          const KernelParams& kp, double sn2, double jitter0, int max_iters, double* out);
int launch_score_ensemble(vzgp_handle* const* hs, int E, const double* Xs, const int32_t* Zs, int M,
                          const vzgp_acq* acq, double* score, double* mu, double* sigma, double* linf,
                          const AcqFn* fn = nullptr);
int launch_pack_topk(vzgp_handle* h, const double* X, int dc, const long long* idx, const double* val,
                     int count, int64_t M, int64_t index_base, double* payload);
int launch_merge_topk(vzgp_handle* h, const double* rows, int n_rows, int width, int count, double* out);

// Device-resident eagle optimiser state (pointers into handle->eagle).
struct EagleDev {
  double* pool;         // [P x D]
  double* rewards;      // [P]
  double* pert;         // [P]
  double* best_reward;  // [1]
  int* iter;            // [1]
  double* batch;        // [B x D] candidates of the current step
  double* batch_r;      // [B] their scores
  double* best_x;       // [count x D]
  double* best_r;       // [count]
  long long* best_id;   // [count] evaluation ids (t*B + b), tie-break
  double* tmp_x;
  double* tmp_r;
  long long* tmp_id;
  // categorical features (Dk may be 0)
  int32_t* pool_z;   // [P x Dk]
  int32_t* batch_z;  // [B x Dk]
  int32_t* best_z;   // [count x Dk]
  int32_t* tmp_z;    // [count x Dk]
  int P, B, D, Dk, smax, count;
  int norm_dim;   // feature dimensions of ONE point (Dc + Dk of the model): normalises the force exponent
  int q;          // points per fly (n_parallel); D = q * Dc
  int sizes[kMaxDk];
  vzgp_eagle_config cfg;
  uint64_t seed;
};
// Single-CTA persistent Eagle loop for N <= 64 trials (eagle.cu).
struct SmallModel {
  const double* XTu;     // [dc][64] unscaled trial features, transposed
  const int32_t* Z;      // [64][dk]
  const double* Linv;    // [64][64]
  const double* alpha;   // [64]
  KernelParams kp;
  double sn2;
  int n_valid;
};
struct SmallAcq {
  AcqFn fn;                             // pe_mode < 0: acquisition function of (mean, stddev)
  double coef;                          // GP-UCB-PE mode 0
  double explore, penalty, threshold;   // GP-UCB-PE
  int pe_mode;                          // -1: UCB on one model; 0 / 1: GP-UCB-PE modes (vzgp_pe_params.mode)
  int want_linf;
  TrustRegion tr;
};
bool eagle_persistent_eligible(const vzgp_handle* h, const vzgp_handle* hB, const EagleDev& e);
int launch_eagle_persistent64(vzgp_handle* h, vzgp_handle* hB, const EagleDev& e, const vzgp_acq* acq,
                              const vzgp_pe_params* pe, int steps, const AcqFn* fn = nullptr);
// Multi-CTA persistent Eagle loop (eagle_grid.cu): cooperative launch, batch <= 512 candidates.
bool eagle_grid_eligible(const vzgp_handle* h, const vzgp_handle* hB, const EagleDev& e);
int launch_eagle_grid(vzgp_handle* h, vzgp_handle* hB, const EagleDev& e, const vzgp_acq* acq,
                      const vzgp_pe_params* pe, int steps, const AcqFn* fn = nullptr);
size_t eagle_suggest_smem(const EagleDev& e);
size_t eagle_update_smem(const EagleDev& e);
size_t eagle_suggest_cta_smem(const EagleDev& e);
int launch_eagle_init(vzgp_handle* h, const EagleDev& e);
int launch_eagle_seed_priors(vzgp_handle* h, const EagleDev& e, const double* prior, const int32_t* prior_z,
                             const double* prior_r, int n, int* ord, double* chosen_r);
int launch_random_fill_cat(vzgp_handle* h, int32_t* Z, int64_t M, int dk, const int* sizes, int64_t index_base,
                           uint64_t seed, uint32_t stream);
int launch_gather_rows_i32(vzgp_handle* h, const int32_t* Z, int dk, const long long* idx, int count, int64_t M,
                           int32_t* out);
int eagle_prepare(const EagleDev& e);
int launch_eagle_suggest(vzgp_handle* h, const EagleDev& e);
int launch_eagle_update(vzgp_handle* h, const EagleDev& e);

}  // namespace vzgp
