// Multi-metric acquisition: hyper-volume scalarised UCB over the independent multi-task GP.
//
// Replaces (reference): the scoring function VizierGPBandit builds for multi-objective problems,
// vizier/_src/algorithms/designers/gp_bandit.py:214-242 -
//   ScalarizeOverAcquisitions(UCB, HyperVolumeScalarization(weights [S, M], reference point),
//                             reduction = mean over the S scalarisations, max with the best observed value)
// (vizier/_src/algorithms/designers/gp/acquisitions.py:571-625, scalarization.py:85-111) evaluated on the
// posterior of tfde.MultiTaskGaussianProcess with tfpke.Independent (tuned_gp_models.py:282-288): the M
// metrics share kernel, hyper-parameters and factor, so sigma is common and only mu_m = K* alpha_m differs.
//
//   k_mean_multi   mu_m(x*) = sum_n k(x*, x_n) alpha_m[n] for every metric, one CTA per 64 candidates,
//                  the kernel row recomputed on the FP64 FMA pipe (N (3D+25) flops per candidate)
//   k_scalarize    u_m = mu_m + c sigma;  score = mean_s max( (min_m max(u_m - ref_m, 0) / w_sm)^M, best_s )
// sigma comes from the single-metric scoring path (k_score / the small-pool kernels).
#include "launchers.h"
#include "tiles.cuh"

namespace vzgp {

using G64 = GemmCfg<64, 64, 16, 4, 4>;

// WIDE (Dk > kMaxDk): the categorical features of both sides are staged kCatTile at a time per trial block (tiles.cuh).
template <bool WIDE>
__global__ void __launch_bounds__(256) k_mean_multi(const double* __restrict__ Xs, const int32_t* __restrict__ Zs,
                                                    int M, const double* __restrict__ X, const int32_t* __restrict__ Z,
                                                    int np, int n_valid, KernelParams kp,
                                                    const double* __restrict__ alpha, int n_metrics,
                                                    double* __restrict__ mu, int mpad) {
  extern __shared__ double smem[];
  constexpr int LD = 66;
  const int dc = kp.dc, dk = kp.dk;
  double* sa = smem;                       // [dc][LD] candidates
  double* sb = sa + dc * LD;               // [dc][LD] trials
  double* sal = sb + dc * LD;              // [n_metrics][64] alpha chunk
  int32_t* za = reinterpret_cast<int32_t*>(sal + kMaxMetrics * 64);
  int32_t* zb = za + (WIDE ? kCatTile : dk) * LD;
  const int m0 = blockIdx.x * 64;
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  stage_rows_T(Xs, M, dc, m0, 64, sa, LD);
  if (!WIDE && dk > 0) stage_rows_T_i32(Zs, M, dk, m0, 64, za, LD);
  double acc[4][kMaxMetrics];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int m = 0; m < kMaxMetrics; ++m) acc[i][m] = 0.0;
  for (int j0 = 0; j0 < n_valid; j0 += 64) {
    __syncthreads();
    stage_rows_T(X, np, dc, j0, 64, sb, LD);
    if (!WIDE && dk > 0) stage_rows_T_i32(Z, np, dk, j0, 64, zb, LD);
    for (int e = tid; e < n_metrics * 64; e += 256) {
      const int m = e >> 6, c = e & 63;
      sal[m * 64 + c] = (j0 + c < n_valid) ? alpha[(size_t)m * np + j0 + c] : 0.0;
    }
    __syncthreads();
    double d2[4][4], unused[4][4];
    tile_d2<G64, 4, 4, false, !WIDE>(sa, LD, sb, LD, za, LD, zb, LD, kp, nullptr, ty, tx, d2, unused);
    if (WIDE)
      for_cat_tiles(Zs, M, m0, 64, Z, np, j0, 64, dk, za, LD, zb, LD, [&](int k0, int kt) {
        tile_hamming<G64, 4, 4>(za, LD, zb, LD, kp.inv_ls2_k_wide + k0, kt, ty, tx, d2);
      });
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int cj = G64::col_of(tx, j);
        const double kv = (j0 + cj < n_valid) ? matern52(d2[i][j], kp.sf2) : 0.0;
#pragma unroll
        for (int m = 0; m < kMaxMetrics; ++m)
          if (m < n_metrics) acc[i][m] = fma(kv, sal[m * 64 + cj], acc[i][m]);
      }
  }
  // combine the 16 threads (tx) that share a candidate row: fixed order, bit-reproducible
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int m = 0; m < kMaxMetrics; ++m) {
      if (m >= n_metrics) continue;
      double v = acc[i][m];
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      const int r = m0 + G64::row_of(ty, i);
      if (tx == 0 && r < M) mu[(size_t)m * mpad + r] = v;
    }
}

// Stages the scalarisation tables of `a` into shared memory: [S][M] inverse weights, then [S] best.
__device__ __forceinline__ void stage_scalarization(const ScalArgs& a, const double* __restrict__ weights_inv,
                                                    const double* __restrict__ best, double* sw) {
  const int nm = a.n_metrics, S = a.n_scal;
  for (int e = threadIdx.x; e < S * nm; e += blockDim.x) sw[e] = weights_inv[e];
  double* sbest = sw + S * nm;
  if (a.has_max) for (int e = threadIdx.x; e < S; e += blockDim.x) sbest[e] = best[e];
}

// mean_s max( (min_m u_m / w_sm) ^ n_metrics, best_s ) for u_m already shifted by the reference point and
// clamped at 0; sw as staged by stage_scalarization.
__device__ __forceinline__ double scalarized_mean(const ScalArgs& a, const double (&u)[kMaxMetrics],
                                                  const double* sw) {
  const int nm = a.n_metrics, S = a.n_scal;
  const double* sbest = sw + S * nm;
  double total = 0.0;
  for (int s = 0; s < S; ++s) {
    double mn = u[0] * sw[s * nm];
#pragma unroll
    for (int m = 1; m < kMaxMetrics; ++m)
      if (m < nm) mn = fmin(mn, u[m] * sw[s * nm + m]);
    double pw = mn;
    for (int m = 1; m < nm; ++m) pw *= mn;            // mn ** n_metrics
    if (a.has_max) pw = fmax(pw, sbest[s]);
    total += pw;
  }
  return total / S;
}

// weights_inv [S][M] = 1 / w_sm, best [S] (max over the observed labels of the scalarisation).
__global__ void __launch_bounds__(256) k_scalarize(int M, ScalArgs a, const double* __restrict__ mu, int mpad,
                                                   const double* __restrict__ sigma,
                                                   const double* __restrict__ weights_inv,
                                                   const double* __restrict__ best, double* __restrict__ score) {
  extern __shared__ double sw[];   // [S][M] inverse weights, then [S] best
  const int nm = a.n_metrics;
  stage_scalarization(a, weights_inv, best, sw);
  __syncthreads();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= M) return;
  double u[kMaxMetrics];
  const double sd = sigma[c];
#pragma unroll
  for (int m = 0; m < kMaxMetrics; ++m)
    u[m] = (m < nm) ? fmax(fma(a.coef, sd, mu[(size_t)m * mpad + c]) - a.ref[m], 0.0) : 0.0;
  score[c] = scalarized_mean(a, u, sw);
}

// Multi-metric GP-UCB-PE (gp_ucb_pe.py:344-381, :434-492, :63-78) on the pieces of models A and B.  sigma is shared
// by the metrics of the independent multi-task GP, so mean_m(stddev_B) is stddev_B itself.
//   mode 0: u_m = mu_A,m + ucb sigma_B, then the floored mean HV scalarisation (as k_scalarize)
//   mode 1: sigma_B + agg_m( penalty min(mu_A,m + explore sigma_A - thr_m, 0) ),  agg = mean / max / min
// followed by the strict trust region of :221-242.
struct PeMultiCombine {
  int mode, agg;
  double explore, penalty;
  double thr[kMaxMetrics];
  TrustRegion tr;
};
__global__ void __launch_bounds__(256) k_pe_multi_combine(int M, PeMultiCombine p, ScalArgs a,
                                                          const double* __restrict__ mu, int mpad,
                                                          const double* __restrict__ sd_a,
                                                          const double* __restrict__ sd_b,
                                                          const double* __restrict__ linf,
                                                          const double* __restrict__ weights_inv,
                                                          const double* __restrict__ best,
                                                          double* __restrict__ score) {
  extern __shared__ double sw[];   // mode 0: the scalarisation tables
  const int nm = a.n_metrics;
  if (p.mode == 0) stage_scalarization(a, weights_inv, best, sw);
  __syncthreads();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= M) return;
  const double sb = sd_b[c];
  double acq;
  if (p.mode == 0) {
    double u[kMaxMetrics];
#pragma unroll
    for (int m = 0; m < kMaxMetrics; ++m)
      u[m] = (m < nm) ? fmax(fma(a.coef, sb, mu[(size_t)m * mpad + c]) - a.ref[m], 0.0) : 0.0;
    acq = scalarized_mean(a, u, sw);
  } else {
    const double sa = sd_a[c];
    double agg = 0.0;
#pragma unroll
    for (int m = 0; m < kMaxMetrics; ++m) {
      if (m >= nm) continue;
      const double pen = p.penalty * fmin(fma(sa, p.explore, mu[(size_t)m * mpad + c]) - p.thr[m], 0.0);
      if (m == 0) agg = pen;
      else if (p.agg == VZGP_REGION_UNION) agg = fmax(agg, pen);
      else if (p.agg == VZGP_REGION_INTERSECTION) agg = fmin(agg, pen);
      else agg += pen;
    }
    if (p.agg == VZGP_REGION_AVERAGE) agg /= nm;
    acq = sb + agg;
  }
  score[c] = tr_apply(p.tr, acq, linf[c]);
}

// Uploads 1 / weights and the best observed scalarised values, keeps the small parameters in the handle.
// Not capturable (synchronises): call once before a loop of launch_score_multi.
int prepare_scalarization(vzgp_handle* h, const vzgp_scalarization* sc, int n_metrics) {
  VZ_ARG(sc != nullptr, "scalarization");
  const int nm = n_metrics > 0 ? n_metrics : h->n_metrics, S = sc->n_scalarizations;
  VZ_ARG(sc->n_metrics == nm, "scalarization.n_metrics must equal the fitted model's number of metrics");
  VZ_ARG(S >= 1 && S <= 4096, "1 <= n_scalarizations <= 4096");
  VZ_ARG(sc->weights != nullptr && sc->reference_point != nullptr, "weights / reference_point");
  const size_t wn = (size_t)S * nm;
  VZ_TRY(h->scal.reserve(sizeof(double) * (wn + S)));
  std::vector<double> host(wn + S, 0.0);
  for (size_t e = 0; e < wn; ++e) host[e] = 1.0 / sc->weights[e];
  if (sc->max_scalarized) for (int s = 0; s < S; ++s) host[wn + s] = sc->max_scalarized[s];
  VZ_CUDA(cudaMemcpyAsync(h->scal.ptr, host.data(), sizeof(double) * (wn + S), cudaMemcpyHostToDevice, h->stream));
  VZ_CUDA(cudaStreamSynchronize(h->stream));   // pageable source going out of scope
  ScalArgs& a = h->scal_args;
  a.n_metrics = nm; a.n_scal = S; a.has_max = sc->max_scalarized ? 1 : 0; a.coef = sc->ucb_coefficient;
  for (int m = 0; m < kMaxMetrics; ++m) a.ref[m] = m < nm ? sc->reference_point[m] : 0.0;
  return 0;
}

// The k_mean_multi form for kp and its dynamic shared memory.
static auto mean_multi_kernel(const KernelParams& kp, size_t* sm) {
  const bool wide = kp.dk > kMaxDk;
  *sm = sizeof(double) * (2 * kp.dc * 66 + kMaxMetrics * 64) + sizeof(int32_t) * 2 * (wide ? kCatTile : kp.dk) * 66;
  return wide ? k_mean_multi<true> : k_mean_multi<false>;
}

// mu [n_metrics][M] of the M candidates on the model fitted on `h` (k_mean_multi; not counted in h->launches).
static int launch_mean_multi(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, double* mu) {
  size_t sm;
  const auto kfn = mean_multi_kernel(h->kp, &sm);
  VZ_TRY(raise_dyn_smem((const void*)kfn, sm));
  kfn<<<(M + 63) / 64, 256, sm, h->stream>>>(Xs, Zs, M, h->X.as<double>(), h->Z.as<int32_t>(), h->np, h->n_valid,
                                                      h->kp, h->alpha.as<double>(), h->n_metrics, mu, M);
  VZ_CHECK_LAUNCH();
  return 0;
}

// Scores M candidates with the scalarisation last prepared on `h`.  mu_out: optional [n_metrics][M]
// (leading dimension M); sigma_out optional [M].  Asynchronous, capturable.
int launch_score_multi(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, double* score, double* mu_out,
                       double* sigma_out) {
  if (M <= 0) return 0;
  const ScalArgs& a = h->scal_args;
  const int nm = h->n_metrics, S = a.n_scal;
  if (a.n_metrics != nm || S < 1) { set_error("multi-metric scoring without a prepared scalarization"); return VZGP_ERR_STATE; }
  const size_t wn = (size_t)S * nm;
  // sigma through the single-metric path (UCB coefficient 0, no trust region: gp_bandit.py:241)
  VZ_TRY(h->pe_tmp.reserve(sizeof(double) * ((size_t)nm + 2) * (size_t)M));
  double* t = h->pe_tmp.as<double>();
  double* mu = mu_out ? mu_out : t;
  double* sd = sigma_out ? sigma_out : t + (size_t)nm * M;
  double* dummy = t + ((size_t)nm + 1) * M;
  const vzgp_acq none = posterior_request();
  VZ_TRY(launch_score(h, Xs, Zs, M, &none, dummy, nullptr, sd, nullptr));
  VZ_TRY(launch_mean_multi(h, Xs, Zs, M, mu));
  const size_t sm2 = sizeof(double) * (wn + S);
  VZ_TRY(raise_dyn_smem((const void*)k_scalarize, sm2));
  k_scalarize<<<(M + 255) / 256, 256, sm2, h->stream>>>(M, a, mu, M, sd, h->scal.as<double>(),
                                                        h->scal.as<double>() + wn, score);
  VZ_CHECK_LAUNCH();
  h->launches += 2;
  return 0;
}

// Stacked residual GPs of independent multi-task levels (transfer learning with several metrics): every level has one
// factor, so its stddev is shared by the metrics, and one alpha per metric.  mean_m = sum_l mu_l,m; the stddevs are
// stacked bottom-up as in k_stack_ensemble_combine, s <- sd_l^alpha_l * s^(1 - alpha_l); then u_m = mean_m + c s and the
// floored HV scalarisation of k_scalarize, without a trust region (gp_bandit.py:242).
// mu: [L][n_metrics][M], sd: [L][M]; mu_out optional [n_metrics][M], sigma_out optional [M].
struct StackMultiCombine {
  int L;
  double alpha[kMaxStackLevels];
};
__global__ void __launch_bounds__(256) k_stack_multi_combine(int M, StackMultiCombine p, ScalArgs a,
                                                             const double* __restrict__ mu,
                                                             const double* __restrict__ sd,
                                                             const double* __restrict__ weights_inv,
                                                             const double* __restrict__ best,
                                                             double* __restrict__ score, double* __restrict__ mu_out,
                                                             double* __restrict__ sigma_out) {
  extern __shared__ double sw[];
  const int nm = a.n_metrics;
  stage_scalarization(a, weights_inv, best, sw);
  __syncthreads();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= M) return;
  const size_t level = (size_t)nm * M;
  double mean[kMaxMetrics];
#pragma unroll
  for (int m = 0; m < kMaxMetrics; ++m) mean[m] = (m < nm) ? mu[(size_t)m * M + c] : 0.0;
  double s = sd[c];
  for (int l = 1; l < p.L; ++l) {
#pragma unroll
    for (int m = 0; m < kMaxMetrics; ++m)
      if (m < nm) mean[m] += mu[l * level + (size_t)m * M + c];
    s = pow(sd[(size_t)l * M + c], p.alpha[l]) * pow(s, 1.0 - p.alpha[l]);
  }
  double u[kMaxMetrics];
#pragma unroll
  for (int m = 0; m < kMaxMetrics; ++m) {
    u[m] = (m < nm) ? fmax(fma(a.coef, s, mean[m]) - a.ref[m], 0.0) : 0.0;
    if (m < nm && mu_out) mu_out[(size_t)m * M + c] = mean[m];
  }
  score[c] = scalarized_mean(a, u, sw);
  if (sigma_out) sigma_out[c] = s;
}

// hs[0 .. L): one multi-metric handle per level, the scalarisation prepared on the top one (prepare_scalarization).
// Per level the stddev (launch_score, UCB-0 request) and the per-metric means (k_mean_multi), then
// k_stack_multi_combine.  The pieces live in the top handle's pe_tmp: [L n_metrics + L + 1][M] = mu | sd | dummy.
// Asynchronous, capturable.
int launch_score_stack_multi(vzgp_handle* const* hs, int L, const double* alphas, const double* Xs, const int32_t* Zs,
                             int M, double* score, double* mu_out, double* sigma_out) {
  if (M <= 0) return 0;
  vzgp_handle* top = hs[L - 1];
  const ScalArgs& a = top->scal_args;
  const int nm = top->n_metrics, S = a.n_scal;
  if (a.n_metrics != nm || S < 1) { set_error("stacked multi-metric scoring without a prepared scalarization"); return VZGP_ERR_STATE; }
  VZ_TRY(top->pe_tmp.reserve(sizeof(double) * ((size_t)L * nm + L + 1) * (size_t)M));
  double* mu = top->pe_tmp.as<double>();
  double* sd = mu + (size_t)L * nm * M;
  double* dummy = sd + (size_t)L * M;
  const vzgp_acq none = posterior_request();
  for (int l = 0; l < L; ++l) {
    VZ_TRY(launch_score(hs[l], Xs, Zs, M, &none, dummy, nullptr, sd + (size_t)l * M, nullptr));
    VZ_TRY(launch_mean_multi(hs[l], Xs, Zs, M, mu + (size_t)l * nm * M));
    hs[l]->launches++;
  }
  StackMultiCombine p;
  p.L = L;
  for (int l = 0; l < kMaxStackLevels; ++l) p.alpha[l] = l < L ? alphas[l] : 0.0;
  const size_t wn = (size_t)S * nm;
  const size_t sm = sizeof(double) * (wn + S);
  VZ_TRY(raise_dyn_smem((const void*)k_stack_multi_combine, sm));
  k_stack_multi_combine<<<(M + 255) / 256, 256, sm, top->stream>>>(M, p, a, mu, sd, top->scal.as<double>(),
                                                                   top->scal.as<double>() + wn, score, mu_out,
                                                                   sigma_out);
  VZ_CHECK_LAUNCH();
  top->launches++;
  return 0;
}

// Multi-metric GP-UCB-PE, mode 0: uploads the scalarisation of `pe` to hA (synchronises, not capturable).  Mode 1
// carries everything it needs in the kernel arguments.  Call once before a loop of launch_score_pe_multi.
int prepare_score_pe_multi(vzgp_handle* hA, const vzgp_pe_multi_params* pe) {
  if (pe->mode == 0) VZ_TRY(prepare_scalarization(hA, pe->scalarization));
  return 0;
}

// sigma_A (launch_score on A) -> mu_A,m (k_mean_multi on A) -> sigma_B and the L-inf distance to the first tr_rows
// trials of B (launch_score on B) -> k_pe_multi_combine.  Optional outputs: mu [n_metrics][M], sigma / sigma_all [M].
// Asynchronous, capturable; the intermediate pieces live in hA->pe_multi_tmp, which none of the launchers called
// here touches.
int launch_score_pe_multi(vzgp_handle* hA, vzgp_handle* hB, const double* Xs, const int32_t* Zs, int M,
                          const vzgp_pe_multi_params* pe, double* score, double* mu, double* sigma, double* sigma_all) {
  if (M <= 0) return 0;
  const int nm = hA->n_metrics;
  ScalArgs a;
  if (pe->mode == 0) {
    a = hA->scal_args;
    if (a.n_metrics != nm || a.n_scal < 1) {
      set_error("multi-metric GP-UCB-PE (mode 0) without a prepared scalarization");
      return VZGP_ERR_STATE;
    }
    a.coef = pe->ucb_coefficient;
  } else {
    a.n_metrics = nm; a.n_scal = 0; a.has_max = 0; a.coef = pe->ucb_coefficient;
  }
  VZ_TRY(hA->pe_multi_tmp.reserve(sizeof(double) * ((size_t)nm + 5) * (size_t)M));
  double* t = hA->pe_multi_tmp.as<double>();
  double* mu_a = mu ? mu : t;
  double* sd_a = sigma ? sigma : t + (size_t)nm * M;
  double* sd_b = sigma_all ? sigma_all : t + ((size_t)nm + 1) * M;
  double* linf_b = t + ((size_t)nm + 2) * M;
  double* dummy_a = t + ((size_t)nm + 3) * M;
  double* dummy_b = t + ((size_t)nm + 4) * M;
  const vzgp_acq none = posterior_request(), accb = posterior_request(pe->tr_dim_mask, pe->tr_rows);
  PeMultiCombine p;
  p.mode = pe->mode; p.agg = pe->region_penalty;
  p.explore = pe->explore_coefficient; p.penalty = pe->penalty_coefficient;
  p.tr = trust_region_of(hB, *pe, true);
  VZ_TRY(launch_score(hA, Xs, Zs, M, &none, dummy_a, nullptr, sd_a, nullptr));
  VZ_TRY(launch_mean_multi(hA, Xs, Zs, M, mu_a));
  VZ_TRY(launch_score(hB, Xs, Zs, M, &accb, dummy_b, nullptr, sd_b, tr_needs_distance(p.tr) ? linf_b : nullptr));
  for (int m = 0; m < kMaxMetrics; ++m) p.thr[m] = (pe->mode == 1 && m < nm) ? pe->thresholds[m] : 0.0;
  const size_t wn = (size_t)a.n_scal * nm;
  const size_t sm = pe->mode == 0 ? sizeof(double) * (wn + a.n_scal) : 0;
  if (sm) VZ_TRY(raise_dyn_smem((const void*)k_pe_multi_combine, sm));
  k_pe_multi_combine<<<(M + 255) / 256, 256, sm, hA->stream>>>(M, p, a, mu_a, M, sd_a, sd_b, linf_b,
                                                               hA->scal.as<double>(), hA->scal.as<double>() + wn, score);
  VZ_CHECK_LAUNCH();
  hA->launches += 2;
  return 0;
}

// ---- separable multi-task GP: Sigma = K_s (x) T + sn2 I with T = Q diag(lambda) Q^T -----------------------------------
// The rotation I (x) Q splits the model into n_tasks single-metric GPs (eigen-tasks) with signal variances
// s^2 lambda_j and labels Y Q[:, j]; every member handle holds one of them.
struct TaskRot {
  double q[kMaxMetrics * kMaxMetrics];   // row-major [t][j], row stride kMaxMetrics
  int m;
};
static TaskRot task_rot(const double* q, int m) {
  TaskRot r;
  for (int e = 0; e < kMaxMetrics * kMaxMetrics; ++e) r.q[e] = q[e];
  r.m = m;
  return r;
}

// Yt[j][n] = sum_t Q[t][j] Y[t][n]  (metric-major [m][N] in and out)
__global__ void __launch_bounds__(256) k_rotate_labels(const double* __restrict__ Y, int N, TaskRot r,
                                                       double* __restrict__ Yt) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  double y[kMaxMetrics];
#pragma unroll
  for (int t = 0; t < kMaxMetrics; ++t) y[t] = t < r.m ? Y[(size_t)t * N + n] : 0.0;
  for (int j = 0; j < r.m; ++j) {
    double v = 0.0;
#pragma unroll
    for (int t = 0; t < kMaxMetrics; ++t) v = fma(r.q[t * kMaxMetrics + j], y[t], v);
    Yt[(size_t)j * N + n] = v;
  }
}

int launch_rotate_labels(vzgp_handle* h, const double* Y, int N, int n_metrics, const double* q, double* Yt) {
  k_rotate_labels<<<(N + 255) / 256, 256, 0, h->stream>>>(Y, N, task_rot(q, n_metrics), Yt);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

// mu_t = sum_j Q[t][j] mu_j,  sigma_t^2 = sum_j Q[t][j]^2 sigma_j^2  (the rows of Q have unit norm, so the noise
// variance each eigen-task adds comes out once per metric), then u_t = mu_t + c sigma_t and the scalarisation of
// k_scalarize.  mu_j / sd_j: [n_tasks][ld]; mu_out / sigma_out optional [n_tasks][M].
__global__ void __launch_bounds__(256) k_separable_combine(int M, TaskRot r, ScalArgs a, const double* __restrict__ mu,
                                                           const double* __restrict__ sd, int ld,
                                                           const double* __restrict__ weights_inv,
                                                           const double* __restrict__ best, double* __restrict__ score,
                                                           double* __restrict__ mu_out, double* __restrict__ sigma_out) {
  extern __shared__ double sw[];
  __shared__ double sq[kMaxMetrics * kMaxMetrics];
  stage_scalarization(a, weights_inv, best, sw);
  for (int e = threadIdx.x; e < kMaxMetrics * kMaxMetrics; e += blockDim.x) sq[e] = r.q[e];
  __syncthreads();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= M) return;
  double mj[kMaxMetrics], vj[kMaxMetrics], u[kMaxMetrics];
#pragma unroll
  for (int j = 0; j < kMaxMetrics; ++j) {
    const double s = j < r.m ? sd[(size_t)j * ld + c] : 0.0;
    mj[j] = j < r.m ? mu[(size_t)j * ld + c] : 0.0;
    vj[j] = s * s;
  }
#pragma unroll
  for (int t = 0; t < kMaxMetrics; ++t) {
    double m = 0.0, v = 0.0;
#pragma unroll
    for (int j = 0; j < kMaxMetrics; ++j) {
      const double qq = sq[t * kMaxMetrics + j];
      m = fma(qq, mj[j], m);
      v = fma(qq * qq, vj[j], v);
    }
    const double s = sqrt(v);
    u[t] = t < r.m ? fmax(fma(a.coef, s, m) - a.ref[t], 0.0) : 0.0;
    if (t < r.m && mu_out) mu_out[(size_t)t * M + c] = m;
    if (t < r.m && sigma_out) sigma_out[(size_t)t * M + c] = s;
  }
  score[c] = scalarized_mean(a, u, sw);
}

// Scores M candidates on the separable model of hs[0 .. n_tasks) with the scalarisation prepared on hs[0]: the
// posterior of every eigen-task (launch_score, UCB-0 request), then k_separable_combine.  Asynchronous, capturable;
// the per-task pieces live in hs[0]->pe_tmp, which launch_score does not touch.
int launch_score_separable(vzgp_handle* const* hs, int n_tasks, const double* Xs, const int32_t* Zs, int M,
                           double* score, double* mu_out, double* sigma_out) {
  if (M <= 0) return 0;
  vzgp_handle* h = hs[0];
  const ScalArgs& a = h->scal_args;
  if (a.n_metrics != n_tasks || a.n_scal < 1) {
    set_error("separable scoring without a prepared scalarization");
    return VZGP_ERR_STATE;
  }
  VZ_TRY(h->pe_tmp.reserve(sizeof(double) * (2 * (size_t)n_tasks + 1) * (size_t)M));
  double* mu = h->pe_tmp.as<double>();
  double* sd = mu + (size_t)n_tasks * M;
  double* dummy = sd + (size_t)n_tasks * M;
  const vzgp_acq none = posterior_request();
  for (int j = 0; j < n_tasks; ++j)
    VZ_TRY(launch_score(hs[j], Xs, Zs, M, &none, dummy, mu + (size_t)j * M, sd + (size_t)j * M, nullptr));
  const size_t wn = (size_t)a.n_scal * n_tasks;
  const size_t sm = sizeof(double) * (wn + a.n_scal);
  VZ_TRY(raise_dyn_smem((const void*)k_separable_combine, sm));
  k_separable_combine<<<(M + 255) / 256, 256, sm, h->stream>>>(M, task_rot(h->sep_q, n_tasks), a, mu, sd, M,
                                                               h->scal.as<double>(), h->scal.as<double>() + wn, score,
                                                               mu_out, sigma_out);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

// gram[j][k] = sum_{n < n_valid} alpha_j[n] ka_k[n]  (one CTA per entry, fixed-order tree: bit-reproducible)
__global__ void __launch_bounds__(256) k_task_gram(const double* __restrict__ alpha, const double* __restrict__ ka,
                                                   int np, int n_valid, double* __restrict__ gram) {
  __shared__ double red[256];
  const int j = blockIdx.x, k = blockIdx.y;
  double v = 0.0;
  for (int n = threadIdx.x; n < n_valid; n += 256) v = fma(alpha[(size_t)j * np + n], ka[(size_t)k * np + n], v);
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) gram[j * gridDim.x + k] = red[0];
}

// The Gram A^T (K A) of the eigen-task alphas (packed [n_tasks][np]) under the kernel kp (unit amplitude for the
// gradient of the task covariance): K A by k_mean_multi with the trials as candidates, then k_task_gram.
int launch_task_gram(vzgp_handle* h, const double* X, const int32_t* Z, int np, int n_valid, const KernelParams& kp,
                     const double* alphas, int n_tasks, double* ka, double* gram) {
  size_t sm;
  const auto kfn = mean_multi_kernel(kp, &sm);
  VZ_TRY(raise_dyn_smem((const void*)kfn, sm));
  kfn<<<(n_valid + 63) / 64, 256, sm, h->stream>>>(X, Z, n_valid, X, Z, np, n_valid, kp, alphas, n_tasks, ka,
                                                            np);
  k_task_gram<<<dim3(n_tasks, n_tasks), 256, 0, h->stream>>>(alphas, ka, np, n_valid, gram);
  VZ_CHECK_LAUNCH();
  h->launches += 2;
  return 0;
}

// Joint posterior over M points x n_tasks metrics, metric-major blocks:
//   cov[t M + a][u M + b] = sum_j Q[t][j] Q[u][j] C_j[a][b],  mean[t][a] = sum_j Q[t][j] mean_j[a]
// from the eigen-task posteriors mean_t [n_tasks][M], cov_t [n_tasks][M][M].
__global__ void __launch_bounds__(256) k_separable_joint(TaskRot r, int M, const double* __restrict__ mean_t,
                                                         const double* __restrict__ cov_t, double* __restrict__ mean,
                                                         double* __restrict__ cov, int ldc) {
  __shared__ double sq[kMaxMetrics * kMaxMetrics];
  for (int e = threadIdx.x; e < kMaxMetrics * kMaxMetrics; e += blockDim.x) sq[e] = r.q[e];
  __syncthreads();
  const int col = blockIdx.x * blockDim.x + threadIdx.x, row = blockIdx.y;
  const int nm = r.m, W = nm * M;
  if (col >= W) return;
  const int t = row / M, a = row % M, u = col / M, b = col % M;
  const double* cj = cov_t + (size_t)a * M + b;
  const size_t plane = (size_t)M * M;
  double v = 0.0;
  for (int j = 0; j < nm; ++j, cj += plane) v = fma(sq[t * kMaxMetrics + j] * sq[u * kMaxMetrics + j], *cj, v);
  cov[(size_t)row * ldc + col] = v;
  if (col == 0) {
    double m = 0.0;
    for (int j = 0; j < nm; ++j) m = fma(sq[t * kMaxMetrics + j], mean_t[(size_t)j * M + a], m);
    mean[(size_t)t * M + a] = m;
  }
}

int launch_separable_joint(vzgp_handle* h, int n_tasks, const double* q, int M, const double* mean_t,
                           const double* cov_t, double* mean, double* cov, int ldc) {
  const int W = n_tasks * M;
  k_separable_joint<<<dim3((W + 255) / 256, W), 256, 0, h->stream>>>(task_rot(q, n_tasks), M, mean_t, cov_t, mean, cov,
                                                                      ldc);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

}  // namespace vzgp
