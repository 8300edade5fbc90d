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
  int32_t* zb = za + dk * LD;
  const int m0 = blockIdx.x * 64;
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  stage_rows_T(Xs, M, dc, m0, 64, sa, LD);
  if (dk > 0) stage_rows_T_i32(Zs, M, dk, m0, 64, za, LD);
  double acc[4][kMaxMetrics];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int m = 0; m < kMaxMetrics; ++m) acc[i][m] = 0.0;
  for (int j0 = 0; j0 < n_valid; j0 += 64) {
    __syncthreads();
    stage_rows_T(X, np, dc, j0, 64, sb, LD);
    if (dk > 0) stage_rows_T_i32(Z, np, dk, j0, 64, zb, LD);
    for (int e = tid; e < n_metrics * 64; e += 256) {
      const int m = e >> 6, c = e & 63;
      sal[m * 64 + c] = (j0 + c < n_valid) ? alpha[(size_t)m * np + j0 + c] : 0.0;
    }
    __syncthreads();
    double d2[4][4], unused[4][4];
    tile_d2<G64, 4, 4, false>(sa, LD, sb, LD, za, LD, zb, LD, kp, nullptr, ty, tx, d2, unused);
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
int prepare_scalarization(vzgp_handle* h, const vzgp_scalarization* sc) {
  VZ_ARG(sc != nullptr, "scalarization");
  const int nm = h->n_metrics, S = sc->n_scalarizations;
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

// mu [n_metrics][M] of the M candidates on the model fitted on `h` (k_mean_multi; not counted in h->launches).
static int launch_mean_multi(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, double* mu) {
  const size_t sm = sizeof(double) * (2 * h->dc * 66 + kMaxMetrics * 64) + sizeof(int32_t) * 2 * h->dk * 66;
  VZ_TRY(raise_dyn_smem((const void*)k_mean_multi, sm));
  k_mean_multi<<<(M + 63) / 64, 256, sm, h->stream>>>(Xs, Zs, M, h->X.as<double>(), h->Z.as<int32_t>(), h->np, h->n_valid,
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

}  // namespace vzgp
