// GP-UCB-PE over uniform ensembles (gp_ucb_pe.py with ensemble_size > 1): models A (completed trials) and B
// (completed + pending trials) are each E members, one per kept ARD restart, and every prediction is their
// equal-weight mixture (MixtureSameFamily, stochastic_process_model.py:835-868):
//   mean = (1/E) sum_e mu_e,   var = (1/E) sum_e sd_e^2 + (1/E) sum_e (mu_e - mean)^2
// in the two-pass (law of total variance) form, members summed in index order.  The one-pass
// avg(sd^2 + mu^2) - mean^2 of k_ensemble_combine cancels badly when sd << |mu| (model B in high-noise mode:
// sd ~ 1e-5 at the trials, |mu| ~ 1), so it is not used here.
// Shared by k_pe_ensemble_combine (score.cu) and the cooperative Eagle loop (eagle_grid.cu).
#pragma once
#include "acq_fn.cuh"
#include "launchers.h"

namespace vzgp {

constexpr int kMaxPeEnsemble = 8;   // members per model (vzgp_score_pe_ensemble)

struct PeEnsCombine {
  int E, mode;
  double ucb, explore, penalty, threshold;
  TrustRegion tr;   // strict, measured on model B's trials
};

inline PeEnsCombine pe_ensemble_args(const vzgp_handle* hB0, int E, const vzgp_pe_params* pe) {
  PeEnsCombine p;
  p.E = E; p.mode = pe->mode; p.ucb = pe->ucb_coefficient; p.explore = pe->explore_coefficient;
  p.penalty = pe->penalty_coefficient; p.threshold = pe->threshold;
  p.tr = trust_region_of(hB0, *pe, true);
  return p;
}

// Mixture moments of the E members at candidate m: mu / sd are [E][ld].
__device__ __forceinline__ void pe_mixture(int E, const double* __restrict__ mu, const double* __restrict__ sd,
                                           size_t ld, int m, double& mean, double& stddev) {
  double s = 0.0;
  for (int e = 0; e < E; ++e) s += mu[(size_t)e * ld + m];
  mean = s / E;
  double v = 0.0, w = 0.0;
  for (int e = 0; e < E; ++e) {
    const double a = sd[(size_t)e * ld + m], d = mu[(size_t)e * ld + m] - mean;
    v = fma(a, a, v);
    w = fma(d, d, w);
  }
  stddev = sqrt(v / E + w / E);
}

// UCB (mode 0): mean_A + c stddev_B;  PE (mode 1): stddev_B + p min(mean_A + e stddev_A - threshold, 0);
// then the strict trust region on the distance to B's trials.
__device__ __forceinline__ double pe_ensemble_score(const PeEnsCombine& p, double mean_a, double sd_a, double sd_b,
                                                    double dist) {
  double acq;
  if (p.mode == 0) {
    acq = fma(p.ucb, sd_b, mean_a);
  } else {
    const double explore_ucb = fma(sd_a, p.explore, mean_a);
    acq = sd_b + p.penalty * fmin(explore_ucb - p.threshold, 0.0);
  }
  return tr_apply(p.tr, acq, dist);
}

}  // namespace vzgp
