// Pointwise acquisition functions of the posterior (mean, stddev) at one candidate: UCB, LCB, EI, PI and the
// thresholded pair of AcquisitionTrustRegion (vizier/_src/algorithms/designers/gp/acquisitions.py:213-274,
// :390-492), and the L-inf trust region applied after them.  Every pointwise scoring epilogue (emit_score,
// k_general_finalize, k_stack_combine, k_ensemble_combine, score_batch64) evaluates acq_value on its final
// (mean, stddev); those and the GP-UCB-PE combines (k_pe_combine, k_pe_multi_combine, score_batch64, k_eagle_grid)
// then call tr_apply.  The set scorers (k_set_pe_combine, k_qacq_mc) add tr_set_term per point instead.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/vzgp.h"

namespace vzgp {

constexpr int kMaxDc = 64;     // continuous feature dims supported by the tile kernels

struct AcqTerm {
  int kind;             // vzgp_acq_kind
  double coefficient;   // UCB / LCB
  double best_label;    // EI / PI: best observed (warped) label
  double exploration;   // EI / PI: subtracted from the improvement
};

struct AcqFn {
  AcqTerm main;
  AcqTerm thr;          // AcquisitionTrustRegion: the thresholding acquisition
  int use_thr;          // 0: main only (also when the host resolved a NaN threshold or apply_tr_after)
  double threshold, bad_value;
};

// Plain UCB with coefficient c: what every call computes unless the handle was given another acquisition.
inline AcqFn ucb_acq_fn(double c) {
  AcqFn f;
  f.main.kind = VZGP_ACQ_UCB; f.main.coefficient = c; f.main.best_label = 0.0; f.main.exploration = 0.0;
  f.thr = f.main;
  f.use_thr = 0;
  f.threshold = 0.0; f.bad_value = 0.0;
  return f;
}

// The acquisition function of a scoring call: `fn`, or without one UCB with the request's coefficient.
inline AcqFn acq_fn_of(const vzgp_acq* acq, const AcqFn* fn) { return fn ? *fn : ucb_acq_fn(acq->ucb_coefficient); }

inline bool acq_fn_is_ucb(const AcqFn& f) { return f.main.kind == VZGP_ACQ_UCB && !f.use_thr; }

// sd = 0 is reachable only through the clamped variance: EI is then max(imp, 0) and PI the step imp > 0, the
// limits as sd -> 0 (the reference evaluates 0/0 there).
__device__ __forceinline__ double acq_term(const AcqTerm& t, double mean, double sd) {
  if (t.kind == VZGP_ACQ_LCB) return mean - t.coefficient * sd;
  if (t.kind == VZGP_ACQ_EI || t.kind == VZGP_ACQ_PI) {
    const double imp = (mean - t.best_label) - t.exploration;
    if (!(sd > 0.0)) return t.kind == VZGP_ACQ_EI ? fmax(imp, 0.0) : (imp > 0.0 ? 1.0 : 0.0);
    const double u = imp / sd;
    if (t.kind == VZGP_ACQ_PI) return normcdf(u);
    return imp * normcdf(u) + sd * (0.3989422804014327 * exp(-0.5 * u * u));
  }
  return fma(t.coefficient, sd, mean);   // UCB: the same expression as the UCB-only epilogues had
}

// AcquisitionTrustRegion.__call__ (:466-492): where the thresholding value is not >= threshold (NaN included) the
// score is bad_value - thresholding value, otherwise the main acquisition.
__device__ __forceinline__ double acq_value(const AcqFn& f, double mean, double sd) {
  const double v = acq_term(f.main, mean, sd);
  if (f.use_thr) {
    const double t = acq_term(f.thr, mean, sd);
    if (!(t >= f.threshold)) return f.bad_value - t;
  }
  return v;
}

// The scoring kernels on the default path are instantiated twice: GENERIC = false evaluates only UCB with the
// main coefficient (the default keeps its register budget), GENERIC = true every acquisition.
template <bool GENERIC>
__device__ __forceinline__ double acq_eval(const AcqFn& f, double mean, double sd) {
  return GENERIC ? acq_value(f, mean, sd) : fma(f.main.coefficient, sd, mean);
}

// L-inf trust region (acquisitions.py:152-174, :779-820), resolved on the host by trust_region_of (launchers.h).
struct TrustRegion {
  int apply;        // the region modifies the score
  int rows;         // trusted points = first rows rows of the trials
  int strict;       // inside test: dist < radius (gp_ucb_pe.py:221-242) instead of <= (acquisitions.py:160-166)
  double radius;    // > 0.5 disables the region
  uint8_t mask[kMaxDc];   // dimensions that take part in the distance
};

// Pointwise rule: a point outside the region scores -1e4 - dist.
__device__ __forceinline__ double tr_apply(const TrustRegion& t, double score, double dist) {
  if (!t.apply) return score;
  const bool inside = (t.strict ? (dist < t.radius) : (dist <= t.radius)) || (t.radius > 0.5);
  return inside ? score : (-1e4 - dist);
}

// Set rule of _apply_trust_region_to_set (gp_ucb_pe.py:245-269): a set's score gains this term for each of its
// points.  It tests dist > radius, which is not the complement of the strict inside test.
__device__ __forceinline__ double tr_set_term(const TrustRegion& t, double dist) {
  return dist > t.radius ? -1e4 - dist : 0.0;
}

// This lane's share (trials lane, lane + 32, ...) of the L-inf distance from candidate x [dc] to the region's
// trials X [rows x dc]; the caller reduces it over the warp.
__device__ __forceinline__ double tr_lane_distance(const TrustRegion& t, const double* x, const double* X, int dc,
                                                   int lane) {
  double dist = INFINITY;
  for (int n = lane; n < t.rows; n += 32) {
    double mx = 0.0;
    for (int d = 0; d < dc; ++d)
      if (t.mask[d]) mx = fmax(mx, fabs(x[d] - X[(size_t)n * dc + d]));
    dist = fmin(dist, mx);
  }
  return dist;
}

}  // namespace vzgp
