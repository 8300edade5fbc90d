// Pointwise acquisition functions of the posterior (mean, stddev) at one candidate: UCB, LCB, EI, PI and the
// thresholded pair of AcquisitionTrustRegion (vizier/_src/algorithms/designers/gp/acquisitions.py:213-274,
// :390-492).  Every scoring epilogue (emit_score, k_general_finalize, k_stack_combine, k_ensemble_combine,
// score_batch64) evaluates acq_value on its final (mean, stddev); the L-inf trust region is applied after it.
#pragma once
#include <cuda_runtime.h>

#include "../../include/vzgp.h"

namespace vzgp {

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

}  // namespace vzgp
