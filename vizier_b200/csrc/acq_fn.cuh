// Pointwise acquisition functions of the posterior (mean, stddev) at one candidate: UCB, LCB, EI, PI and the
// thresholded pair of AcquisitionTrustRegion (vizier/_src/algorithms/designers/gp/acquisitions.py:213-274,
// :390-492), and the L-inf trust region applied after them.  Every pointwise scoring epilogue (emit_score,
// k_general_finalize, k_stack_ensemble_combine, k_ensemble_combine, score_batch64) evaluates acq_value on its final
// (mean, stddev); those and the GP-UCB-PE combines (k_pe_ensemble_combine, k_pe_multi_combine, score_batch64, k_eagle_grid)
// then call tr_apply.  The set scorers (k_set_pe_combine, k_qacq_mc) add tr_set_term per point instead.
// MaxValueEntropySearch (acquisitions.py:293-365) is the main acquisition only, over the handle's max-value samples
// (vzgp_mes_fit / vzgp_set_mes, DESIGN §6k).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/vzgp.h"

namespace vzgp {

constexpr int kMaxDc = 64;     // continuous feature dims supported by the tile kernels
// Set flies of the Eagle optimiser (n_parallel = q > 1): at most kMaxSetPoints points of Dc continuous features,
// q * Dc <= kMaxFlyDim coordinates per fly (k_eagle_suggest_wide walks a fly in 64-column chunks).
constexpr int kMaxSetPoints = 16;
constexpr int kMaxFlyDim = 1024;
constexpr int kMaxMesSamples = 256;   // max-value samples of MaxValueEntropySearch

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
  const double* mes;    // main.kind == VZGP_ACQ_MES: the handle's max-value samples (device) ...
  int mes_k;            // ... and their count
};

// Plain UCB with coefficient c: what every call computes unless the handle was given another acquisition.
inline AcqFn ucb_acq_fn(double c) {
  AcqFn f;
  f.main.kind = VZGP_ACQ_UCB; f.main.coefficient = c; f.main.best_label = 0.0; f.main.exploration = 0.0;
  f.thr = f.main;
  f.use_thr = 0;
  f.threshold = 0.0; f.bad_value = 0.0;
  f.mes = nullptr; f.mes_k = 0;
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

// One max-value sample's MES term t(g) = g r / 2 - log Phi(g), r = phi(g) / Phi(g), and dt/dg = -(r/2)(1 + g^2 + g r),
// at g = (y* - mean) / sd (Wang & Jegelka 2017, eq. 6).  g r / 2 and -log Phi both grow like g^2 / 2 as g -> -inf,
// so c = g + r is formed without cancelling them: directly from erfcx down to g = -12, and below from the
// asymptotic series S = 1 - sqrt(pi) x erfcx(x) = sum_m (-1)^(m+1) (2m-1)!! z^m, x = -g / sqrt 2, z = 1 / g^2, where
// r = |g| / (1 - S), c = |g| S / (1 - S) and 1 + g c = U / (1 - S), U = sum_m (-1)^(m+1) 2m (2m-1)!! z^m.
// tests/mes_oracle.py restates it; tests/test_mes_host.py holds it to mpmath.
constexpr double kMesSeriesG = -12.0;
constexpr int kMesSeriesTerms = 24;

__device__ __forceinline__ void mes_term(double g, double& t, double& dt) {
  if (g >= 0.0) {
    const double ec = erfc(g * 0.7071067811865476);
    const double r = 0.3989422804014327 * exp(-0.5 * g * g) / (1.0 - 0.5 * ec);
    t = 0.5 * g * r - log1p(-0.5 * ec);
    dt = -0.5 * r * (1.0 + g * g + g * r);
  } else if (g >= kMesSeriesG) {
    const double E = erfcx(-g * 0.7071067811865476);
    const double r = 0.7978845608028654 / E, c = g + r;
    t = 0.5 * g * c - log(0.5 * E);
    dt = -0.5 * r * (1.0 + g * c);
  } else {
    const double z = 1.0 / (g * g);
    double s = z, S = 0.0, U = 0.0;
    for (int m = 1; m <= kMesSeriesTerms; ++m) {
      S += s;
      U += (2.0 * m) * s;
      s *= -(2.0 * m + 1.0) * z;
    }
    const double a = -g, r = a / (1.0 - S), c = a * S / (1.0 - S);
    t = 0.5 * g * c - log1p(-S) + (log(a) + 0.9189385332046728);
    dt = -0.5 * r * (U / (1.0 - S));
  }
}

// MES at (mean, sd): the samples' terms summed in index order over K, the same order on every route, so a given
// (mean, sd) scores bit-identically everywhere.  With SLOPES also d/dmean and d/dsd.  sd = 0 (clamped variance) takes
// the limits - a sample above the mean adds 0, one equal to it log 2, one below +inf - and no slope.
template <bool SLOPES>
__device__ __forceinline__ double mes_value(const AcqFn& f, double mean, double sd, double* s_mu = nullptr,
                                            double* s_sd = nullptr) {
  double v = 0.0, a_mu = 0.0, a_sd = 0.0;
  if (sd > 0.0) {
    for (int k = 0; k < f.mes_k; ++k) {
      const double g = (f.mes[k] - mean) / sd;
      double t, dt;
      mes_term(g, t, dt);
      v += t;
      if (SLOPES) { a_mu -= dt / sd; a_sd -= dt * g / sd; }
    }
  } else {
    for (int k = 0; k < f.mes_k; ++k) {
      const double y = f.mes[k];
      v += y > mean ? 0.0 : (y == mean ? 0.6931471805599453 : INFINITY);
    }
  }
  if (SLOPES) { *s_mu = a_mu / f.mes_k; *s_sd = a_sd / f.mes_k; }
  return v / f.mes_k;
}

// mes_value on a group of eight consecutive lanes, for epilogues with idle lanes: lane p of the group evaluates the
// terms of samples k0 + p, eight at a time, and every lane then adds the eight in index order, so the sum is
// mes_value's bit for bit while the costly terms run in parallel.  Every lane of the warp takes part; each group may
// hold its own candidate.
__device__ __forceinline__ double mes_value_8(const AcqFn& f, double mean, double sd, int p) {
  const int base = (threadIdx.x & 31) & ~7;
  double v = 0.0;
  for (int k0 = 0; k0 < f.mes_k; k0 += 8) {
    double t = 0.0;
    if (k0 + p < f.mes_k) {
      const double y = f.mes[k0 + p];
      if (sd > 0.0) {
        double dt;
        mes_term((y - mean) / sd, t, dt);
      } else {
        t = y > mean ? 0.0 : (y == mean ? 0.6931471805599453 : INFINITY);
      }
    }
    const int n = f.mes_k - k0 < 8 ? f.mes_k - k0 : 8;
    for (int j = 0; j < 8; ++j) {
      const double tj = __shfl_sync(0xffffffffu, t, base + j);
      if (j < n) v += tj;
    }
  }
  return v / f.mes_k;
}

// AcquisitionTrustRegion.__call__ (:466-492): where the thresholding value is not >= threshold (NaN included) the
// score is bad_value - thresholding value, otherwise the main acquisition.  MES = false leaves MaxValueEntropySearch
// out, for kernels that never see it (multi-model combines) or have an instance of their own for it.
template <bool MES = true>
__device__ __forceinline__ double acq_value(const AcqFn& f, double mean, double sd) {
  const double v = MES && f.main.kind == VZGP_ACQ_MES ? mes_value<false>(f, mean, sd) : acq_term(f.main, mean, sd);
  if (f.use_thr) {
    const double t = acq_term(f.thr, mean, sd);
    if (!(t >= f.threshold)) return f.bad_value - t;
  }
  return v;
}

// The scoring kernels on the default path are instantiated twice: GENERIC = false evaluates only UCB with the
// main coefficient (the default keeps its register budget), GENERIC = true every acquisition.
template <bool GENERIC, bool MES = true>
__device__ __forceinline__ double acq_eval(const AcqFn& f, double mean, double sd) {
  return GENERIC ? acq_value<MES>(f, mean, sd) : fma(f.main.coefficient, sd, mean);
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
