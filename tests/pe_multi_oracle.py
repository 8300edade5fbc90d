"""Multi-metric GP-UCB-PE restated on top of oracle/gp_oracle.py (gp_ucb_pe.py:63-78, :175-218, :221-242,
:344-381, :434-492).  Model A is the independent multi-task GP (a Predictive fitted on labels [N, M]: means
[B, M], one stddev [B]), model B the GP on completed + pending trials."""
import numpy as np

from oracle import gp_oracle as go

AVERAGE, UNION, INTERSECTION = 0, 1, 2   # MultimetricPromisingRegionPenaltyType / vzgp_region_penalty


def ucb_thresholds_multi(pred_a, pred_b, ucb_coefficient: float = 1.8) -> np.ndarray:
  """_compute_ucb_threshold, multi-metric branch: per metric, the mean of A at the row of B's features with the
  largest mean_m + ucb_coefficient * stddev (invalid rows excluded)."""
  mu, sd = go.predict(pred_a, pred_b.x, pred_b.z)
  mu = np.asarray(mu, np.float64).reshape(pred_b.x.shape[0], -1)
  u = np.where(np.asarray(pred_b.row_valid, bool)[:, None], mu + ucb_coefficient * np.asarray(sd)[:, None], -np.inf)
  best = np.argmax(u, axis=0)
  return mu[best, np.arange(mu.shape[1])]


def combine(mu, sd, sd_all, *, mode: int, ucb_coefficient=1.8, explore_coefficient=0.5, penalty_coefficient=10.0,
            thresholds=None, region_penalty=AVERAGE, weights=None, reference_point=None, max_scalarized=None,
            dist=None, trust_radius_value=None) -> np.ndarray:
  """The acquisition from the per-candidate pieces: mu [B, M], sd / sd_all / dist [B]."""
  sd = np.asarray(sd, np.float64)
  sd_all = np.asarray(sd_all, np.float64)
  mu = np.asarray(mu, np.float64).reshape(sd.shape[0], -1)
  n_metrics = mu.shape[1]
  if mode == 0:
    # UCBScoreFunction: ScalarizeOverAcquisitions of mean_A + c * stddev_B, floored at the best scalarised label
    acq = go.scalarized_ucb(mu, sd_all, weights, reference_point, max_scalarized, ucb_coefficient)
  else:
    # PEScoreFunction: stddev_from_all has one column per metric (all equal for the independent GP)
    penalty = penalty_coefficient * np.minimum(mu + sd[:, None] * explore_coefficient
                                               - np.asarray(thresholds, np.float64)[None, :], 0.0)
    agg = {AVERAGE: np.mean, UNION: np.max, INTERSECTION: np.min}[region_penalty](penalty, axis=-1)
    acq = np.mean(np.repeat(sd_all[:, None], n_metrics, axis=1), axis=-1) + agg
  if dist is not None:
    acq = np.where((dist < trust_radius_value) | (trust_radius_value > 0.5), acq, -1e4 - dist)
  return acq


def ucb_pe_multi_score(pred_a, pred_b, xs, zs=None, *, mode: int, ucb_coefficient=1.8, explore_coefficient=0.5,
                       penalty_coefficient=10.0, thresholds=None, region_penalty=AVERAGE, weights=None,
                       reference_point=None, max_scalarized=None, tr_dim_mask=None, tr_rows=None,
                       trust_radius_value=None, use_trust_region=True):
  """Score and aux {'mean' [B, M], 'stddev' [B], 'stddev_from_all' [B]} of the multi-metric UCB (mode 0) or PE
  (mode 1) acquisition, with the strict trust region over the first tr_rows rows of B."""
  xs = np.asarray(xs, np.float64)
  mu, sd = go.predict(pred_a, xs, zs)
  mu = np.asarray(mu, np.float64).reshape(xs.shape[0], -1)
  _, sd_all = go.predict(pred_b, xs, zs)
  dist = None
  if use_trust_region:
    if tr_dim_mask is None:
      tr_dim_mask = np.ones(xs.shape[-1], bool)
    n_tr = pred_b.x.shape[0] if tr_rows is None else tr_rows
    dist = go.min_linf_distance(xs, pred_b.x[:n_tr], tr_dim_mask)
  acq = combine(mu, sd, sd_all, mode=mode, ucb_coefficient=ucb_coefficient, explore_coefficient=explore_coefficient,
                penalty_coefficient=penalty_coefficient, thresholds=thresholds, region_penalty=region_penalty,
                weights=weights, reference_point=reference_point, max_scalarized=max_scalarized, dist=dist,
                trust_radius_value=trust_radius_value)
  return acq, {'mean': mu, 'stddev': sd, 'stddev_from_all': sd_all}
