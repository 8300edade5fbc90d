"""GP-UCB-PE over uniform ensembles restated on top of oracle/gp_oracle.py (gp_ucb_pe.py:175-217, :344-381, :434-492,
:1018-1021; stochastic_process_model.py:835-868).  Models A and B are lists of E Predictives, member e of both with
the same hyper-parameters; every prediction is the equal-weight mixture of the members."""
import numpy as np

from oracle import gp_oracle as go


def mixture(mus, sds):
  """Two-pass mixture moments of E members: mus / sds [E, B] -> mean, stddev [B].
  var = (1/E) sum sd_e^2 + (1/E) sum (mu_e - mean)^2 (law of total variance)."""
  mus = np.asarray(mus, np.float64)
  sds = np.asarray(sds, np.float64)
  mean = np.mean(mus, axis=0)
  var = np.mean(sds * sds, axis=0) + np.mean((mus - mean) ** 2, axis=0)
  return mean, np.sqrt(var)


def one_pass_mixture(mus, sds):
  """The one-pass form avg(sd^2 + mu^2) - mean^2 (k_ensemble_combine), for comparison only."""
  mus = np.asarray(mus, np.float64)
  sds = np.asarray(sds, np.float64)
  mean = np.mean(mus, axis=0)
  var = np.mean(sds * sds + mus * mus, axis=0) - mean * mean
  return mean, np.sqrt(np.maximum(var, 0.0))


def predict_mixture(preds, xs, zs=None):
  mus, sds = zip(*[go.predict(p, xs, zs) for p in preds])
  return mixture(np.stack(mus), np.stack(sds))


def ucb_threshold(preds_a, preds_b, ucb_coefficient: float = 1.8) -> float:
  """_compute_ucb_threshold on the mixture of A: its mean at the row of B's features with the largest mixture UCB."""
  pb = preds_b[0]
  mu, sd = predict_mixture(preds_a, pb.x, pb.z)
  u = np.where(pb.row_valid, mu + ucb_coefficient * sd, -np.inf)
  return float(mu[int(np.argmax(u))])


def noise_is_high(params, threshold: float) -> bool:
  """snr_e < threshold for ALL members (gp_ucb_pe.py:1018-1021)."""
  return all(p.signal_variance / max(p.observation_noise_variance, 1e-12) < threshold for p in params)


def combine(mean_a, sd_a, sd_b, dist=None, *, mode: int, ucb_coefficient=1.8, explore_coefficient=0.5,
            penalty_coefficient=10.0, threshold=0.0, trust_radius_value=None):
  """UCB (mode 0) / PE (mode 1) of the mixtures, then the strict trust region when `dist` is given."""
  if mode == 0:
    acq = mean_a + ucb_coefficient * sd_b
  else:
    acq = sd_b + penalty_coefficient * np.minimum(mean_a + sd_a * explore_coefficient - threshold, 0.0)
  if dist is not None:
    acq = np.where((dist < trust_radius_value) | (trust_radius_value > 0.5), acq, -1e4 - dist)
  return acq


def ucb_pe_ensemble_score(preds_a, preds_b, xs, zs=None, *, mode: int, ucb_coefficient=1.8, explore_coefficient=0.5,
                          penalty_coefficient=10.0, threshold=0.0, tr_dim_mask=None, tr_rows=None,
                          trust_radius_value=None, use_trust_region=True):
  """Score and aux {'mean', 'stddev', 'stddev_from_all'} (mixtures) with the strict trust region over the first
  tr_rows rows of B (all members of B share their trials)."""
  xs = np.asarray(xs, np.float64)
  mean_a, sd_a = predict_mixture(preds_a, xs, zs)
  _, sd_b = predict_mixture(preds_b, xs, zs)
  dist = None
  if use_trust_region:
    if tr_dim_mask is None:
      tr_dim_mask = np.ones(xs.shape[-1], bool)
    n_tr = preds_b[0].x.shape[0] if tr_rows is None else tr_rows
    dist = go.min_linf_distance(xs, preds_b[0].x[:n_tr], tr_dim_mask)
  acq = combine(mean_a, sd_a, sd_b, dist, mode=mode, ucb_coefficient=ucb_coefficient,
                explore_coefficient=explore_coefficient, penalty_coefficient=penalty_coefficient, threshold=threshold,
                trust_radius_value=trust_radius_value)
  return acq, {'mean': mean_a, 'stddev': sd_a, 'stddev_from_all': sd_b}
