"""Transfer-learning stacks whose levels follow the designer's model spec, restated on top of oracle/gp_oracle.py
(gp_bandit.py:402-447; gp/gp_models.py:91-140, :226-299; gp/transfer_learning.py:62-152;
stochastic_process_model.py:835-868).

A stack is a list of levels, base first.  A level is a list of E Predictives (the members of a uniform ensemble, all
fitted on the level's trials); a multi-metric level is one Predictive whose alpha is [N, M].  Each level's prediction
is the equal-weight mixture of its members in the two-pass form; the levels combine as in `go.predict_stack`:
mean = sum of the level means, stddev s <- sd_l^alpha_l * s^(1 - alpha_l) bottom-up, alpha_l from the training-set
sizes of levels l and l-1 with Dc + Dk + 2 hyper-parameters."""
import numpy as np

from oracle import gp_oracle as go


def mixture(mus, sds):
  """Two-pass mixture moments: mus / sds [E, B] -> mean, stddev [B];
  var = (1/E) sum sd_e^2 + (1/E) sum (mu_e - mean)^2."""
  mus = np.asarray(mus, np.float64)
  sds = np.asarray(sds, np.float64)
  mean = np.mean(mus, axis=0)
  var = np.mean(sds * sds, axis=0) + np.mean((mus - mean) ** 2, axis=0)
  return mean, np.sqrt(var)


def level_alpha(levels, l):
  """Weight of level l's stddev against the stack below it."""
  p, below = levels[l][0], levels[l - 1][0]
  h = p.x.shape[1] + (0 if p.z is None else p.z.shape[1]) + 2
  return go.transfer_alpha(int(np.sum(p.row_valid)), int(np.sum(below.row_valid)), h)


def predict_level(level, xs, zs=None):
  """Mixture of the level's members: mean [B] (or [B, M] for a multi-metric level) and stddev [B]."""
  mus, sds = zip(*[go.predict(p, xs, zs) for p in level])
  if np.ndim(mus[0]) == 2:                   # multi-metric level: one member, stddev shared by the metrics
    assert len(level) == 1
    return mus[0], sds[0]
  return mixture(np.stack(mus), np.stack(sds))


def predict(levels, xs, zs=None):
  """Combined prediction of the stack: mean [B] or [B, M], stddev [B]."""
  mean, sd = predict_level(levels[0], xs, zs)
  for l in range(1, len(levels)):
    a = level_alpha(levels, l)
    mean_l, sd_l = predict_level(levels[l], xs, zs)
    mean = mean + mean_l
    sd = sd_l ** a * sd ** (1.0 - a)
  return mean, sd


def residual_labels(levels, x, y, z=None):
  """Labels of the next level: y [N] or [N, M] minus the mean of the whole stack built so far (each metric against
  that metric's stack mean)."""
  if not levels:
    return np.asarray(y, np.float64)
  return np.asarray(y, np.float64) - predict(levels, x, z)[0]


def score(levels, xs, zs=None, *, coefficient=1.8, trust_radius_value=None, tr_dim_mask=None):
  """UCB on the combined prediction with the non-strict trust region measured against the TOP level's trials.
  Returns score, mean, stddev and the distance (None without a trust region)."""
  xs = np.asarray(xs, np.float64)
  mean, sd = predict(levels, xs, zs)
  acq = go.ucb(mean, sd, coefficient)
  dist = None
  if trust_radius_value is not None:
    top = levels[-1][0]
    mask = np.ones(xs.shape[-1], bool) if tr_dim_mask is None else tr_dim_mask
    dist = go.min_linf_distance(xs, top.x, mask, top.row_valid)
    acq = go.apply_trust_region(acq, dist, trust_radius_value)
  return acq, mean, sd, dist


def scalarized_score(levels, xs, weights, reference_point, max_scalarized=None, coefficient=1.8, zs=None):
  """Multi-metric stack: u_m = mean_m + c s through the floored HV scalarisation, no trust region."""
  mean, sd = predict(levels, xs, zs)
  return go.scalarized_ucb(mean, sd, weights, reference_point, max_scalarized, coefficient), mean, sd
