"""NumPy oracle of the pointwise acquisition functions (acquisitions.py:213-274, :390-492) on a posterior
(mean, stddev), with the TFP formulas of GaussianProcessExpectedImprovement (exploration 0.01) and
GaussianProcessProbabilityOfImprovement (exploration 0).  With stddev = 0 (a clamped variance) EI is
max(imp, 0) and PI is imp > 0 - the limits as stddev -> 0; the reference evaluates 0/0 there.

`evaluate` interprets the acquisition objects of vizier_b200.acquisitions from their own fields (best labels,
labels, threshold, apply_tr_after) without the host lowering; `score_with_aux` is gp_oracle.score_with_aux with
the acquisition replaced."""
import numpy as np
from scipy.special import ndtr

from oracle import gp_oracle as go

EI_EXPLORATION = 0.01
PI_EXPLORATION = 0.0
_INV_SQRT_2PI = 0.3989422804014327


def ucb(mu, sd, c):
  return mu + c * sd


def lcb(mu, sd, c):
  return mu - c * sd


def ei(mu, sd, best, exploration=EI_EXPLORATION):
  mu, sd = np.asarray(mu, np.float64), np.asarray(sd, np.float64)
  imp = (mu - best) - exploration
  with np.errstate(divide='ignore', invalid='ignore'):
    u = imp / sd
    v = imp * ndtr(u) + sd * (_INV_SQRT_2PI * np.exp(-0.5 * u * u))
  return np.where(sd > 0, v, np.maximum(imp, 0.0))


def pi(mu, sd, best, exploration=PI_EXPLORATION):
  mu, sd = np.asarray(mu, np.float64), np.asarray(sd, np.float64)
  imp = (mu - best) - exploration
  with np.errstate(divide='ignore', invalid='ignore'):
    v = ndtr(imp / sd)
  return np.where(sd > 0, v, (imp > 0).astype(np.float64))


def _best(best_labels) -> float:
  return float(np.asarray(best_labels, np.float64).reshape(-1)[0])


def evaluate(fn, mu, sd):
  """Value of the acquisition object `fn` (UCB / LCB / EI / PI / AcquisitionTrustRegion) at (mu, sd)."""
  name = type(fn).__name__
  if name == 'UCB':
    return ucb(mu, sd, fn.coefficient)
  if name == 'LCB':
    return lcb(mu, sd, fn.coefficient)
  if name == 'EI':
    return ei(mu, sd, _best(fn.best_labels))
  if name == 'PI':
    return pi(mu, sd, _best(fn.best_labels))
  if name == 'AcquisitionTrustRegion':
    t = evaluate(fn.thresholding_acquisition, mu, sd)
    a = evaluate(fn.main_acquisition, mu, sd)
    threshold, apply_tr = -np.inf, False
    if fn.labels is not None:
      labels = np.asarray(fn.labels.padded_array, np.float64)
      with np.errstate(all='ignore'), np.testing.suppress_warnings() as sup:
        sup.filter(RuntimeWarning)
        threshold = np.minimum(np.nanmean(labels), np.nanmedian(labels)) if labels.size else np.nan
      apply_tr = labels.shape[0] <= fn.apply_tr_after
    if fn.threshold is not None:
      threshold = fn.threshold
    cond = np.isnan(threshold) | (t >= threshold) | apply_tr
    return np.where(cond, a, fn.bad_acq_value - t)
  raise NotImplementedError(name)


def evaluate_spec(spec, mu, sd):
  """Value of a lowered gp.AcqFnSpec (kinds 0..3 = UCB, LCB, EI, PI) at (mu, sd)."""
  def term(t):
    return [lambda: ucb(mu, sd, t.coefficient), lambda: lcb(mu, sd, t.coefficient),
            lambda: ei(mu, sd, t.best_label, t.exploration), lambda: pi(mu, sd, t.best_label, t.exploration)][t.kind]()
  v = term(spec.main)
  if spec.thresholding is None:
    return v
  t = term(spec.thresholding)
  return np.where(t >= spec.threshold, v, spec.bad_acq_value - t)


def score_with_aux(pred, xs, zs=None, *, acq_fn, tr_dim_mask=None, categorical_dof: int = 0,
                   use_trust_region: bool = True, radius=None, predict=None):
  """go.score_with_aux with `acq_fn` (an acquisition object) in place of UCB.  `predict(xs, zs) -> (mu, sd)`
  overrides the single-GP posterior (ensembles, stacks); `radius` overrides the trust radius."""
  mu, sd = (predict or (lambda a, b: go.predict(pred, a, b)))(xs, zs)
  acq = evaluate(acq_fn, mu, sd)
  aux = {'mean': mu, 'stddev': sd, 'raw_acquisition': acq}
  if use_trust_region:
    xs = np.asarray(xs, np.float64)
    if tr_dim_mask is None:
      tr_dim_mask = np.ones(xs.shape[-1], bool)
    dist = go.min_linf_distance(xs, pred.x, tr_dim_mask, pred.row_valid)
    if radius is None:
      radius = go.trust_radius(int(np.sum(pred.row_valid)), int(np.sum(tr_dim_mask)), categorical_dof)
    acq = go.apply_trust_region(acq, dist, radius)
    aux.update(linf_distance=dist, radius=np.ones_like(dist) * radius)
  return acq, aux
