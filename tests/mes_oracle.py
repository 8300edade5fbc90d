"""NumPy restatement of MaxValueEntropySearch as libvzgp evaluates it (vzgp_mes_fit, the MES branch of every scoring
epilogue, and its slopes in k_grad_combine).  DESIGN §6k states the contract; this module is its executable form.

Max values (Wang & Jegelka, ICML 2017, §3.1, and the authors' Gumbel-sampling code): with mu_i, sd_i the posterior
predictive at the N valid trials (sd^2 includes the observation noise, as in every scoring call),
  P(y) = prod_i Phi((y - mu_i) / sd_i)           (sd_i = 0: the step y > mu_i)
  left = best observed label, floor = left + 5 sqrt(sn2)
  P(left) >= 0.25: every sample is `floor`; otherwise the quantiles r_q (q = .25, .5, .75) by bisection on
  [left, left + w] (w doubled from max(mu + 5 sd) - left, or 1, until P(left + w) >= .75; FIT_ITERS halvings), the
  Gumbel fit b = (r_.75 - r_.25) / (log(-log .25) - log(-log .75)), a = r_.5 - b log(-log .5), and
  y*_k = max(a - b log(-log u_k), floor) with u_k = philox_uniform(seed, STREAM_MES, 0, k).

MES value: MES(mu, sd) = (1/K) sum_k t(gamma_k), gamma_k = (y*_k - mu) / sd, t(g) = g r(g) / 2 - log Phi(g), r = phi/Phi,
summed in k order.  Each branch avoids the cancellations of the textbook form:
  g >= 0:            log Phi = log1p(-erfc(g/sqrt2)/2), r = phi(g) / (1 - erfc(g/sqrt2)/2);
  SERIES_G <= g < 0: E = erfcx(-g/sqrt2), r = sqrt(2/pi)/E, c = g + r, t = g c / 2 - log(E/2);
  g < SERIES_G:      S = 1 - sqrt(pi) x erfcx(x) (x = -g/sqrt2) by its asymptotic series in z = 1/g^2,
                     S = sum_m (-1)^(m+1) (2m-1)!! z^m, r = |g|/(1-S), c = g + r = |g| S/(1-S),
                     t = g c / 2 - log1p(-S) + log(sqrt(2 pi) |g|).
(g r/2 and -log Phi both grow like g^2/2 as g -> -inf and cancel; c is formed without that cancellation.)
dt/dg = -(r/2)(1 + g^2 + g r) = -(r/2)(1 + g c); on the series branch 1 + g c = U/(1-S) with
U = sum_m (-1)^(m+1) 2m (2m-1)!! z^m.  d gamma/d mu = -1/sd, d gamma/d sd = -gamma/sd.
sd = 0 (clamped variance): y* > mu contributes 0, y* = mu log 2, y* < mu +inf; no gradient.
"""
import math

import numpy as np
from scipy.special import erfc, erfcx

from oracle import eagle_oracle as eo
from oracle import gp_oracle as go

STREAM_MES = 14            # next to kStreamQacqMember = 13 (csrc/eagle_dev.cuh)
FIT_ITERS = 64             # bisection halvings per quantile
BRACKET_DOUBLINGS = 128    # at most this many doublings of the bracket
SERIES_G = -12.0           # gamma below this takes the asymptotic series
SERIES_TERMS = 24
MAX_SAMPLES = 256
DEFAULT_SAMPLES = 100      # acquisitions.py:328-338: num_max_value_samples=100
DEFAULT_SEED = 123         # seed=jax.random.PRNGKey(123)

_SQRT2 = math.sqrt(2.0)
_INV_SQRT_2PI = 0.3989422804014327
_SQRT_2_OVER_PI = 0.7978845608028654
_LOG_SQRT_2PI = 0.9189385332046728
_LOGLOG = {q: math.log(-math.log(q)) for q in (0.25, 0.5, 0.75)}


def log_ndtr(z):
  """log Phi(z) without log(ndtr(z)) (which is -inf below z ~ -38); z = +-inf allowed."""
  z = np.asarray(z, np.float64)
  out = np.empty_like(z)
  neg = z < 0
  with np.errstate(over='ignore', divide='ignore', invalid='ignore'):
    zn = z[neg]
    out[neg] = np.log(0.5 * erfcx(-zn / _SQRT2)) - 0.5 * zn * zn
    out[~neg] = np.log1p(-0.5 * erfc(z[~neg] / _SQRT2))
  out[z == -np.inf] = -np.inf
  return out


def _series(g):
  """(S, U) of the asymptotic branch at g < SERIES_G, summed from the leading term."""
  z = 1.0 / (g * g)
  s = z.copy()
  S = np.zeros_like(g)
  U = np.zeros_like(g)
  for m in range(1, SERIES_TERMS + 1):
    S = S + s
    U = U + (2.0 * m) * s
    s = s * (-(2.0 * m + 1.0) * z)
  return S, U


def terms(g):
  """(t(g), dt/dg) elementwise for finite g."""
  g = np.asarray(g, np.float64)
  t = np.empty_like(g)
  d = np.empty_like(g)
  pos = g >= 0
  mid = (g < 0) & (g >= SERIES_G)
  low = g < SERIES_G
  with np.errstate(under='ignore'):
    gp = g[pos]
    ec = erfc(gp / _SQRT2)
    r = _INV_SQRT_2PI * np.exp(-0.5 * gp * gp) / (1.0 - 0.5 * ec)
    t[pos] = 0.5 * gp * r - np.log1p(-0.5 * ec)
    d[pos] = -0.5 * r * (1.0 + gp * gp + gp * r)
  gm = g[mid]
  E = erfcx(-gm / _SQRT2)
  r = _SQRT_2_OVER_PI / E
  c = gm + r
  t[mid] = 0.5 * gm * c - np.log(0.5 * E)
  d[mid] = -0.5 * r * (1.0 + gm * c)
  gl = g[low]
  S, U = _series(gl)
  a = -gl
  r = a / (1.0 - S)
  c = a * S / (1.0 - S)
  t[low] = 0.5 * gl * c - np.log1p(-S) + (np.log(a) + _LOG_SQRT_2PI)
  d[low] = -0.5 * r * (U / (1.0 - S))
  return t, d


def value_and_slopes(ys, mu, sd):
  """(MES, dMES/dmu, dMES/dsd) at posterior moments mu, sd [M] with max values ys [K]; k summed in order."""
  ys = np.asarray(ys, np.float64).reshape(-1)
  mu = np.asarray(mu, np.float64)
  sd = np.asarray(sd, np.float64)
  pos = sd > 0
  sds = np.where(pos, sd, 1.0)
  v = np.zeros_like(mu)
  s_mu = np.zeros_like(mu)
  s_sd = np.zeros_like(mu)
  for y in ys:
    g = (y - mu) / sds
    t, dt = terms(np.where(pos, g, 0.0))
    lim = np.where(y > mu, 0.0, np.where(y == mu, math.log(2.0), np.inf))
    v = v + np.where(pos, t, lim)
    s_mu = s_mu + np.where(pos, -dt / sds, 0.0)
    s_sd = s_sd + np.where(pos, -dt * g / sds, 0.0)
  K = ys.shape[0]
  return v / K, s_mu / K, s_sd / K


def value(ys, mu, sd):
  return value_and_slopes(ys, mu, sd)[0]


# -- the max-value fit ------------------------------------------------------------------------------------------------
def log_p(y, mu, sd):
  """log P(y* < y) = sum_i log Phi((y - mu_i) / sd_i), sd_i = 0 as the step y > mu_i."""
  pos = sd > 0
  z = np.where(pos, (y - mu) / np.where(pos, sd, 1.0), np.where(y > mu, np.inf, -np.inf))
  return float(np.sum(log_ndtr(z)))


def fit(mu, sd, best_label, sn2, num_samples=DEFAULT_SAMPLES, seed=DEFAULT_SEED):
  """{'samples' [K], 'degenerate', 'a', 'b', 'r' (quantiles .25/.5/.75), 'floor'} of the trials' moments mu, sd."""
  mu = np.asarray(mu, np.float64)
  sd = np.asarray(sd, np.float64)
  left = float(best_label)
  floor = left + 5.0 * math.sqrt(sn2)
  out = {'floor': floor, 'degenerate': False, 'a': np.nan, 'b': np.nan, 'r': None}
  if log_p(left, mu, sd) >= math.log(0.25):
    out['degenerate'] = True
    out['samples'] = np.full(num_samples, floor)
    return out
  w = float(np.max(mu + 5.0 * sd)) - left
  if not w > 0:
    w = 1.0
  for _ in range(BRACKET_DOUBLINGS):
    if log_p(left + w, mu, sd) >= math.log(0.75):
      break
    w *= 2.0
  r = {}
  for q in (0.25, 0.5, 0.75):
    lo, hi, lq = left, left + w, math.log(q)
    for _ in range(FIT_ITERS):
      m = 0.5 * (lo + hi)
      if log_p(m, mu, sd) < lq:
        lo = m
      else:
        hi = m
    r[q] = 0.5 * (lo + hi)
  b = (r[0.75] - r[0.25]) / (_LOGLOG[0.25] - _LOGLOG[0.75])
  a = r[0.5] - b * _LOGLOG[0.5]
  u = eo.philox_uniform(seed, STREAM_MES, 0, num_samples)
  out.update(a=a, b=b, r=r, samples=np.fmax(a - b * np.log(-np.log(u)), floor))
  return out


def trial_moments(pred: go.Predictive):
  """(mu, sd) at the valid trials, as the scoring calls compute them."""
  valid = np.asarray(pred.row_valid, bool)
  return go.predict(pred, np.asarray(pred.x)[valid])


def fit_predictive(pred: go.Predictive, best_label, num_samples=DEFAULT_SAMPLES, seed=DEFAULT_SEED):
  mu, sd = trial_moments(pred)
  return fit(mu, sd, best_label, pred.params.observation_noise_variance, num_samples, seed)


def score_with_aux(pred: go.Predictive, xs, ys, *, use_trust_region=True, radius=None, tr_dim_mask=None,
                   moments=None):
  """(score, aux) of BayesianScoringFunction-style scoring with MES and the trust region; `moments` = (mu, sd)
  replaces the oracle's posterior (to score the device's own moments)."""
  xs = np.asarray(xs, np.float64)
  mu, sd = moments if moments is not None else go.predict(pred, xs)
  raw = value(ys, mu, sd)
  aux = {'mean': mu, 'stddev': sd, 'raw_acquisition': raw}
  acq = raw
  if use_trust_region:
    if tr_dim_mask is None:
      tr_dim_mask = np.ones(xs.shape[-1], bool)
    dist = go.min_linf_distance(xs, pred.x, tr_dim_mask, pred.row_valid)
    if radius is None:
      radius = go.trust_radius(int(np.sum(pred.row_valid)), int(np.sum(tr_dim_mask)), 0)
    acq = go.apply_trust_region(raw, dist, radius)
    aux.update(linf_distance=dist, radius=np.ones_like(dist) * radius)
  return acq, aux


def score_and_grad(pred: go.Predictive, xs, acq, ys, slopes_at=None):
  """{'score', 'grad', 'mean', 'stddev', 'linf_distance'} of vzgp_score_grad with MES under `acq` (gp.Acquisition:
  the trust region), from lbfgsb_oracle's moment gradients; `slopes_at` = (mu, sd) takes the MES slopes there."""
  import lbfgsb_oracle as lo
  xs = np.asarray(xs, np.float64)
  mu, var, dmu, dvar = lo.moment_grads(pred, xs)
  clamped = var < 0
  var = np.where(clamped, 0.0, var)
  dvar = np.where(clamped[:, None], 0.0, dvar)
  sd = np.sqrt(var)
  v, s_mu, s_sd = value_and_slopes(ys, mu, sd)
  if slopes_at is not None:
    _, s_mu, s_sd = value_and_slopes(ys, *slopes_at)
  with np.errstate(divide='ignore', invalid='ignore'):
    dsd = np.where(sd[:, None] > 0, dvar / (2.0 * sd[:, None]), 0.0)
  grad = s_mu[:, None] * dmu + s_sd[:, None] * dsd
  dist = np.full(xs.shape[0], np.inf)
  if acq.use_trust_region and acq.trust_radius <= 0.5:
    dist, ddist = lo._trust(pred, xs, acq)
    inside = (dist < acq.trust_radius) if acq.tr_strict else (dist <= acq.trust_radius)
    v = np.where(inside, v, -1e4 - dist)
    grad = np.where(inside[:, None], grad, -ddist)
  return {'score': v, 'grad': grad, 'mean': mu, 'stddev': sd, 'linf_distance': dist}
