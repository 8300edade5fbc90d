"""NumPy restatement of `vzgp_score_grad` / `vzgp_score_grad_ensemble`: the acquisition of one GP or of the two-pass
mixture of E GPs, with the trust region, and its analytic gradient in the candidates' continuous features.

Moments come from the oracle's fitted `Predictive` (L, alpha): mu = k.alpha + prior mean, var = kss - |L^-1 k|^2 + sn2,
restated here so that they also take complex inputs (`moments`, used by the complex-step check); on real inputs they
are `gp_oracle.predict` before its clamp.  Gradient rules (DESIGN §6j):
  * d mu / dx_d = sum_n dk_n/dx_d alpha_n,  d var / dx_d = dkss/dx_d - 2 sum_n dk_n/dx_d (K_y^-1 k)_n;
  * Matern-5/2: dk_n/dx_d = -(5/3) sf2 (1 + s_n) e^-s_n (x_d - X_nd) / l_d^2, s_n = sqrt(5 d2_n);
    linear_coef: + a u_nd / l_d, dkss/dx_d = 2 a u_d / l_d, u(x)_d = x_d / l_d - coef shift, a = (coef slope)^2;
  * a clamped variance (var < 0 -> 0) contributes no variance gradient;
  * mixture: var = mean_e var_e + mean_e (mu_e - mean)^2,  d var = mean_e d var_e + (2/E) sum_e (mu_e - mean) d mu_e;
  * the acquisition's selected branch (AcquisitionTrustRegion: main, or bad_value - thresholding);
  * outside the trust region the score is -1e4 - dist and the gradient -d dist / dx: at the nearest trusted trial
    (lowest index on ties) the first masked coordinate attaining the L-inf maximum (lowest index on ties) gets
    -sign(x_d - X_nd), sign(0) = 0.  JAX would split a tie's gradient equally; ties have measure zero on real data.

`variant` injects the deliberate breaks the device tests must tell apart: 'one_pass' (the mixture variance as
mean(var + mu^2) - mean^2, differentiated as such), 'no_dkss' (no dkss/dx for the linear kernel), 'dvar_as_dsd' (d var
used where d sd is needed).
"""
import numpy as np
import scipy.linalg as sla
from scipy.special import ndtr

from oracle import gp_oracle as go

_INV_SQRT_2PI = 0.3989422804014327
UCB, LCB, EI, PI = 0, 1, 2, 3


def _u(params, x):
  lin = params.linear
  return x / np.sqrt(params.continuous_length_scale_squared)[None, :] - lin.coef * lin.shift


def moments(pred: go.Predictive, xs):
  """(mu [M], var [M]) unclamped, complex-safe in xs."""
  p = pred.params
  X = np.asarray(pred.x, np.float64)
  ls2 = p.continuous_length_scale_squared
  d2 = sum((xs[:, d, None] - X[None, :, d]) ** 2 / ls2[d] for d in range(X.shape[1]))
  s = np.sqrt(5.0 * d2)
  k = p.signal_variance * (1.0 + s + s * s / 3.0) * np.exp(-s)
  kss = p.signal_variance
  if p.linear is not None:
    a = (p.linear.coef * p.linear.slope_amplitude) ** 2
    k = k + a * (_u(p, xs) @ _u(p, X).T)
    kss = kss + a * np.sum(_u(p, xs) ** 2, axis=1)
  k = k * pred.row_valid[None, :]
  mu = k @ pred.alpha + go.prior_mean(p)
  w = sla.solve_triangular(pred.chol, k.T, lower=True)
  return mu, kss - np.sum(w * w, axis=0) + p.observation_noise_variance


def moment_grads(pred: go.Predictive, xs, variant: str = ''):
  """(mu, var, dmu [M, Dc], dvar [M, Dc]) at real xs."""
  p = pred.params
  X = np.asarray(pred.x, np.float64)
  ls2 = p.continuous_length_scale_squared
  mu, var = moments(pred, xs)
  diff = xs[:, None, :] - X[None, :, :]                              # [M, N, Dc]
  s = np.sqrt(5.0 * np.sum(diff ** 2 / ls2, axis=-1))
  f = -(5.0 / 3.0) * p.signal_variance * (1.0 + s) * np.exp(-s)       # [M, N]
  dk = f[:, :, None] * diff / ls2
  k = p.signal_variance * (1.0 + s + s * s / 3.0) * np.exp(-s)
  dkss = np.zeros_like(xs)
  if p.linear is not None:
    a = (p.linear.coef * p.linear.slope_amplitude) ** 2
    il = 1.0 / np.sqrt(ls2)
    dk = dk + (a * _u(p, X) * il)[None, :, :]
    k = k + a * (_u(p, xs) @ _u(p, X).T)
    if variant != 'no_dkss':
      dkss = 2.0 * a * _u(p, xs) * il
  valid = pred.row_valid.astype(np.float64)
  dk = dk * valid[None, :, None]
  k = k * valid[None, :]
  w = sla.solve_triangular(pred.chol, k.T, lower=True)
  v = sla.solve_triangular(pred.chol.T, w, lower=False)               # [N, M] = K_y^-1 k
  dmu = np.einsum('mnd,n->md', dk, pred.alpha)
  dvar = dkss - 2.0 * np.einsum('mnd,nm->md', dk, v)
  return mu, var, dmu, dvar


def _term(t, mu, sd):
  """Value and slopes (d/dmu, d/dsd) of one lowered acquisition term (gp.AcqTermSpec); complex-safe for sd > 0."""
  if t.kind == UCB:
    return mu + t.coefficient * sd, 1.0, t.coefficient
  if t.kind == LCB:
    return mu - t.coefficient * sd, 1.0, -t.coefficient
  imp = (mu - t.best_label) - t.exploration
  u = imp / sd
  phi = _INV_SQRT_2PI * np.exp(-0.5 * u * u)
  if t.kind == EI:
    return imp * ndtr(u) + sd * phi, ndtr(u), phi
  return ndtr(u), phi / sd, -u * phi / sd


def acq_value_and_slopes(spec, coefficient, mu, sd):
  """The acquisition of a gp.AcqFnSpec (None: UCB with `coefficient`) and its slopes, elementwise."""
  from vizier_b200 import gp
  if spec is None:
    spec = gp.AcqFnSpec(gp.AcqTermSpec(UCB, coefficient))
  v, smu, ssd = _term(spec.main, mu, sd)
  v, smu, ssd = [np.broadcast_to(np.asarray(a), np.shape(mu)).copy() for a in (v, smu, ssd)]
  if spec.thresholding is not None:
    t, tmu, tsd = _term(spec.thresholding, mu, sd)
    bad = ~(np.real(t) >= spec.threshold)
    v = np.where(bad, spec.bad_acq_value - t, v)
    smu = np.where(bad, -np.broadcast_to(tmu, np.shape(mu)), smu)
    ssd = np.where(bad, -np.broadcast_to(tsd, np.shape(mu)), ssd)
  return v, smu, ssd


def _trust(pred, xs, acq):
  """(dist [M], dist gradient [M, Dc]) of the trust region of `acq` (gp.Acquisition) on pred's trials."""
  X = np.asarray(pred.x, np.float64)
  n_valid = int(np.sum(pred.row_valid))
  rows = acq.tr_rows if 0 < acq.tr_rows < n_valid else n_valid
  mask = np.ones(X.shape[1], bool) if acq.tr_dim_mask is None else np.asarray(acq.tr_dim_mask, bool)
  Xt = X[:rows]
  adiff = np.abs(xs[:, None, :] - Xt[None, :, :]) * mask               # [M, rows, Dc]
  per = adiff.max(axis=-1) if X.shape[1] else np.zeros((xs.shape[0], rows))
  dist = per.min(axis=1)
  grad = np.zeros_like(xs)
  for m in range(xs.shape[0]):
    n = int(np.argmin(per[m]))                                         # first minimiser
    if dist[m] > 0:
      d = int(np.argmax(adiff[m, n] == dist[m]))                       # first coordinate attaining it
      grad[m, d] = np.sign(xs[m, d] - Xt[n, d])
  return dist, grad


def score_and_grad(preds, xs, acq, variant: str = ''):
  """{'score', 'grad', 'mean', 'stddev', 'linf_distance'} of the members `preds` (one Predictive or a list) at xs
  [M, Dc] under `acq` (gp.Acquisition: acq_fn or UCB, trust region)."""
  preds = [preds] if isinstance(preds, go.Predictive) else list(preds)
  xs = np.asarray(xs, np.float64)
  E = len(preds)
  parts = [moment_grads(p, xs, variant) for p in preds]
  mus = np.stack([q[0] for q in parts])
  vars_ = np.stack([q[1] for q in parts])
  dmus = np.stack([q[2] for q in parts])
  dvars = np.stack([q[3] for q in parts])
  clamped = vars_ < 0
  vars_ = np.where(clamped, 0.0, vars_)
  dvars = np.where(clamped[:, :, None], 0.0, dvars)
  mean = mus.mean(0)
  dmean = dmus.mean(0)
  if variant == 'one_pass' and E > 1:
    var = np.maximum((vars_ + mus ** 2).mean(0) - mean ** 2, 0.0)
    dvar = dvars.mean(0) + 2.0 * (mus[:, :, None] * dmus).mean(0) - 2.0 * mean[:, None] * dmean
  else:
    var = vars_.mean(0) + ((mus - mean) ** 2).mean(0)
    dvar = dvars.mean(0) + (2.0 / E) * np.einsum('em,emd->md', mus - mean, dmus)
  sd = np.sqrt(var)
  value, smu, ssd = acq_value_and_slopes(acq.acq_fn, acq.ucb_coefficient, mean, sd)
  with np.errstate(divide='ignore', invalid='ignore'):
    dsd = dvar if variant == 'dvar_as_dsd' else np.where(sd[:, None] > 0, dvar / (2.0 * sd[:, None]), 0.0)
  grad = smu[:, None] * dmean + np.where(sd[:, None] > 0, ssd[:, None] * dsd, 0.0)
  dist = np.full(xs.shape[0], np.inf)
  if acq.use_trust_region and acq.trust_radius <= 0.5:
    dist, ddist = _trust(preds[0], xs, acq)
    inside = (dist < acq.trust_radius) if acq.tr_strict else (dist <= acq.trust_radius)
    value = np.where(inside, value, -1e4 - dist)
    grad = np.where(inside[:, None], grad, -ddist)
  return {'score': value, 'grad': grad, 'mean': mean, 'stddev': sd, 'linf_distance': dist}


def value_fn(preds, acq):
  """Complex-safe value of `score_and_grad` on the smooth branch the real point takes (no clamp, inside the region or
  without one): for the complex-step check."""
  preds = [preds] if isinstance(preds, go.Predictive) else list(preds)

  def f(xs):
    mv = [moments(p, xs) for p in preds]
    mus = np.stack([a for a, _ in mv])
    vs = np.stack([b for _, b in mv])
    mean = mus.mean(0)
    var = vs.mean(0) + ((mus - mean) ** 2).mean(0)
    return acq_value_and_slopes(acq.acq_fn, acq.ucb_coefficient, mean, np.sqrt(var))[0]
  return f


# -- fixtures shared by the host and device tests -------------------------------------------------------------------
def make_model(rng, n, dc, *, linear: bool = False, seed_params: int = 0, noise: float = 1e-3, n_valid=None):
  """(x [n, dc], y [n], oracle GPParams) of a smooth random problem; `seed_params` varies the hyper-parameters so that
  ensemble members differ."""
  x = rng.uniform(size=(n, dc))
  y = np.sin(3.0 * x @ np.linspace(1.0, 0.3, dc)) + 0.1 * rng.standard_normal(n)
  prng = np.random.default_rng(1000 + seed_params)
  ls2 = np.exp(prng.uniform(np.log(0.3), np.log(3.0), dc)) * max(1.0, dc / 4.0)
  lin = go.LinearParams(0.1, slope_amplitude=float(prng.uniform(0.5, 2.0)), shift=float(prng.normal()),
                        mean_constant=float(prng.normal())) if linear else None
  params = go.GPParams(float(prng.uniform(0.5, 2.0)), ls2, noise, linear=lin)
  return x, y, params


def predictive(x, y, params, n_valid=None):
  row_valid = None if n_valid is None else np.arange(x.shape[0]) < n_valid
  return go.precompute_predictive(params, x, y, row_valid=row_valid)


def device_params(params):
  """gp.GPHyperParams of an oracle GPParams (continuous features)."""
  from vizier_b200 import gp
  lin = params.linear
  v = np.concatenate([params.continuous_length_scale_squared,
                      [] if lin is None else [lin.shift, lin.slope_amplitude, lin.mean_constant],
                      [params.observation_noise_variance, params.signal_variance]])
  return gp.GPHyperParams.from_vector(v, params.continuous_length_scale_squared.shape[0], 0,
                                      None if lin is None else lin.coef)


def acquisitions(best_label: float):
  """name -> gp.AcqFnSpec (None: UCB 1.8) of every lowered acquisition."""
  from vizier_b200 import gp
  T = gp.AcqTermSpec
  return {
      'ucb': None,
      'lcb': gp.AcqFnSpec(T(LCB, 1.8)),
      'ei': gp.AcqFnSpec(T(EI, best_label=best_label, exploration=0.01)),
      'pi': gp.AcqFnSpec(T(PI, best_label=best_label, exploration=0.0)),
      # AcquisitionTrustRegion.default_ucb_pi: UCB where PI >= 0.3, else -1e4 - PI
      'atr_ucb_pi': gp.AcqFnSpec(T(UCB, 1.8), thresholding=T(PI, best_label=best_label), threshold=0.3,
                                 bad_acq_value=-1e4),
      # default_ucb_lcb with its label threshold
      'atr_ucb_lcb': gp.AcqFnSpec(T(UCB, 1.8), thresholding=T(LCB, 1.8), threshold=0.0, bad_acq_value=-1e4),
  }
