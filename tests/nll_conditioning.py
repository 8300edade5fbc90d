"""Problems and the error bound shared by the ill-conditioned NLL tests (test_hp_nll_oracle_host.py on the CPU,
test_gpu_nll_conditioning.py on the device).

On a deterministic objective ARD drives the noise variance to its 1e-10 floor while the length scales grow, and K_y
approaches singularity (cond 1e8 - 1e13 here).  Each gradient entry is 0.5 sum_ij G_ij dK_ij/dtheta_k, N^2 terms that
cancel by 10^5-10^6, and an fp64 evaluation loses digits in proportion.  The tests measure an evaluation's error
against the long-double oracle (oracle/hp_oracle.loss_and_grad_ld) in units of its terms, S_k + |reg_k| per component
(data part + |regulariser| for the loss), and hold it to FACTOR times the fp64 oracle's own error in the same units,
plus FLOOR_EPS machine epsilons.
"""
import numpy as np

from oracle import gp_oracle as go
from oracle import hp_oracle as hp

EPS = np.finfo(np.float64).eps
FACTOR = 4.0
FLOOR_EPS = 64.0
SN2_CORNER = (go.NOISE_VARIANCE_BOUNDS[0] + 2 * go.BOUNDARY_EPS, 1e-9, 1e-8)   # 1e-10 + BOUNDARY_EPS, 1e-9, 1e-8
LIN = dict(coef=0.7, slope_amplitude=0.9, shift=0.2, mean_constant=-0.3)


def data(n, dc, dk, n_metrics=1, seed=0):
  """(x [n, dc], y [n] or [n, M], z [n, dk] or None): distinct trials, labels a smooth function of the features with
  no noise, the kind of objective that sends the noise variance to its floor.  The first two categorical features
  take their first value on 90% of the trials and the others keep it on all of them (a wide search space with few
  parameters in play), so most pairs of trials differ in their continuous features only and the categorical length
  scales do not make K_y well conditioned."""
  rng = np.random.default_rng(seed + 1000 * n + 10 * dc + dk)
  x = rng.uniform(size=(n, dc))
  z = rng.choice(3, size=(n, dk), p=[0.9, 0.05, 0.05]).astype(np.int32) if dk else None
  if dk > 2:
    z[:, 2:] = 0
  y = np.sin(3.0 * x.sum(1)) - np.sum((x - 0.4) ** 2, 1)
  if dk:
    y = y + 0.3 * np.cos(z.sum(1))
  if n_metrics > 1:
    y = np.stack([(1.0 + 0.25 * m) * y + 0.1 * m for m in range(n_metrics)], axis=1)
  return x, y, z


def corner_points(dc, dk, count, linear=False, seed=0, ls2_low=1.0):
  """`count` parameter vectors (to_vector order) in the ill-conditioned corner: the noise variance cycles through
  SN2_CORNER, length scales squared log-uniform in [ls2_low, 100], the signal variance in [0.5, 10].  Studies of a
  few dozen trials reach cond(K_y) ~ 1e10 only at the long end, so they take ls2_low = 10."""
  rng = np.random.default_rng(seed + 17 * dc + dk)
  out = []
  for i in range(count):
    ls = np.exp(rng.uniform(np.log(ls2_low), np.log(100.0), size=dc + dk))
    sf2 = float(np.exp(rng.uniform(np.log(0.5), np.log(10.0))))
    lin = [LIN['shift'], LIN['slope_amplitude'], LIN['mean_constant']] if linear else []
    out.append(np.concatenate([ls, lin, [SN2_CORNER[i % 3], sf2]]))
  return out


def fitted_point(x, y, z=None, row_valid=None, maxiter=40):
  """The point the fp64 oracle's L-BFGS-B ARD fit reaches on this data: the noise variance at its floor and the
  gradient small against its terms, where the optimiser reads it."""
  dc, dk = x.shape[1], 0 if z is None else z.shape[1]
  t0 = np.concatenate([np.full(dk + dc, 3.0), [1e-6, 1.0]])
  return go.ard_fit(x, y, z, init_thetas=t0[None, :], maxiter=maxiter, row_valid=row_valid)[0]


def linear_coef(linear):
  return LIN['coef'] if linear else None


def params(theta, dc, dk, linear=False):
  return go.GPParams.from_vector(theta, dc, dk, linear_coef(linear))


def lapack_retries(theta, x, z, row_valid, linear=False):
  po = params(theta, x.shape[1], 0 if z is None else z.shape[1], linear)
  return go.retrying_cholesky(go.kernel_matrix(po, x, z, row_valid))[2]


def summary(errs):
  """errs [points, components] normalised errors -> (max, rms) per component."""
  errs = np.atleast_2d(np.asarray(errs, np.float64))
  return errs.max(axis=0), np.sqrt(np.mean(errs * errs, axis=0))


def within_bound(got, ref, factor=FACTOR, floor_eps=FLOOR_EPS):
  """Per component: max and rms over the points of `got` at most factor times those of `ref` plus floor_eps * eps."""
  (gm, gr), (fm, fr) = summary(got), summary(ref)
  floor = floor_eps * EPS
  return bool(np.all(gm <= factor * fm + floor) and np.all(gr <= factor * fr + floor))


def exercised(ref, level=1e-10):
  """The fp64 oracle's normalised error exceeds `level` somewhere: the case is in the regime it is meant to test."""
  return float(np.max(ref)) > level


def reference(cache, key, theta, x, y, z, row_valid, linear=False):
  """loss_and_grad_ld of one (problem, point), memoised in `cache` under key + the point's bytes."""
  k = key + (np.asarray(theta, np.float64).tobytes(),)
  if k not in cache:
    cache[k] = hp.loss_and_grad_ld(theta, x, y, z, row_valid, linear_coef=linear_coef(linear))
  return cache[k]
