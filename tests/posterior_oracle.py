"""Joint posterior predictive of a fitted GP in fp64, with categorical queries, the linear kernel and several metrics.

`gp_oracle.predictive_covariance` has no categorical queries and no mean; this is the quantity `vzgp_posterior_multi`
(csrc/c_abi.cu) returns: for queries (xs, zs) and the training set (x, z) of `pred`,

  mean = K(xs, x) alpha + mean_const          one row per metric when alpha is [N, n_metrics]
  cov  = K(xs, xs) - V^T V (+ sn2 I)          V = L^-1 K(xs, x)^T

with the padded training rows (row_valid False) masked out of K(xs, x), and K including the feature-scaled linear
part when the parameters carry one.  The designers' `sample()` draws are rebuilt from it by `designer_samples`."""
import numpy as np
import scipy.linalg as sla

from oracle import gp_oracle as go


def joint_posterior(pred: go.Predictive, xs, zs=None, add_noise: bool = True):
  """(mean [M] or [n_metrics, M], cov [M, M]) at xs [M, Dc] (and zs [M, Dk])."""
  xs = np.asarray(xs, np.float64)
  p = pred.params
  ks = go.kernel(p, xs, pred.x, zs, pred.z, pred.cont_dim_valid, pred.cat_dim_valid) * pred.row_valid[None, :]
  mean = ks @ pred.alpha + go.prior_mean(p)
  v = sla.solve_triangular(pred.chol, ks.T, lower=True)
  cov = go.kernel(p, xs, xs, zs, zs, pred.cont_dim_valid, pred.cat_dim_valid) - v.T @ v
  if add_noise:
    cov = cov + p.observation_noise_variance * np.eye(xs.shape[0])
  return (mean.T if mean.ndim == 2 else mean), cov


def to_oracle_params(hp) -> go.GPParams:
  """`gp.GPHyperParams` (what a designer fitted) -> `gp_oracle.GPParams`."""
  lin = None
  if hp.linear_coef:
    lin = go.LinearParams(float(hp.linear_coef), float(hp.linear_slope_amplitude), float(hp.linear_shift),
                          float(hp.mean_constant))
  dk = hp.categorical_length_scale_squared
  return go.GPParams(float(hp.signal_variance), np.array(hp.continuous_length_scale_squared, np.float64),
                     float(hp.observation_noise_variance), np.array(dk, np.float64) if dk.size else None, lin)


def factor(cov: np.ndarray) -> np.ndarray:
  """The factor the designers sample with: `cholesky_retry(cov, jitter=1e-10, max_iters=8)`."""
  l, _, retries = go.retrying_cholesky(cov, 1e-10, 8)
  assert retries <= 8 and np.all(np.isfinite(l))
  return l


def mixture_draws(comps, g: np.random.Generator, num_samples: int) -> np.ndarray:
  """`gp_bandit.mixture_samples` on host moments [(mean [n], cov [n, n])]: the normals first, then one member
  index per sample when there is more than one member."""
  factors = [(mean, factor(cov)) for mean, cov in comps]
  n = factors[0][0].shape[0]
  normals = g.standard_normal((num_samples, n))
  member = g.integers(0, len(factors), size=num_samples) if len(factors) > 1 else np.zeros(num_samples, int)
  return np.stack([factors[e][0] + normals[i] @ factors[e][1].T for i, e in enumerate(member)])
