"""Extended-precision posterior for ill-conditioned scoring tests.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE (see oracle/gp_oracle.py).

The fp64 oracle (``gp_oracle.predict``) goes through LAPACK, which loses about as many digits as the
device kernels do when K_y is ill-conditioned (sn2 = 1e-8, short length scales, duplicated trials).  Against
it a kernel that is as accurate as fp64 LAPACK cannot be told apart from one that is 100x worse.  This
module evaluates the same posterior mean and stddev in ``np.longdouble`` (the x87 80-bit format on x86-64: a
64-bit mantissa, 11 more bits than fp64): the kernel, the Cholesky factor and the forward substitutions are
plain vectorised loops, no LAPACK.  Its own error is then far below the fp64 error it is used to measure.
Meant for N up to a few hundred trials (the factor is O(N^3) in software floating point).
"""

from __future__ import annotations

import dataclasses
from typing import Optional

import numpy as np

from oracle import gp_oracle as go

LD = np.longdouble


def has_extended_precision() -> bool:
  """True where np.longdouble has more mantissa bits than fp64 (x86-64 Linux: 64 bits)."""
  return np.finfo(LD).nmant > np.finfo(np.float64).nmant


def kernel_ld(params: go.GPParams, x1, x2, z1=None, z2=None) -> np.ndarray:
  """Matern-5/2 of gp_oracle.kernel in long double (plain Matern models: no linear part, no feature masks)."""
  assert params.linear is None
  x1 = np.asarray(x1, np.float64).astype(LD)
  x2 = np.asarray(x2, np.float64).astype(LD)
  ls2 = np.asarray(params.continuous_length_scale_squared, np.float64).astype(LD)
  d2 = np.zeros((x1.shape[0], x2.shape[0]), LD)
  for d in range(x1.shape[1]):
    diff = x1[:, d][:, None] - x2[:, d][None, :]
    d2 += diff * diff / ls2[d]
  if z1 is not None and np.asarray(z1).shape[1] > 0:
    lk = np.asarray(params.categorical_length_scale_squared, np.float64).astype(LD)
    for k in range(z1.shape[1]):
      d2 += (z1[:, k][:, None] != z2[:, k][None, :]).astype(LD) / lk[k]
  s = np.sqrt(LD(5) * d2)
  return LD(params.signal_variance) * (LD(1) + s + s * s / LD(3)) * np.exp(-s)


def cholesky_ld(a: np.ndarray) -> np.ndarray:
  """Left-looking Cholesky in long double; raises ValueError on a non-positive pivot."""
  a = np.asarray(a, LD)
  n = a.shape[0]
  l = np.zeros((n, n), LD)
  for j in range(n):
    piv = a[j, j] - np.dot(l[j, :j], l[j, :j])
    if not piv > 0:
      raise ValueError(f'cholesky_ld: pivot {j} is {piv}')
    l[j, j] = np.sqrt(piv)
    l[j + 1:, j] = (a[j + 1:, j] - l[j + 1:, :j] @ l[j, :j]) / l[j, j]
  return l


def forward_ld(l: np.ndarray, b: np.ndarray) -> np.ndarray:
  """L^-1 b for lower-triangular L; b [n] or [n, m]."""
  b = np.asarray(b, LD)
  v = np.zeros_like(b)
  for i in range(l.shape[0]):
    v[i] = (b[i] - l[i, :i] @ v[:i]) / l[i, i]
  return v


def backward_ld(l: np.ndarray, b: np.ndarray) -> np.ndarray:
  """L^-T b for lower-triangular L; b [n]."""
  b = np.asarray(b, LD)
  n = l.shape[0]
  v = np.zeros_like(b)
  for i in range(n - 1, -1, -1):
    v[i] = (b[i] - l[i + 1:, i] @ v[i + 1:]) / l[i, i]
  return v


@dataclasses.dataclass
class HpPredictive:
  params: go.GPParams
  x: np.ndarray
  z: Optional[np.ndarray]
  chol: np.ndarray    # long double, lower
  alpha: np.ndarray   # long double
  row_valid: np.ndarray


def precompute_predictive(params: go.GPParams, x, y, z=None, row_valid=None) -> HpPredictive:
  """K_y = K + sn2 I with padded rows replaced by identity, its factor and alpha = K_y^-1 y, in long double.
  No jitter retry: an ill-conditioned test problem must factor as it stands."""
  x = np.asarray(x, np.float64)
  n = x.shape[0]
  row_valid = np.ones(n, bool) if row_valid is None else np.asarray(row_valid, bool)
  ky = kernel_ld(params, x, x, z, z)
  ky[np.diag_indices(n)] += LD(params.observation_noise_variance)
  inv = ~row_valid
  ky[inv, :] = 0
  ky[:, inv] = 0
  ky[inv, inv] = 1
  l = cholesky_ld(ky)
  yv = np.where(row_valid, np.asarray(y, np.float64), 0.0).astype(LD)
  alpha = backward_ld(l, forward_ld(l, yv))
  return HpPredictive(params, x, z, l, alpha, row_valid)


def predict(pred: HpPredictive, xs, zs=None, chunk: int = 2048) -> tuple[np.ndarray, np.ndarray]:
  """Posterior mean and stddev at xs in long double (returned as long double arrays); var clamped at 0 like
  gp_oracle.predict."""
  xs = np.asarray(xs, np.float64)
  mus, sds = [], []
  for c0 in range(0, xs.shape[0], chunk):
    xc = xs[c0:c0 + chunk]
    zc = None if zs is None else np.asarray(zs)[c0:c0 + chunk]
    ks = kernel_ld(pred.params, xc, pred.x, zc, pred.z) * pred.row_valid[None, :]
    mus.append(ks @ pred.alpha)
    v = forward_ld(pred.chol, ks.T)
    var = LD(pred.params.signal_variance) - np.sum(v * v, axis=0) + LD(pred.params.observation_noise_variance)
    sds.append(np.sqrt(np.maximum(var, LD(0))))
  return np.concatenate(mus), np.concatenate(sds)
