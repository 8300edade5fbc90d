"""Extended-precision posterior for ill-conditioned scoring tests.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE (see oracle/gp_oracle.py).

The fp64 oracle (``gp_oracle.predict``) goes through LAPACK, which loses about as many digits as the
device kernels do when K_y is ill-conditioned (sn2 = 1e-8, short length scales, duplicated trials).  Against
it a kernel that is as accurate as fp64 LAPACK cannot be told apart from one that is 100x worse.  This
module evaluates the same posterior mean and stddev in ``np.longdouble`` (the x87 80-bit format on x86-64: a
64-bit mantissa, 11 more bits than fp64): the kernel, the Cholesky factor and the forward substitutions are
plain vectorised loops, no LAPACK.  Its own error is then far below the fp64 error it is used to measure.
Meant for N up to a few hundred trials (the factor is O(N^3) in software floating point).

``loss_and_grad_ld`` does the same for the ARD loss and its gradient (``gp_oracle.loss_and_grad``), where every
gradient entry is a sum of N^2 terms that cancel by a factor of 10^5-10^6 once K_y is near singular; it also
returns the size of those terms, the unit in which the conditioning tests measure an fp64 evaluation's error.
"""

from __future__ import annotations

import concurrent.futures
import dataclasses
import os
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


_BLOCK = 64


def _blocks(n: int):
  return [(a, min(a + _BLOCK, n)) for a in range(0, n, _BLOCK)]


def _threaded(fn, items):
  """fn over items on a thread pool: NumPy's long-double loops release the GIL, and each item writes its own block."""
  with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as pool:
    list(pool.map(fn, items))


def inverse_ld(l: np.ndarray) -> np.ndarray:
  """K^-1 = L^-T L^-1 in long double.  L^-1 column block [a, b) is zero above row a, so it is a forward solve with
  L[a:, a:]; K^-1 row block [a, b), columns [0, b), only sums over rows k >= a of L^-1.  About a sixth of the
  multiply-adds of the dense forms, which matters where long double has no BLAS."""
  n = l.shape[0]
  linv = np.zeros((n, n), LD)
  kinv = np.zeros((n, n), LD)

  def solve(blk):
    a, b = blk
    linv[a:, a:b] = forward_ld(l[a:, a:], np.eye(n - a, b - a, dtype=LD))

  def gram(blk):
    a, b = blk
    kinv[a:b, :b] = linv[a:, a:b].T @ linv[a:, :b]

  _threaded(solve, _blocks(n))
  _threaded(gram, _blocks(n))
  return np.tril(kinv) + np.tril(kinv, -1).T


@dataclasses.dataclass
class HpLossGrad:
  """loss_and_grad_ld's result, every field in long double.

  loss = data + reg; data = quadratic form + log det + the 2 pi constant, data_scale = the sum of their absolute
  values.  grad [P] in GPParams.to_vector() order; grad_scale[k] = S_k = 0.5 sum_ij |G_ij dK_ij/dtheta_k| (for the
  mean constant coef * sum_i |alpha_i|), the size of the terms whose sum is the data part of grad[k]; grad_reg[k]
  the regulariser's part of grad[k].  alpha [N, M] = K_y^-1 (y - mean), for the fit tests."""
  loss: LD
  data: LD
  data_scale: LD
  reg: LD
  grad: np.ndarray
  grad_scale: np.ndarray
  grad_reg: np.ndarray
  alpha: np.ndarray

  def errors(self, loss, grad=None) -> tuple[float, Optional[np.ndarray]]:
    """(|loss - self.loss| / (data_scale + |reg|), |grad_k - self.grad_k| / (S_k + |reg_k|) per component): the
    error of an fp64 evaluation in units of the terms it sums, the quantity the conditioning tests bound."""
    e_loss = abs(LD(loss) - self.loss) / (self.data_scale + abs(self.reg))
    if grad is None:
      return float(e_loss), None
    e_grad = np.abs(np.asarray(grad, np.float64).astype(LD) - self.grad) / (self.grad_scale + np.abs(self.grad_reg))
    return float(e_loss), e_grad.astype(np.float64)


def _log(v) -> LD:
  return np.log(LD(v))


def loss_and_grad_ld(theta, x, y, z=None, row_valid=None, linear_coef: Optional[float] = None,
                     shift: float = 0.0) -> HpLossGrad:
  """gp_oracle.loss_and_grad in long double: the same to_vector() order, padded-row identity, M metrics (y [N, M]),
  linear kernel and regulariser.  K_y, its factor, L^-1 (a forward solve against I), K_y^-1 = L^-T L^-1,
  G = M K_y^-1 - alpha alpha^T and every gradient sum are formed in np.longdouble from the fp64 inputs.  No jitter
  retry: `shift` is added to the diagonal of the masked K_y (the jitter an fp64 evaluation used), so a problem
  compares the matrix that evaluation factored.  O(N^3) in software floating point: seconds at N = 1000."""
  x = np.asarray(x, np.float64)
  n, dc = x.shape
  y = np.asarray(y, np.float64).reshape(n, -1)
  n_metrics = y.shape[1]
  dk = 0 if z is None else z.shape[1]
  p = go.GPParams.from_vector(theta, dc, dk, linear_coef)
  row_valid = np.ones(n, bool) if row_valid is None else np.asarray(row_valid, bool)
  xl = x.astype(LD)
  ls2 = p.continuous_length_scale_squared.astype(LD)
  lk = p.categorical_length_scale_squared.astype(LD)
  sf2, sn2 = LD(p.signal_variance), LD(p.observation_noise_variance)
  lin = p.linear
  mean = LD(0) if lin is None else LD(lin.coef) * LD(lin.mean_constant)

  sq = [(xl[:, d][:, None] - xl[:, d][None, :]) ** 2 for d in range(dc)]
  neq = [(z[:, k][:, None] != z[:, k][None, :]).astype(LD) for k in range(dk)]
  d2 = np.zeros((n, n), LD)
  for d in range(dc):
    d2 += sq[d] / ls2[d]
  for k in range(dk):
    d2 += neq[k] / lk[k]
  s = np.sqrt(LD(5) * d2)
  es = np.exp(-s)
  kmat = sf2 * (LD(1) + s + s * s / LD(3)) * es
  e = -(LD(5) / LD(6)) * sf2 * (LD(1) + s) * es     # dk / d(d2)
  ky = kmat.copy()
  if lin is not None:
    u = xl / np.sqrt(ls2)[None, :] - LD(lin.coef) * LD(lin.shift)
    lin_a = (LD(lin.coef) * LD(lin.slope_amplitude)) ** 2
    uu = u @ u.T
    ky += lin_a * uu
  ky[np.diag_indices(n)] += sn2
  inv = ~row_valid
  ky[inv, :] = 0
  ky[:, inv] = 0
  ky[inv, inv] = 1
  ky[np.diag_indices(n)] += LD(shift)
  l = cholesky_ld(ky)
  yv = np.where(row_valid[:, None], y.astype(LD) - mean, LD(0))
  w = forward_ld(l, yv)
  alpha = backward_ld(l, w)
  nv = int(np.sum(row_valid))
  quad = np.sum(w * w) / LD(2)
  logdet = n_metrics * np.sum(np.log(np.diag(l)))
  const = LD(n_metrics * nv) * np.log(LD(2) * LD(np.pi)) / LD(2)
  data = quad + logdet + const
  data_scale = quad + n_metrics * np.sum(np.abs(np.log(np.diag(l)))) + const

  kinv = inverse_ld(l)
  g = n_metrics * kinv - alpha @ alpha.T
  vm = np.outer(row_valid, row_valid)
  g = np.where(vm, g, LD(0))
  ge = g * e

  def reg_term(v, centre):
    return go.REG_WEIGHT * _log(v / centre) ** 2, 2 * go.REG_WEIGHT * _log(v / centre) / LD(v)

  grads, scales, regs = [], [], []

  def add(dkdt, reg_grad):
    t = g * dkdt
    grads.append(np.sum(t) / LD(2) + reg_grad)
    scales.append(np.sum(np.abs(t)) / LD(2))
    regs.append(reg_grad)

  reg = LD(0)
  for k in range(dk):
    r, rg = reg_term(lk[k], go.REG_CENTER_LENGTH)
    reg += r
    add(e * (-neq[k] / lk[k] ** 2), rg)
  for d in range(dc):
    r, rg = reg_term(ls2[d], go.REG_CENTER_LENGTH)
    reg += r
    dkdt = e * (-sq[d] / ls2[d] ** 2)
    if lin is not None:
      # dK_lin / d ls2_d = lin_a (x_id u_jd + u_id x_jd) (-ls2_d^-3/2 / 2)
      dkdt = dkdt + lin_a * (np.outer(xl[:, d], u[:, d]) + np.outer(u[:, d], xl[:, d])) * (-ls2[d] ** LD(-1.5) / LD(2))
    add(dkdt, rg)
  if lin is not None:
    coef = LD(lin.coef)
    su = u.sum(axis=1)
    add(-(su[:, None] + su[None, :]) * lin_a * coef, LD(lin.shift))
    r, rg = reg_term(lin.slope_amplitude, go.REG_CENTER_SIGNAL)
    reg += r + (LD(lin.shift) ** 2 + LD(lin.mean_constant) ** 2) / LD(2)
    add(uu * LD(2) * coef ** 2 * LD(lin.slope_amplitude), rg)
    # d/d mean_constant: -coef * sum of alpha over the valid rows and the metrics (no G sum)
    av = alpha[row_valid]
    grads.append(-coef * np.sum(av) + LD(lin.mean_constant))
    scales.append(abs(coef) * np.sum(np.abs(av)))
    regs.append(LD(lin.mean_constant))
  r, rg = reg_term(p.observation_noise_variance, go.REG_CENTER_NOISE)
  reg += r
  add(np.eye(n, dtype=LD), rg)
  r, rg = reg_term(p.signal_variance, go.REG_CENTER_SIGNAL)
  reg += r
  add(kmat / sf2, rg)
  return HpLossGrad(data + reg, data, data_scale, reg, np.array(grads, LD), np.array(scales, LD),
                    np.array(regs, LD), alpha)


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
