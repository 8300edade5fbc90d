"""NumPy restatement of the reference's OptaxTrain ARD (optax_wrappers.py:36-150; optimizers/core.py:103-130) with
optax.adam, for the tests of vizier_b200.ard.OptaxTrain and of the fused kernel (csrc/ard_adam.cu).

Per-parameter bijector: SoftClip(low, high, hinge_softness=c), c = 1e-2, with the bounds of the model
(tuned_gp_models.py:83-95, :150-270: already widened by _boundary_epsilon = 1e-12 in gp.param_bounds):

    y = high - sp(high - low - sp(u - low)),   sp(v) = c log(1 + exp(v / c))
    dy/du = sigmoid(w / c) sigmoid((u - low) / c),   w = high - low - sp(u - low)
    u = low + sp^-1(high - low - sp^-1(high - y)),   sp^-1(s) = c log(expm1(s / c))

Parameters without a finite bound (linear_shift, mean_fn; tuned_gp_models.py:230-245) use the identity.

Adam (optax scale_by_adam, then scale by -lr), count t = 1, 2, ...:

    mu <- b1 mu + (1 - b1) g,   nu <- b2 nu + (1 - b2) g^2
    u  <- u - lr (mu / (1 - b1^t)) / (sqrt(nu / (1 - b2^t) + eps_root) + eps),   g = d loss(SoftClip(u)) / du

Loop: every epoch evaluates once and then updates.  The final losses are those of the LAST evaluation (before the
last update); the parameters returned are those AFTER the last update; best_n is a stable argsort of the final losses.
A restart whose loss or gradient is not finite (the retrying Cholesky exhausted) stops: NaN losses from that epoch on,
its parameters those of that evaluation, and it sorts last.

UNVERIFIED: the TFP SoftClip composition and optax's Adam update above are restated from memory; neither library is
part of the reference tree, so neither can be checked against its source here (like the [T] items of SURVEY
Appendix A).  This file is written independently of vizier_b200/ard.py: softplus through np.logaddexp, bias
corrections through powers b^t, one restart at a time.
"""
from __future__ import annotations

import math

import numpy as np

HINGE = 1e-2


def softplus(v):
  return HINGE * np.logaddexp(0.0, np.asarray(v, np.float64) / HINGE)


def softplus_inv(s):
  s = np.asarray(s, np.float64)
  return s + HINGE * np.log(-np.expm1(-s / HINGE))


def sigmoid(z):
  return 0.5 * (1.0 + np.tanh(0.5 * np.asarray(z, np.float64)))


def _box(lo, hi):
  return np.isfinite(lo) & np.isfinite(hi)


def soft_clip(u, lo, hi):
  u = np.asarray(u, np.float64)
  box = _box(lo, hi)
  lo_b, hi_b = np.where(box, lo, 0.0), np.where(box, hi, 1.0)
  y = hi_b - softplus(hi_b - lo_b - softplus(u - lo_b))
  return np.where(box, y, u)


def soft_clip_grad(u, lo, hi):
  u = np.asarray(u, np.float64)
  box = _box(lo, hi)
  lo_b, hi_b = np.where(box, lo, 0.0), np.where(box, hi, 1.0)
  w = hi_b - lo_b - softplus(u - lo_b)
  return np.where(box, sigmoid(w / HINGE) * sigmoid((u - lo_b) / HINGE), 1.0)


def soft_clip_inverse(y, lo, hi):
  y = np.asarray(y, np.float64)
  box = _box(lo, hi)
  lo_b, hi_b = np.where(box, lo, 0.0), np.where(box, hi, 1.0)
  tiny = np.finfo(np.float64).tiny
  inner = np.maximum(hi_b - lo_b - softplus_inv(np.maximum(hi_b - y, tiny)), tiny)
  return np.where(box, lo_b + softplus_inv(inner), y)


def adam_train(theta0, lo, hi, loss_and_grad, *, learning_rate, epochs, b1=0.9, b2=0.999, eps=1e-8, eps_root=0.0):
  """theta0 [R, P]; loss_and_grad(theta) -> (loss, grad) (may raise: a failed evaluation).  Returns
  (theta [R, P] after the last update, final losses [R], loss trace [epochs, R])."""
  theta0 = np.atleast_2d(np.asarray(theta0, np.float64))
  r = theta0.shape[0]
  out = np.zeros_like(theta0)
  trace = np.full((epochs, r), np.nan)
  for i in range(r):
    u = soft_clip_inverse(theta0[i], lo, hi)
    mu = np.zeros_like(u)
    nu = np.zeros_like(u)
    for t in range(1, epochs + 1):
      th = soft_clip(u, lo, hi)
      try:
        loss, g = loss_and_grad(th)
        g = np.asarray(g, np.float64)
      except (ValueError, np.linalg.LinAlgError):
        loss, g = math.nan, np.full_like(u, math.nan)
      if not (np.isfinite(loss) and np.all(np.isfinite(g))):
        break
      trace[t - 1, i] = loss
      gu = g * soft_clip_grad(u, lo, hi)
      mu = b1 * mu + (1.0 - b1) * gu
      nu = b2 * nu + (1.0 - b2) * gu ** 2
      mhat = mu / (1.0 - b1 ** t)
      nhat = nu / (1.0 - b2 ** t)
      u = u - learning_rate * mhat / (np.sqrt(nhat + eps_root) + eps)
    else:
      out[i] = soft_clip(u, lo, hi)
      continue
    out[i] = th
  return out, trace[-1].copy(), trace


def best_n(final_losses, n):
  """Indices of the n best restarts: a stable argsort with NaN last."""
  return np.argsort(np.asarray(final_losses, np.float64), kind='stable')[:max(1, n)]
