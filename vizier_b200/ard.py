"""ARD: fits the GP hyper-parameters by multi-restart L-BFGS-B (the default) or Adam on the device loss/gradient.

Mirrors `gp_models._train_gp` (vizier/_src/algorithms/designers/gp/gp_models.py:169-223) with the
default optimiser `JaxoptScipyLbfgsB(LbfgsBOptions(maxiter=50))`
(vizier/_src/jax/optimizers/jaxopt_wrappers.py:108-199; vizier/jax/optimizers.py:30-37):
  * `random_restarts` initial points drawn log-uniformly inside the box
    (tuned_gp_models.py:42-63),
  * each refined by SciPy's L-BFGS-B in the CONSTRAINED space with box bounds, gtol=1e-8,
    maxls=20 (the same Fortran routine jaxopt.ScipyBoundedMinimize reaches),
  * the `best_n` lowest final losses are kept (optimizers/core.py:104-132).
loss(theta) and its gradient come from `vzgp_nll_grad` (CUDA); SciPy only drives.
The draws use NumPy's Generator rather than JAX threefry: seeded trajectories are reproducible
but not bit-identical to a JAX run (SURVEY 8c).

`OptaxTrain(adam(lr), epochs=T)` is the reference's second ARD optimiser (optax_wrappers.py:36-150): Adam on the
unconstrained u of each parameter's SoftClip(low, high, hinge_softness=1e-2) bijector (unbounded parameters: the
identity), all restarts for a fixed number of epochs; each epoch evaluates once, then updates; the `best_n` restarts
with the lowest loss of the LAST evaluation are kept (their parameters after the last update).  Single-metric studies
of N <= 64 trials without `linear_coef` run every epoch of every restart in ONE kernel launch (`vzgp_ard_adam_small`,
csrc/ard_adam.cu: route 'fused'); every other study runs one device evaluation per epoch on the loss callables below
with the SoftClip and Adam arithmetic in NumPy (route 'host').  `OptaxTrain.last_metrics` holds the loss trace
[epochs, R], the final losses and the route of its last run.  Separable multi-task types raise NotImplementedError
with it (their task parameters have non-box bijectors in the reference).
"""

from __future__ import annotations

import dataclasses
import logging
from typing import Any, List, Optional, Tuple

import numpy as np
import scipy.optimize as sopt

from vizier_b200 import gp
from vizier_b200 import task_kernels

DEFAULT_RANDOM_RESTARTS = 4


@dataclasses.dataclass(frozen=True)
class LbfgsBOptions:
  num_line_search_steps: int = 20
  tol: float = 1e-8
  maxiter: int = 50


try:  # SciPy's compiled L-BFGS-B step routine (the one `minimize(method='L-BFGS-B')` drives)
  from scipy.optimize import _lbfgsb as _lbfgsb_mod
  import scipy.optimize._lbfgsb_py as _lbfgsb_py
  _setulb = _lbfgsb_mod.setulb
  _INT = np.int64 if getattr(_lbfgsb_py, 'HAS_ILP64', False) else np.int32
  # The lean driver below speaks the C translation's calling convention (SciPy >= 1.15: integer `task`
  # and `ln_task` arrays, no iprint/csave).  The older f2py/Fortran routine takes other arguments and
  # could misread these, so it is recognised by its docstring and left to `scipy.optimize.minimize`.
  _doc = _setulb.__doc__ or ''
  if 'csave' in _doc or 'iprint' in _doc or 'ln_task' not in _doc:
    _setulb = None
except Exception:  # pylint: disable=broad-except
  _setulb = None
  _INT = np.int32


def _lean_lbfgsb_steps(x0: np.ndarray, bounds, *, maxiter: int, gtol: float, maxls: int,
                       ftol: float = 2.220446049250313e-09, maxcor: int = 10, maxfun: int = 15000):
  """The loop of `scipy.optimize._lbfgsb_py._minimize_lbfgsb` around the same compiled `setulb` routine as a
  GENERATOR: it yields the point it wants evaluated and is sent back (loss, gradient); its return value
  (StopIteration.value) is (x, f).  Identical iterates and results to `scipy.optimize.minimize`, without the
  per-evaluation Python layers (ScalarFunction wrappers, OptimizeResult per iteration).  The reverse-
  communication form is what lets several restarts advance in lock step, one batched device evaluation per
  round (`_lockstep`).  All bounds must be finite (they are: param_bounds)."""
  n, m = x0.shape[0], maxcor
  low = np.array([b[0] for b in bounds], np.float64)
  up = np.array([b[1] for b in bounds], np.float64)
  # SciPy's codes: 0 unbounded, 1 lower only, 2 both, 3 upper only (the linear_coef model has free parameters)
  fl, fu = np.isfinite(low), np.isfinite(up)
  nbd = np.where(fl & fu, 2, np.where(fl, 1, np.where(fu, 3, 0))).astype(_INT)
  x = np.clip(np.array(x0, dtype=np.float64), low, up)
  f = np.array(0.0, dtype=np.float64)
  g = np.zeros(n, np.float64)
  wa = np.zeros(2 * m * n + 5 * n + 11 * m * m + 8 * m, np.float64)
  iwa = np.zeros(3 * n, dtype=_INT)
  task = np.zeros(2, dtype=_INT)
  ln_task = np.zeros(2, dtype=_INT)
  lsave = np.zeros(4, dtype=_INT)
  isave = np.zeros(44, dtype=_INT)
  dsave = np.zeros(29, np.float64)
  factr = ftol / np.finfo(float).eps
  nit = nfev = 0
  while True:
    _setulb(m, x, low, up, nbd, f, g, factr, gtol, wa, iwa, task, lsave, isave, dsave, maxls, ln_task)
    if task[0] == 3:
      fv, gv = yield x
      nfev += 1
      f = np.array(fv, dtype=np.float64)
      g = np.asarray(gv, np.float64)
    elif task[0] == 1:
      nit += 1
      if nit >= maxiter:
        task[0], task[1] = 5, 504
      elif nfev > maxfun:
        task[0], task[1] = 5, 502
    else:
      break
  return x, float(f)


def _lean_lbfgsb(fun, x0: np.ndarray, bounds, **kw):
  """One restart driven to completion with `fun(x) -> (loss, gradient)`."""
  steps = _lean_lbfgsb_steps(x0, bounds, **kw)
  try:
    x = next(steps)
    while True:
      x = steps.send(fun(x))
  except StopIteration as done:
    return done.value


def _lockstep(batch_fn, inits, bounds, stop_nonfinite: bool = False, **kw):
  """All restarts at once: every round collects the point each unfinished restart asks for and evaluates
  them with ONE call of `batch_fn(indices, points) -> (losses, grads)` (one CUDA graph launch for all
  restarts, gp.DeviceGP.make_batch_loss_fn).  Each restart's sequence of iterates is exactly the one it
  would have had alone.  With stop_nonfinite, a restart sent a non-finite loss or gradient ends at that point
  with that loss."""
  gens = [_lean_lbfgsb_steps(np.asarray(t0, np.float64), bounds, **kw) for t0 in inits]
  pending, results = {}, {}
  for i, gen in enumerate(gens):
    try:
      pending[i] = next(gen)
    except StopIteration as done:
      results[i] = done.value
  while pending:
    idx = sorted(pending)
    losses, grads = batch_fn(idx, [pending[i] for i in idx])
    for k, i in enumerate(idx):
      if stop_nonfinite and not (np.isfinite(losses[k]) and np.all(np.isfinite(grads[k]))):
        results[i] = (np.array(pending[i], np.float64), float(losses[k]))
        del pending[i]
        continue
      try:
        pending[i] = gens[i].send((losses[k], grads[k]))
      except StopIteration as done:
        results[i] = done.value
        del pending[i]
  return [results[i] for i in range(len(gens))]


def log_uniform_init(rng: np.random.Generator, dc: int, dk: int, n: int, linear: bool = False,
                     multitask_type: Optional[str] = None, n_metrics: int = 1) -> np.ndarray:
  lo, hi = gp.param_bounds(dc, dk)
  u = rng.uniform(size=(n, lo.shape[0]))
  th = np.exp(u * np.log(hi / lo) + np.log(lo))
  if multitask_type:   # the task parameters' own initialisers (task_kernels.init), in jaxopt's order
    task = task_kernels.init(multitask_type, rng, n_metrics, n)
    return np.stack([task_kernels.join(multitask_type, th[i], task[i], dc, dk) for i in range(n)])
  if linear:   # slope: log-uniform in the amplitude bounds; shift and mean: standard normal (tuned_gp_models.py:209-240)
    o = dk + dc
    slo, shi = gp.SIGNAL_VARIANCE_BOUNDS
    slope = np.exp(rng.uniform(size=(n, 1)) * np.log(shi / slo) + np.log(slo))
    th = np.concatenate([th[:, :o], rng.standard_normal((n, 1)), slope, rng.standard_normal((n, 1)), th[:, o:]], axis=1)
  return th


@dataclasses.dataclass
class ScipyLbfgsB:
  """The reference's default ARD optimiser, driving the CUDA loss.

  `loss_and_grad` is one callable, or a sequence of equivalent callables (one per libvzgp handle,
  `loss_functions` below): the restarts are independent, so they then run concurrently, one host
  thread per handle/stream (ctypes releases the GIL while the device works).  An evaluation at
  N ~ 1000 is a chain of small latency-bound kernels, so four restarts overlap almost perfectly on
  one GPU.  Results do not depend on the number of workers.
  """

  options: LbfgsBOptions = LbfgsBOptions()

  def _one(self, fn, t0, bounds):
    if _setulb is not None:
      try:
        return _lean_lbfgsb(fn, np.asarray(t0, np.float64), bounds, maxiter=self.options.maxiter,
                            gtol=self.options.tol, maxls=self.options.num_line_search_steps)
      except Exception:   # pylint: disable=broad-except  # private SciPy entry point changed: use the public one
        pass
    res = sopt.minimize(fn, t0, jac=True, method='L-BFGS-B', bounds=bounds,
                        options={'maxiter': self.options.maxiter, 'gtol': self.options.tol,
                                 'maxls': self.options.num_line_search_steps})
    return res.x, float(res.fun)

  def __call__(self, init_thetas: np.ndarray, loss_and_grad, bounds, best_n: int = 1):
    inits = np.atleast_2d(init_thetas)
    if hasattr(loss_and_grad, 'n_restarts') and _setulb is not None and loss_and_grad.n_restarts >= inits.shape[0]:
      # batched device evaluation: the restarts advance in lock step, one graph launch per round
      results = _lockstep(loss_and_grad, inits, bounds, maxiter=self.options.maxiter, gtol=self.options.tol,
                          maxls=self.options.num_line_search_steps)
      finals = [r[0] for r in results]
      losses = np.asarray([r[1] for r in results])
      order = np.argsort(losses, kind='stable')[:max(1, best_n)]
      return [finals[i] for i in order], losses
    fns = list(loss_and_grad) if isinstance(loss_and_grad, (list, tuple)) else [loss_and_grad]
    if len(fns) == 1 or inits.shape[0] == 1:
      results = [self._one(fns[0], t0, bounds) for t0 in inits]
    else:
      import concurrent.futures as cf
      import queue
      free = queue.SimpleQueue()
      for fn in fns:
        free.put(fn)

      def run(t0):
        fn = free.get()
        try:
          return self._one(fn, t0, bounds)
        finally:
          free.put(fn)

      with cf.ThreadPoolExecutor(max_workers=len(fns)) as pool:
        results = list(pool.map(run, inits))
    finals = [r[0] for r in results]
    losses = np.asarray([r[1] for r in results])
    order = np.argsort(losses, kind='stable')[:max(1, best_n)]
    return [finals[i] for i in order], losses


HINGE_SOFTNESS = 1e-2   # SoftClip(low, high, hinge_softness=1e-2) of every bounded parameter (tuned_gp_models.py)


def _softplus(v):
  """c log1p(exp(v / c)), c = HINGE_SOFTNESS, in the overflow-free form max(v, 0) + c log1p(exp(-|v| / c))."""
  return np.maximum(v, 0.0) + HINGE_SOFTNESS * np.log1p(np.exp(-np.abs(v) / HINGE_SOFTNESS))


def _softplus_inv(s):
  """The inverse of `_softplus` for s > 0: s + c log(-expm1(-s / c))."""
  return s + HINGE_SOFTNESS * np.log(-np.expm1(-s / HINGE_SOFTNESS))


def _sigmoid(z):
  with np.errstate(over='ignore'):
    e = np.exp(np.minimum(z, 0.0))
    return np.where(z >= 0.0, 1.0 / (1.0 + np.exp(-np.maximum(z, 0.0))), e / (1.0 + e))


def soft_clip(u, lo, hi):
  """theta = hi - sp(hi - lo - sp(u - lo)) and dtheta/du, elementwise; the identity where a bound is infinite.
  The operations are those of csrc/ard_adam.cu, in the same order."""
  u = np.asarray(u, np.float64)
  box = np.isfinite(lo) & np.isfinite(hi)
  lo_b, hi_b = np.where(box, lo, 0.0), np.where(box, hi, 1.0)
  a = u - lo_b
  w = (hi_b - lo_b) - _softplus(a)
  th = hi_b - _softplus(w)
  d = _sigmoid(w / HINGE_SOFTNESS) * _sigmoid(a / HINGE_SOFTNESS)
  return np.where(box, th, u), np.where(box, d, 1.0)


def soft_clip_inverse(theta, lo, hi):
  """u with soft_clip(u) = theta; the arguments of sp^-1 are kept >= the smallest normal double, so a point on or past a
  bound maps to a finite u (where the bijector is flat)."""
  theta = np.asarray(theta, np.float64)
  box = np.isfinite(lo) & np.isfinite(hi)
  lo_b, hi_b = np.where(box, lo, 0.0), np.where(box, hi, 1.0)
  tiny = np.finfo(np.float64).tiny
  r = _softplus_inv(np.maximum(hi_b - theta, tiny))
  u = lo_b + _softplus_inv(np.maximum((hi_b - lo_b) - r, tiny))
  return np.where(box, u, theta)


@dataclasses.dataclass(frozen=True)
class adam:  # pylint: disable=invalid-name  # stands in for optax.adam (optax is not a dependency)
  """optax.adam(learning_rate, b1, b2, eps, eps_root): scale_by_adam, then scale by -learning_rate."""

  learning_rate: float
  b1: float = 0.9
  b2: float = 0.999
  eps: float = 1e-8
  eps_root: float = 0.0


class _Evaluator:
  """(indices, thetas) -> (losses, grads) over any of the loss-callable forms ScipyLbfgsB takes: a batched callable
  (`n_restarts`: one call), a sequence of equivalent callables on distinct handles (the restarts split between them, one
  host thread per handle, so their evaluations overlap on the GPU) or one callable (the restarts one after another).
  Results do not depend on the number of handles."""

  def __init__(self, loss_and_grad):
    self._batch = loss_and_grad if hasattr(loss_and_grad, 'n_restarts') else None
    fns = list(loss_and_grad) if isinstance(loss_and_grad, (list, tuple)) else [loss_and_grad]
    self._fns = fns
    self._pool = None
    if self._batch is None and len(fns) > 1:
      import concurrent.futures as cf
      self._pool = cf.ThreadPoolExecutor(max_workers=len(fns))

  def __call__(self, indices, thetas):
    if self._batch is not None:
      return self._batch(indices, thetas)
    w = min(len(self._fns), len(thetas))
    if self._pool is None or w <= 1:
      out = [self._fns[0](t) for t in thetas]
    else:
      parts = [self._pool.submit(lambda j: [self._fns[j](t) for t in thetas[j::w]], j) for j in range(w)]
      done = [p.result() for p in parts]
      out = [done[k % w][k // w] for k in range(len(thetas))]
    return [o[0] for o in out], [o[1] for o in out]

  def close(self):
    if self._pool is not None:
      self._pool.shutdown()


def adam_host_epochs(opt: adam, epochs: int, init_thetas: np.ndarray, lo, hi, evaluate):
  """The host-stepped Adam loop: one `evaluate(indices, thetas)` per epoch over the restarts still running, SoftClip and
  Adam in NumPy with the operations of csrc/ard_adam.cu.  A restart whose loss (or gradient) is not finite - the loss
  callables return 1e300 for a non-finite loss - stops there: NaN losses from that epoch on and the parameters of that
  evaluation.  Returns (theta [R, P], final losses [R], loss trace [epochs, R])."""
  th0 = np.atleast_2d(np.asarray(init_thetas, np.float64))
  r = th0.shape[0]
  lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
  u = soft_clip_inverse(th0, lo, hi)
  mu, nu = np.zeros_like(u), np.zeros_like(u)
  trace = np.full((epochs, r), np.nan)
  alive = np.ones(r, bool)
  stopped_at = np.zeros_like(u)
  b1t = b2t = 1.0
  for e in range(epochs):
    idx = np.flatnonzero(alive)
    if not idx.size:
      break
    th, dth = soft_clip(u[idx], lo, hi)
    losses, grads = evaluate(list(idx), list(th))
    good = np.zeros(idx.size, bool)
    g = np.zeros((idx.size, u.shape[1]))
    for k, i in enumerate(idx):
      gk = np.asarray(grads[k], np.float64)
      if np.isfinite(losses[k]) and losses[k] < 1e300 and np.all(np.isfinite(gk)):
        good[k] = True
        trace[e, i] = losses[k]
        g[k] = gk
      else:
        alive[i] = False
        stopped_at[i] = th[k]
    b1t = b1t * opt.b1
    b2t = b2t * opt.b2
    j = idx[good]
    gu = g[good] * dth[good]
    mu[j] = (1.0 - opt.b1) * gu + opt.b1 * mu[j]
    nu[j] = (1.0 - opt.b2) * (gu * gu) + opt.b2 * nu[j]
    upd = (mu[j] / (1.0 - b1t)) / (np.sqrt(nu[j] / (1.0 - b2t) + opt.eps_root) + opt.eps)
    u[j] = u[j] + (-opt.learning_rate) * upd
  theta = np.where(alive[:, None], soft_clip(u, lo, hi)[0], stopped_at)
  final = np.where(alive, trace[-1], np.nan)
  return theta, final, trace


@dataclasses.dataclass
class OptaxTrain:
  """The reference's `OptaxTrain(optimizer, *, epochs, verbose=0)` with `optimizer=adam(...)`; see the module
  docstring.  Called like ScipyLbfgsB on loss callables it runs the host-stepped epochs; `fit` picks the fused kernel
  where the study allows it."""

  optimizer: Any
  epochs: int = dataclasses.field(kw_only=True)
  verbose: int = dataclasses.field(default=0, kw_only=True)
  # of the last run: 'loss' [epochs, R], 'final_loss' [R], 'route' ('fused' or 'host'), 'status' [R] (fused: the
  # Cholesky retries of each restart's last evaluation; host: None)
  last_metrics: Optional[dict] = dataclasses.field(default=None, init=False, repr=False, compare=False)

  def __post_init__(self):
    if not isinstance(self.optimizer, adam):
      raise NotImplementedError(f'OptaxTrain takes the ard.adam optimiser only, not {type(self.optimizer).__name__}.')
    if int(self.epochs) < 1:
      raise NotImplementedError('OptaxTrain needs epochs >= 1.')
    self.epochs = int(self.epochs)
    self.verbose = int(self.verbose)

  def _finish(self, thetas, final, trace, route, status, best_n):
    self.last_metrics = {'loss': trace, 'final_loss': final, 'route': route, 'status': status}
    if self.verbose >= 1:
      for e, row in enumerate(trace):
        logging.info('Epoch %s: loss %s', e, row)
    order = np.argsort(final, kind='stable')[:max(1, best_n)]
    return [thetas[i] for i in order], final

  def __call__(self, init_thetas: np.ndarray, loss_and_grad, bounds, best_n: int = 1):
    """Host-stepped epochs on `loss_and_grad` (any form ScipyLbfgsB takes); returns (best_n thetas, final losses)."""
    lo = np.array([b[0] for b in bounds], np.float64)
    hi = np.array([b[1] for b in bounds], np.float64)
    evaluate = _Evaluator(loss_and_grad)
    try:
      thetas, final, trace = adam_host_epochs(self.optimizer, self.epochs, init_thetas, lo, hi, evaluate)
    finally:
      evaluate.close()
    return self._finish(thetas, final, trace, 'host', None, best_n)

  def fit(self, dev: gp.DeviceGP, xt, yt, zt, init_thetas: np.ndarray, lo, hi, *, best_n: int = 1,
          n_valid: Optional[int] = None, linear_coef: Optional[float] = None):
    """ARD of one model on device tensors: the fused kernel for a single-metric study of N <= 64 trials without
    linear_coef (when its shared memory fits one CTA), else host-stepped epochs on the batched loss callable (N > 64,
    2-16 restarts, no linear_coef) or on up to MAX_ARD_WORKERS handles evaluating the restarts concurrently.  Returns
    (best_n thetas, final losses)."""
    from vizier_b200 import _lib
    inits = np.atleast_2d(np.asarray(init_thetas, np.float64))
    n, dc = xt.shape
    dk = 0 if zt is None else zt.shape[1]
    single = yt.ndim == 1 or yt.shape[1] == 1
    opt = self.optimizer
    if single and not linear_coef and _lib.load().vzgp_ard_adam_small_supported(n, dc, dk):
      thetas, final, status, trace = dev.ard_adam_small(
          xt, yt.reshape(-1), inits, lo, hi, learning_rate=opt.learning_rate, b1=opt.b1, b2=opt.b2, eps=opt.eps,
          eps_root=opt.eps_root, epochs=self.epochs, z=zt, n_valid=n_valid)
      return self._finish(list(thetas), final, trace, 'fused', status, best_n)
    r = inits.shape[0]
    if n > 64 and 1 < r <= 16 and not linear_coef:
      fns = batch_loss_function(dev, xt, yt, zt, r, n_valid)
    else:
      fns = loss_functions(dev, xt, yt, zt, dc, dk, n_valid, workers=min(MAX_ARD_WORKERS, r), linear_coef=linear_coef)
    return self(inits, fns, list(zip(lo, hi)), best_n=best_n)


MAX_ARD_WORKERS = 8


def _cta_share(n_concurrent: int) -> int:
  """Worker CTAs of the dataflow factorisation per concurrent evaluation (0 = every slot, a lone evaluation).
  The persistent CTAs of k_chol_dataflow fill an SM's shared memory and registers two by two; the small kernels
  around the factorisation (kernel matrix, alpha solve, gradient tiles) of the OTHER evaluations need somewhere
  to run meanwhile, so the restarts together take only part of the 2 x 132 slots."""
  import os
  if n_concurrent <= 1:
    return 0
  env = os.environ.get('VZGP_ARD_SHARE')
  if env:
    return int(env)
  return max(16, ARD_SLOT_BUDGET // n_concurrent - 1)


ARD_SLOT_BUDGET = 192


def loss_functions(dev: gp.DeviceGP, xt, yt, zt, dc: int, dk: int, n_valid: Optional[int] = None,
                   workers: int = MAX_ARD_WORKERS, linear_coef: Optional[float] = None):
  """One loss/gradient callable per worker handle (the designer's own handle first; extra handles on
  their own streams are created once and cached on `dev`)."""
  workers = max(1, int(workers))
  pool = getattr(dev, '_ard_workers', None)
  if pool is None:
    pool = []
    dev._ard_workers = pool  # pylint: disable=protected-access
  while len(pool) < workers - 1:
    pool.append(gp.DeviceGP(dev.device.index))
  devs = [dev] + pool[:workers - 1]
  # The evaluations of the restarts run concurrently, one dataflow-factorisation launch each: an equal
  # share of the 2 x 132 resident CTA slots keeps all of them on the GPU at once (csrc/dataflow.cu).
  share = _cta_share(len(devs))
  for d in devs:
    d.set_int('dataflow_ctas', share)

  return [d.make_loss_fn(xt, yt, zt, n_valid, linear_coef=linear_coef) for d in devs]


def batch_loss_function(dev: gp.DeviceGP, xt, yt, zt, restarts: int, n_valid: Optional[int] = None):
  """One batched loss/gradient callable for `restarts` concurrent evaluations (worker handles cached on
  `dev`, as in `loss_functions`), each with an equal share of the dataflow factorisation's CTA slots."""
  pool = getattr(dev, '_ard_workers', None)
  if pool is None:
    pool = []
    dev._ard_workers = pool  # pylint: disable=protected-access
  while len(pool) < restarts - 1:
    pool.append(gp.DeviceGP(dev.device.index))
  devs = [dev] + pool[:restarts - 1]
  share = _cta_share(len(devs))
  for d in devs:
    d.set_int('dataflow_ctas', share)
  return gp.DeviceGP.make_batch_loss_fn(devs, xt, yt, zt, n_valid)


BATCHED_ARD = True   # restarts in lock step on one graph launch per round (N > 64); False: one host thread per restart


def separable_loss_function(dev: gp.DeviceGP, xt, yt, zt, restarts: int, n_metrics: int, multitask_type: str,
                            n_valid: Optional[int] = None):
  """Batched loss/gradient of the separable multi-task GP for `restarts` restarts: restarts x n_metrics handles on
  distinct streams (`dev` first, the others created once and cached on it), each with an equal share of the dataflow
  factorisation's CTA slots."""
  pool = getattr(dev, '_separable_workers', None)
  if pool is None:
    pool = []
    dev._separable_workers = pool  # pylint: disable=protected-access
  need = restarts * n_metrics
  while len(pool) < need - 1:
    pool.append(gp.DeviceGP(dev.device.index))
  devs = [dev] + pool[:need - 1]
  share = _cta_share(len(devs))
  for d in devs:
    d.set_int('dataflow_ctas', share)
  return gp.separable_batch_loss_fn(devs, n_metrics, multitask_type, xt, yt, zt, n_valid)


def train_gp(dev: gp.DeviceGP, x, y, z=None, *, rng: np.random.Generator,
             random_restarts: int = DEFAULT_RANDOM_RESTARTS, ensemble_size: int = 1,
             optimizer=None, n_valid: Optional[int] = None,
             workers: int = MAX_ARD_WORKERS, linear_coef: Optional[float] = None,
             multitask_type=None) -> Tuple[List[gp.GPHyperParams], np.ndarray]:
  """Returns the best `ensemble_size` hyper-parameter sets and all final losses.

  optimizer: ScipyLbfgsB (None: the default one) or OptaxTrain (Adam; not with a separable multitask_type).

  x [N,Dc] float64, z [N,Dk] int32 or None, y [N] or [N, M]: device tensors or arrays (copied once).
  multitask_type: a separable type (task_kernels.TYPES, a name or an enum member) fits the separable multi-task GP to
  y [N, M] with the restarts in lock step on `vzgp_nll_grad_separable_batch`; None / INDEPENDENT the independent one.
  """
  multitask_type = task_kernels.resolve(multitask_type)
  if multitask_type and isinstance(optimizer, OptaxTrain):
    raise NotImplementedError(f'OptaxTrain with the separable multi-task type {multitask_type} is not implemented '
                              '(its task parameters have non-box bijectors).')
  import torch  # device-memory handles only
  optimizer = optimizer or ScipyLbfgsB()
  xt = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).to(dev.device)
  if isinstance(y, torch.Tensor):
    yt = y
  else:   # [N], or [N, M] for a multi-metric study (independent multi-task GP)
    ya = np.asarray(y, np.float64)
    ya = ya.reshape(-1) if ya.ndim == 1 or ya.shape[1] == 1 else ya
    yt = torch.from_numpy(np.ascontiguousarray(ya)).to(dev.device)
  zt = None
  if z is not None and np.prod(tuple(z.shape)) > 0:
    zt = z if isinstance(z, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(z, dtype=np.int32)).to(dev.device)
  dc = xt.shape[1]
  dk = 0 if zt is None else zt.shape[1]
  if multitask_type:
    return _train_separable(dev, xt, yt, zt, dc, dk, rng, random_restarts, ensemble_size, optimizer, n_valid,
                            multitask_type)
  lo, hi = gp.param_bounds(dc, dk, linear=bool(linear_coef))
  inits = log_uniform_init(rng, dc, dk, random_restarts, linear=bool(linear_coef))
  if isinstance(optimizer, OptaxTrain):
    try:
      best, losses = optimizer.fit(dev, xt, yt, zt, inits, lo, hi, best_n=ensemble_size, n_valid=n_valid,
                                   linear_coef=linear_coef)
    finally:
      dev.set_int('dataflow_ctas', 0)
    return [gp.GPHyperParams.from_vector(t, dc, dk, linear_coef) for t in best], losses
  if BATCHED_ARD and _setulb is not None and xt.shape[0] > 64 and 1 < random_restarts <= 16 and workers > 1 and not linear_coef:
    fns = batch_loss_function(dev, xt, yt, zt, random_restarts, n_valid)
  else:
    fns = loss_functions(dev, xt, yt, zt, dc, dk, n_valid, workers=min(workers, random_restarts), linear_coef=linear_coef)
  try:
    best, losses = optimizer(inits, fns, list(zip(lo, hi)), best_n=ensemble_size)
  finally:
    dev.set_int('dataflow_ctas', 0)     # the fit that follows runs alone: every slot
  return [gp.GPHyperParams.from_vector(t, dc, dk, linear_coef) for t in best], losses


def _train_separable(dev, xt, yt, zt, dc, dk, rng, random_restarts, ensemble_size, optimizer, n_valid, multitask_type):
  m = yt.shape[1] if yt.ndim == 2 else 1
  if not 2 <= m <= 8 or random_restarts * m > 64:
    raise ValueError('the separable multi-task GP needs 2 <= n_metrics <= 8 and random_restarts * n_metrics <= 64')
  lo, hi = gp.param_bounds(dc, dk, multitask_type=multitask_type, n_metrics=m)
  inits = log_uniform_init(rng, dc, dk, random_restarts, multitask_type=multitask_type, n_metrics=m)
  fn = separable_loss_function(dev, xt, yt, zt, random_restarts, m, multitask_type, n_valid)
  if _setulb is None:   # SciPy without the reverse-communication routine: one restart after the other
    batch = fn

    def fn(theta):
      losses, grads = batch([0], [theta])
      return losses[0], grads[0]
  try:
    best, losses = optimizer(inits, fn, list(zip(lo, hi)), best_n=ensemble_size)
  finally:
    dev.set_int('dataflow_ctas', 0)
  return [gp.GPHyperParams.from_vector(t, dc, dk, multitask_type=multitask_type, n_metrics=m) for t in best], losses
