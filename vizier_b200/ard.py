"""ARD: fits the GP hyper-parameters by multi-restart L-BFGS-B on the device loss/gradient.

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
"""

from __future__ import annotations

import dataclasses
from typing import List, Optional, Tuple

import numpy as np
import scipy.optimize as sopt

from vizier_b200 import gp

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


def _lockstep(batch_fn, inits, bounds, **kw):
  """All restarts at once: every round collects the point each unfinished restart asks for and evaluates
  them with ONE call of `batch_fn(indices, points) -> (losses, grads)` (one CUDA graph launch for all
  restarts, gp.DeviceGP.make_batch_loss_fn).  Each restart's sequence of iterates is exactly the one it
  would have had alone."""
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
      try:
        pending[i] = gens[i].send((losses[k], grads[k]))
      except StopIteration as done:
        results[i] = done.value
        del pending[i]
  return [results[i] for i in range(len(gens))]


def log_uniform_init(rng: np.random.Generator, dc: int, dk: int, n: int, linear: bool = False) -> np.ndarray:
  lo, hi = gp.param_bounds(dc, dk)
  u = rng.uniform(size=(n, lo.shape[0]))
  th = np.exp(u * np.log(hi / lo) + np.log(lo))
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


def train_gp(dev: gp.DeviceGP, x, y, z=None, *, rng: np.random.Generator,
             random_restarts: int = DEFAULT_RANDOM_RESTARTS, ensemble_size: int = 1,
             optimizer: Optional[ScipyLbfgsB] = None, n_valid: Optional[int] = None,
             workers: int = MAX_ARD_WORKERS, linear_coef: Optional[float] = None) -> Tuple[List[gp.GPHyperParams], np.ndarray]:
  """Returns the best `ensemble_size` hyper-parameter sets and all final losses.

  x [N,Dc] float64, z [N,Dk] int32 or None, y [N] or [N, M]: device tensors or arrays (copied once).
  """
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
  lo, hi = gp.param_bounds(dc, dk, linear=bool(linear_coef))
  inits = log_uniform_init(rng, dc, dk, random_restarts, linear=bool(linear_coef))
  if BATCHED_ARD and _setulb is not None and xt.shape[0] > 64 and 1 < random_restarts <= 16 and workers > 1 and not linear_coef:
    fns = batch_loss_function(dev, xt, yt, zt, random_restarts, n_valid)
  else:
    fns = loss_functions(dev, xt, yt, zt, dc, dk, n_valid, workers=min(workers, random_restarts), linear_coef=linear_coef)
  try:
    best, losses = optimizer(inits, fns, list(zip(lo, hi)), best_n=ensemble_size)
  finally:
    dev.set_int('dataflow_ctas', 0)     # the fit that follows runs alone: every slot
  return [gp.GPHyperParams.from_vector(t, dc, dk, linear_coef) for t in best], losses
