"""Acquisition optimisers: the host-side factories of the reference, executing on the device.

Mirrors
  * `VectorizedOptimizerFactory` / `VectorizedOptimizer` / `VectorizedStrategyResults`
    (vizier/_src/algorithms/optimizers/vectorized_base.py:668-710, :278-542, :125-131),
  * `EagleStrategyConfig` / `VectorizedEagleStrategyFactory`
    (vizier/_src/algorithms/optimizers/eagle_strategy.py:111-167, :325-407),
  * `random_strategy_factory` (random_vectorized_optimizer.py:114-123),
  * `LBFGSBOptimizerFactory` / `LBFGSBOptimizer` (lbfgsb_optimizer.py:48-250).
Calling a vectorised optimiser runs the whole ask-evaluate-tell loop inside libvzgp
(`vzgp_eagle_run` / `vzgp_random_search`); only the `count` winners come back to the host.  The L-BFGS-B
optimiser drives SciPy's L-BFGS-B on the host, all restarts in lock step, with the acquisition and its gradient
evaluated on the device (`vzgp_score_grad`), one batched call per round.
"""

from __future__ import annotations

import dataclasses
import enum
import math
from typing import Callable, Dict, Optional, Union

import numpy as np

from vizier_b200 import _lib, ard, gp

MAX_SET_POINTS = 16      # points of one set fly (n_parallel)
MAX_FLY_DIM = 1024       # coordinates of one set fly: n_parallel * Dc
_SET_LIMITS = (f'set acquisitions need the Eagle strategy, continuous features, n_parallel <= {MAX_SET_POINTS} and '
               f'n_parallel * Dc <= {MAX_FLY_DIM}')


class MutateNormalizationType(enum.IntEnum):
  """How the forces on a fly are normalised (eagle_strategy.py:92-98, :847-896)."""
  MEAN = 0          # pulls and pushes each divided by the number of flies exerting them
  RANDOM = 1        # random convex weights over the pulling flies
  UNNORMALIZED = 2  # the raw forces


class ContinuousFeaturePerturbationType(enum.IntEnum):
  """How the perturbation enters a moved continuous feature (eagle_strategy.py:101-108, :917-935)."""
  ADDITIVE = 0        # moved + perturbation
  MULTIPLICATIVE = 1  # moved * exp(perturbation)


@dataclasses.dataclass(frozen=True)
class EagleStrategyConfig:
  visibility: float = 0.45
  gravity: float = 1.5
  negative_gravity: float = 0.008
  perturbation: float = 0.16
  categorical_perturbation_factor: float = 1.0
  pure_categorical_perturbation_factor: float = 30
  prob_same_category_without_perturbation: float = 0.98
  perturbation_lower_bound: float = 7e-5
  penalize_factor: float = 7e-1
  pool_size_exponent: float = 1.2
  pool_size: int = 0
  max_pool_size: int = 100
  normalization_scale: float = 0.5
  prior_trials_pool_pct: float = 0.96
  mutate_normalization_type: int = MutateNormalizationType.MEAN
  continuous_feature_perturbation_type: int = ContinuousFeaturePerturbationType.ADDITIVE

  def __post_init__(self):
    # ValueError for a value the enums do not name, as the reference raises when it builds the features (:892-896,
    # :931-935); plain integers stay accepted.
    MutateNormalizationType(self.mutate_normalization_type)
    ContinuousFeaturePerturbationType(self.continuous_feature_perturbation_type)


@dataclasses.dataclass(frozen=True)
class VectorizedEagleStrategyFactory:
  eagle_config: EagleStrategyConfig = EagleStrategyConfig()

  def pool_size(self, n_features: int, suggestion_batch_size: Optional[int]) -> int:
    """eagle_strategy.py:376-386."""
    cfg = self.eagle_config
    pool = cfg.pool_size
    if pool == 0:
      pool = 10 + int(0.5 * n_features + n_features ** cfg.pool_size_exponent)
      pool = min(pool, cfg.max_pool_size)
      if suggestion_batch_size is not None:
        pool = int(math.ceil(pool / suggestion_batch_size) * suggestion_batch_size)
    return pool


class _RandomStrategyFactory:
  """Marker for RandomVectorizedStrategy (uniform candidates, no state)."""

  def __repr__(self):
    return 'random_strategy_factory'


random_strategy_factory = _RandomStrategyFactory()


@dataclasses.dataclass
class VectorizedStrategyResults:
  features: np.ndarray             # [count, Dc]
  rewards: np.ndarray              # [count]
  aux: Dict[str, np.ndarray] = dataclasses.field(default_factory=dict)
  categorical: Optional[np.ndarray] = None   # [count, Dk] int32


@dataclasses.dataclass
class VectorizedOptimizer:
  strategy_factory: Union[VectorizedEagleStrategyFactory, _RandomStrategyFactory]
  n_continuous: int
  n_categorical: int
  suggestion_batch_size: int = 25
  max_evaluations: int = 75_000
  categorical_sizes: tuple = ()

  def _eagle_config(self):
    f = self.strategy_factory
    pool = f.pool_size(self.n_continuous + self.n_categorical, self.suggestion_batch_size)
    c = f.eagle_config
    return _lib.EagleConfig(c.visibility, c.gravity, c.negative_gravity, c.perturbation,
                            c.perturbation_lower_bound, c.penalize_factor, c.normalization_scale,
                            c.prior_trials_pool_pct, pool, self.suggestion_batch_size, self.max_evaluations,
                            c.categorical_perturbation_factor, c.pure_categorical_perturbation_factor,
                            c.prob_same_category_without_perturbation, c.mutate_normalization_type)

  def _set_perturbation(self, owner) -> None:
    """The perturbation type is a setting of the handle that owns the Eagle loop (vzgp_set_int "eagle_perturbation"):
    set before every run so that no earlier optimiser's choice carries over."""
    owner.set_int('eagle_perturbation', int(self.strategy_factory.eagle_config.continuous_feature_perturbation_type))

  def _stepped_eagle(self, dev, acq, count, prior_features, prior_categorical, seed, other, prior_acquisition):
    """Eagle with the batch scored here: device acquisition + the caller's `prior_acquisition(continuous [m, Dc],
    categorical [m, Dk]) -> [m]` evaluated on the host (gp_ucb_pe.py:376-379, :487-490).  One D2H + H2D round trip
    per iteration; state, suggest and update stay on the device (gp.SteppedEagle)."""
    import torch
    is_pe = isinstance(acq, gp.UcbPeAcquisition)
    is_pe_multi = isinstance(acq, gp.UcbPeMultiAcquisition)
    has_cat = self.n_categorical > 0

    def score(xs, zs):
      with torch.cuda.stream(dev._stream):
        zq = zs if has_cat else None
        if is_pe_multi:
          out = dev.score_pe_multi(other, xs, acq, zs=zq)
        else:
          out = dev.score_pe(other, xs, acq, zs=zq) if is_pe else dev.score(xs, acq, zs=zq)
        xh = xs.cpu().numpy()
        zh = zs.cpu().numpy() if (has_cat and zs is not None) else np.zeros((xh.shape[0], 0), np.int32)
        vals = np.asarray(prior_acquisition(xh, zh), np.float64).reshape(-1)
        return out['score'] + torch.as_tensor(vals, dtype=torch.float64, device=dev.device)

    n_prior = 0 if prior_features is None else len(prior_features)
    self._set_perturbation(dev._lead() if hasattr(dev, '_lead') else dev)
    se = gp.SteppedEagle(dev, self._eagle_config(), count, seed, n_prior, list(self.categorical_sizes))
    if n_prior > 0:
      pt = dev._dev(prior_features, torch.float64)
      pz = dev._dev(prior_categorical, torch.int32) if has_cat else None
      se.seed(prior_features, prior_categorical, score(pt, pz))
    steps = (self.max_evaluations - 1) // self.suggestion_batch_size + 1
    for _ in range(steps):
      xs, zs, rewards = se.ask()
      r = score(xs, zs)
      with torch.cuda.stream(dev._stream):
        rewards.copy_(r)
      se.tell()
    return se.end()

  def optimize_sets(self, dev: gp.DeviceGP, other: gp.DeviceGP, pe: gp.UcbPeAcquisition, *, n_parallel: int,
                    prior_features: Optional[np.ndarray] = None, seed: int = 0,
                    prior_acquisition: Optional[Callable] = None) -> VectorizedStrategyResults:
    """`acquisition_optimizer(scoring_fn.score, ..., count=1, n_parallel=q)` with the set-PE acquisition
    (gp_ucb_pe.py:1178-1202; vectorized_base.py:331-377): a fly is a set of q points, scored by `vzgp_score_set_pe`;
    the Eagle state and kernels run in their n_parallel form through the host-stepped loop.  prior_features [n, Dc]
    are grouped into n // q consecutive sets (vectorized_base.py:108-122).  `prior_acquisition`, if given, is called
    with (continuous [B, q, Dc], categorical [B, q, 0]) and returns [B].  Returns the best set: features [q, Dc],
    rewards [q] (the set's acquisition value repeated), aux per point."""
    import torch
    q, d = int(n_parallel), self.n_continuous
    if isinstance(self.strategy_factory, _RandomStrategyFactory):
      raise NotImplementedError(_SET_LIMITS)

    def score(xs_flat):          # [B, q * Dc] device -> [B] device
      with torch.cuda.stream(dev._stream):
        out = dev.score_set_pe(other, xs_flat.reshape(-1, d), q, pe)['score']
        if prior_acquisition is not None:
          xh = xs_flat.cpu().numpy().reshape(-1, q, d)
          vals = np.asarray(prior_acquisition(xh, np.zeros((xh.shape[0], q, 0), np.int32)), np.float64).reshape(-1)
          out = out + torch.as_tensor(vals, dtype=torch.float64, device=dev.device)
        return out

    best, bs = self._eagle_sets(dev, q, score, prior_features, seed)
    out = dev.score_set_pe(other, best, q, pe)
    dev.synchronize()
    aux = {k: out[k].cpu().numpy() for k in ('mean', 'stddev', 'stddev_from_all')}
    if prior_acquisition is not None:
      aux['prior_acq_values'] = np.asarray(prior_acquisition(best[None], np.zeros((1, q, 0), np.int32)), np.float64).reshape(-1)
    return VectorizedStrategyResults(best, np.full(q, bs), aux, categorical=np.zeros((q, 0), np.int32))

  def _eagle_sets(self, dev, q: int, score: Callable, prior_features: Optional[np.ndarray], seed: int):
    """The n_parallel form of the Eagle optimiser through the host-stepped loop (vectorized_base.py:331-377): a fly is
    a set of q points and `score([B, q * Dc] device) -> [B] device` rates a batch of them.  prior_features [n, Dc] are
    grouped into n // q consecutive sets (vectorized_base.py:108-122).  Returns the best set [q, Dc] and its score."""
    import torch
    d = self.n_continuous
    if self.n_categorical > 0 or q > MAX_SET_POINTS or q * d > MAX_FLY_DIM:
      raise NotImplementedError(_SET_LIMITS)
    cfg = self._eagle_config()
    cfg.n_parallel = q
    lead = getattr(dev, 'members', [dev])[0]     # an ensemble's optimiser state lives on its first member
    n_sets = 0 if prior_features is None else len(prior_features) // q
    self._set_perturbation(lead)
    se = gp.SteppedEagle(lead, cfg, 1, seed, n_sets)
    if n_sets > 0:
      ps = np.ascontiguousarray(np.asarray(prior_features, np.float64)[: n_sets * q].reshape(n_sets, q * d))
      se.seed(ps, None, score(lead._dev(ps, torch.float64)))
    steps = (self.max_evaluations - 1) // self.suggestion_batch_size + 1
    for _ in range(steps):
      xs, _, rewards = se.ask()
      r = score(xs)
      with torch.cuda.stream(lead._stream):
        rewards.copy_(r)
      se.tell()
    bx, _, bs = se.end()
    return bx[0].reshape(q, d), float(bs[0])

  def optimize_qsets(self, dev, qacq: gp.QAcquisition, *, n_parallel: int, prior_features: Optional[np.ndarray] = None,
                     prior_categorical: Optional[np.ndarray] = None, seed: int = 0,
                     acq_seed: int = 0) -> VectorizedStrategyResults:
    """`acquisition_optimizer(scoring_fn.score, ..., count=1, n_parallel=q)` with a parallel acquisition (QEI / QPI /
    QUCB; vectorized_base.py:331-377): sets of q points scored by `score_qsets` (dev: DeviceGP or EnsembleGP) with
    one acquisition seed for the whole run, so the draws depend on a set's position in its batch
    (vectorized_base.py:382-404, :504-520).  Eagle: continuous features, n_parallel * Dc <= 1024.  Random strategy: a
    Philox pool of n_sets * q points (any features), scored at once, device top-1.  Returns the best set: features
    [q, Dc], categorical [q, Dk], rewards [q] (the set's acquisition value repeated), aux per point."""
    import torch
    q, dc, dk = int(n_parallel), self.n_continuous, self.n_categorical
    period = self.suggestion_batch_size
    if q < 1 or q > 16:
      raise NotImplementedError('parallel acquisitions need 1 <= n_parallel <= 16')
    lead = getattr(dev, 'members', [dev])[0]
    if isinstance(self.strategy_factory, _RandomStrategyFactory):
      n_sets = ((self.max_evaluations - 1) // self.suggestion_batch_size + 1) * self.suggestion_batch_size
      m = n_sets * q
      xs = lead.random_pool(m, dc, seed) if dc else torch.zeros((m, 0), dtype=torch.float64, device=lead.device)
      zs = lead.random_pool_cat(m, list(self.categorical_sizes), seed) if dk else None
      out = dev.score_qsets(xs, q, qacq, acq_seed, zs=zs, period=period)
      idx, _ = lead.topk(out['score'], 1)
      rows = torch.arange(q, device=lead.device) + int(max(idx[0], 0)) * q
      best = xs[rows].cpu().numpy()
      best_z = zs[rows].cpu().numpy() if zs is not None else np.zeros((q, 0), np.int32)
    else:
      def score(xs_flat):      # [B, q * Dc] device -> [B] device
        with torch.cuda.stream(lead._stream):
          return dev.score_qsets(xs_flat.reshape(-1, dc), q, qacq, acq_seed, period=period)['score']

      best, _ = self._eagle_sets(dev, q, score, prior_features, seed)
      best_z = np.zeros((q, 0), np.int32)
    # score_with_aux on the winning set (vectorized_base.py:504-526): one set at position 0
    out = dev.score_qsets(best, q, qacq, acq_seed, zs=best_z if dk else None, period=period, with_aux=True)
    dev.synchronize()
    value = float(out['score'].cpu().numpy()[0])
    aux = {'mean': out['mean'].cpu().numpy(), 'stddev': out['stddev'].cpu().numpy()}
    if qacq.use_trust_region:
      aux['linf_distance'] = out['linf_distance'].cpu().numpy()
      aux['radius'] = np.full(q, qacq.trust_radius)
    return VectorizedStrategyResults(best, np.full(q, value), aux, categorical=best_z)

  def __call__(self, dev: gp.DeviceGP, acq, *, count: int = 1,
               prior_features: Optional[np.ndarray] = None, prior_categorical: Optional[np.ndarray] = None,
               seed: int = 0, other: Optional[gp.DeviceGP] = None,
               prior_acquisition: Optional[Callable] = None) -> VectorizedStrategyResults:
    """acq: gp.Acquisition (UCB + trust region on `dev`), gp.ScalarizedUcbAcquisition, or gp.UcbPeAcquisition /
    gp.UcbPeMultiAcquisition (both need `other`; the multi-metric aux 'mean' is [count, n_metrics])."""
    sizes = list(self.categorical_sizes)
    is_pe = isinstance(acq, (gp.UcbPeAcquisition, gp.UcbPeMultiAcquisition))
    is_multi = isinstance(acq, gp.ScalarizedUcbAcquisition)

    def pe_aux(bx, bz):
      if isinstance(acq, gp.UcbPeMultiAcquisition):
        out = dev.score_pe_multi(other, bx, acq, zs=bz if self.n_categorical else None)
        aux = {k: out[k].cpu().numpy() for k in ('stddev', 'stddev_from_all')}
        aux['mean'] = out['mean'].cpu().numpy().T
        return aux
      out = dev.score_pe(other, bx, acq, zs=bz if self.n_categorical else None)
      return {k: out[k].cpu().numpy() for k in ('mean', 'stddev', 'stddev_from_all')}

    if prior_acquisition is not None:
      if is_multi or isinstance(self.strategy_factory, _RandomStrategyFactory):
        raise NotImplementedError('prior_acquisition is supported with the Eagle strategy on single-metric acquisitions')
      bx, bz, bs = self._stepped_eagle(dev, acq, count, prior_features, prior_categorical, seed, other, prior_acquisition)
      zsel = bz if self.n_categorical else None
      prior_vals = np.asarray(prior_acquisition(bx, bz), np.float64).reshape(-1)
      if is_pe:
        aux = pe_aux(bx, bz)
      else:
        out = dev.score(bx, acq, zs=zsel, with_aux=True)
        dev.synchronize()
        aux = {'mean': out['mean'].cpu().numpy(), 'stddev': out['stddev'].cpu().numpy()}
      aux['prior_acq_values'] = prior_vals
      return VectorizedStrategyResults(bx, bs, aux, categorical=bz)
    if isinstance(self.strategy_factory, _RandomStrategyFactory) and is_multi:
      # uniform pool -> scalarised UCB -> device top-k, like vzgp_random_search but with the multi-metric scorer
      import torch
      n = (self.max_evaluations - 1) // self.suggestion_batch_size + 1
      m = n * self.suggestion_batch_size
      xs = dev.random_pool(m, self.n_continuous, seed) if self.n_continuous else torch.zeros((m, 0), dtype=torch.float64, device=dev.device)
      zs = dev.random_pool_cat(m, sizes, seed) if self.n_categorical else None
      out = dev.score_multi(xs, acq, zs=zs)
      idx, bs = dev.topk(out['score'], count)
      it = torch.from_numpy(np.maximum(idx, 0)).to(dev.device)
      bx = xs[it].cpu().numpy()
      bz = zs[it].cpu().numpy() if zs is not None else np.zeros((count, 0), np.int32)
    elif isinstance(self.strategy_factory, _RandomStrategyFactory):
      if is_pe:
        raise NotImplementedError('random strategy with the GP-UCB-PE acquisition')
      # one uniform batch per step; the device scores all max_evaluations candidates in one pass
      n = (self.max_evaluations - 1) // self.suggestion_batch_size + 1
      m = n * self.suggestion_batch_size
      bx, bz, bs, _ = dev.random_search(m, acq, count, seed, cat_sizes=sizes)
    else:
      cfg = self._eagle_config()
      self._set_perturbation(dev._lead() if hasattr(dev, '_lead') else dev)
      bx, bz, bs = dev.eagle_run(cfg, acq, count, seed, prior=prior_features, prior_z=prior_categorical,
                                 cat_sizes=sizes, other=other)
    if is_pe:
      return VectorizedStrategyResults(bx, bs, pe_aux(bx, bz), categorical=bz)
    if is_multi:   # no trust region -> no aux (acquisitions.py:190-207)
      return VectorizedStrategyResults(bx, bs, {}, categorical=bz)
    _, aux = _score_with_aux(dev, acq, bx, bz if self.n_categorical else None)
    return VectorizedStrategyResults(bx, bs, aux, categorical=bz)


def _score_with_aux(dev, acq: gp.Acquisition, bx: np.ndarray, bz: Optional[np.ndarray]):
  """score_with_aux on the winners (vectorized_base.py:504-526): their scores and, with the trust region, the aux
  arrays of acquisitions.py:190-207.  Returns (scores [count], aux)."""
  out = dev.score(bx, acq, zs=bz, with_aux=True)
  dev.synchronize()
  scores = out['score'].cpu().numpy()
  if not acq.use_trust_region:
    return scores, {}
  aux = {
      'mean': out['mean'].cpu().numpy(), 'stddev': out['stddev'].cpu().numpy(),
      'linf_distance': out['linf_distance'].cpu().numpy(),
      'radius': np.full(len(bx), acq.trust_radius),
  }
  # the acquisition before the trust region, evaluated by the same device epilogue as the scores
  raw = dev.score(bx, dataclasses.replace(acq, use_trust_region=False), zs=bz)
  dev.synchronize()
  aux['raw_acquisition'] = raw['score'].cpu().numpy()
  return scores, aux


@dataclasses.dataclass
class VectorizedOptimizerFactory:
  strategy_factory: Union[VectorizedEagleStrategyFactory, _RandomStrategyFactory] = VectorizedEagleStrategyFactory()
  max_evaluations: int = 75_000
  suggestion_batch_size: int = 25
  use_fori: bool = True  # accepted for API compatibility; the loop always runs on the device

  def __call__(self, converter) -> VectorizedOptimizer:
    return VectorizedOptimizer(self.strategy_factory, converter.n_continuous, converter.n_categorical,
                               self.suggestion_batch_size, self.max_evaluations, tuple(converter.categorical_sizes))


@dataclasses.dataclass
class LBFGSBOptimizer:
  """L-BFGS-B over the continuous features (lbfgsb_optimizer.py:48-230): `random_restarts` uniform initial points
  clipped into `bounds`, each minimised on -score by SciPy's L-BFGS-B (gtol 1e-8, maxls 20, `maxiter`), all restarts
  advancing in lock step (`ard._lockstep`); the `count` lowest final losses win.  Prior features are ignored.  A
  restart whose value or gradient is not finite stops at that point and keeps its value."""

  bounds: tuple                 # ((low, high),) per continuous feature: (0, 1), or (0.5, 0.5) for a fixed one
  random_restarts: int = 25
  maxiter: int = 50
  gtol: float = 1e-8
  maxls: int = 20
  rounds: int = dataclasses.field(default=0, init=False)   # batched evaluations of the last device run
  final_losses: Optional[np.ndarray] = dataclasses.field(default=None, init=False)   # the winners' last -score

  @property
  def n_continuous(self) -> int:
    return len(self.bounds)

  def _check(self, count: int, n_parallel: Optional[int]):
    if n_parallel and count > 1:
      raise ValueError("LBFGSBOptimizer doesn't support batch of batches (count > 1 is disallowed when n_parallel "
                       'is set).')
    if not 1 <= count <= self.random_restarts:
      raise ValueError(f'count must be in [1, random_restarts = {self.random_restarts}], got {count}.')

  def _run(self, batch_fn, q: int, count: int, seed: int) -> np.ndarray:
    """The `count` best final points [count, q * Dc] of the restarts from uniform inits drawn with `seed`."""
    inits = np.random.default_rng(seed).uniform(size=(self.random_restarts, q * self.n_continuous))
    bounds = list(self.bounds) * q
    if ard._setulb is None:  # pylint: disable=protected-access
      raise NotImplementedError("LBFGSBOptimizer needs SciPy's reverse-communication L-BFGS-B routine (the C "
                                'setulb of SciPy >= 1.15), which drives the restarts in lock step.')
    results = ard._lockstep(batch_fn, inits, bounds, stop_nonfinite=True, maxiter=self.maxiter,  # pylint: disable=protected-access
                            gtol=self.gtol, maxls=self.maxls)
    losses = np.asarray([r[1] for r in results])
    order = np.argsort(losses, kind='stable')[:count]    # NaN losses sort last
    self.final_losses = losses[order]
    return np.stack([np.asarray(results[i][0], np.float64) for i in order])

  def optimize_host(self, value_and_grad: Callable, *, count: int = 1, n_parallel: Optional[int] = None,
                    seed: int = 0) -> VectorizedStrategyResults:
    """The optimiser on a host function: `value_and_grad(points) -> (values [B], grads)` with points [B, Dc], or
    [B, n_parallel, Dc] when a value rates a set of n_parallel points (grads have the points' shape).  Returns
    features [count, Dc] and their values, or with n_parallel the best set [n_parallel, Dc] with its value repeated."""
    self._check(count, n_parallel)
    q, dc = int(n_parallel or 1), self.n_continuous

    def shaped(pts):
      return pts.reshape(-1, q, dc) if n_parallel else pts.reshape(-1, dc)

    def batch_fn(idx, pts):
      del idx
      values, grads = value_and_grad(shaped(np.stack(pts)))
      return -np.asarray(values, np.float64), -np.asarray(grads, np.float64).reshape(len(pts), -1)

    best = self._run(batch_fn, q, count, seed)
    values = np.asarray(value_and_grad(shaped(best))[0], np.float64).reshape(-1)
    if n_parallel:
      return VectorizedStrategyResults(best.reshape(q, dc), np.full(q, values[0]), {},
                                       categorical=np.zeros((q, 0), np.int32))
    return VectorizedStrategyResults(best, values, {}, categorical=np.zeros((count, 0), np.int32))

  def __call__(self, dev, acq, *, count: int = 1, prior_features: Optional[np.ndarray] = None,
               prior_categorical: Optional[np.ndarray] = None, seed: int = 0) -> VectorizedStrategyResults:
    """`VectorizedOptimizer.__call__` on a single-metric GP (`gp.DeviceGP` or `gp.EnsembleGP`) and a
    `gp.Acquisition`: every round scores the unfinished restarts with one `score_grad` call.  Rewards and aux are
    those of `dev.score` at the winners, as for the Eagle optimiser."""
    import torch
    del prior_features, prior_categorical
    if not isinstance(acq, gp.Acquisition) or not isinstance(dev, (gp.DeviceGP, gp.EnsembleGP)):
      raise NotImplementedError('LBFGSBOptimizer optimises single-metric acquisitions of one GP or a uniform '
                                f'ensemble, not {type(acq).__name__} on {type(dev).__name__}.')
    self._check(count, None)
    self.rounds = 0

    def batch_fn(idx, pts):
      del idx
      out = dev.score_grad(np.stack(pts), acq)
      with torch.cuda.stream(dev.stream):
        flat = out['_flat'].cpu().numpy()        # score [k] then grad [k, Dc]: one copy per round
      k = len(pts)
      self.rounds += 1
      return -flat[:k], -flat[k:].reshape(k, self.n_continuous)

    bx = self._run(batch_fn, 1, count, seed)
    scores, aux = _score_with_aux(dev, acq, bx, None)
    return VectorizedStrategyResults(bx, scores, aux, categorical=np.zeros((count, 0), np.int32))


@dataclasses.dataclass(frozen=True)
class LBFGSBOptimizerFactory:
  """lbfgsb_optimizer.py:233-270."""

  random_restarts: int = 25
  maxiter: int = 100

  def __call__(self, converter) -> LBFGSBOptimizer:
    if converter.n_categorical > 0:
      raise ValueError("LBFGSBOptimizer doesn't support categorical features.")
    # the scaled specs' bounds (converters/core.py:441): a parameter with low == high maps to 0.5
    bounds = tuple((0.5, 0.5) if s.low == s.high else (0.0, 1.0) for s in converter.continuous_specs)
    return LBFGSBOptimizer(bounds, self.random_restarts, self.maxiter)
