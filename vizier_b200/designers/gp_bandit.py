"""`VizierGPBandit`: the GP-UCB designer, with the GP stack running in libvzgp (CUDA, sm_90a).

Drop-in for vizier/_src/algorithms/designers/gp_bandit.py:88-641 on the single-metric default
path: same constructor keywords, `update` / `suggest` / `predict` / `sample` / `from_problem`,
same metadata keys, same errors for unsupported search spaces.  What runs where:

  host (NumPy, O(N*D))   trials -> scaled features (converters.py), label warping
                         (output_warpers.py), SciPy L-BFGS-B driver (ard.py)
  device (libvzgp)       kernel matrix, Cholesky (+retry), L^-1, alpha, NLL + gradient,
                         posterior mean/variance + UCB + trust region, Eagle / random acquisition
                         optimisation, top-k

`ensemble_size > 1` keeps the E best ARD restarts as a uniform mixture (`gp.EnsembleGP`).
Multi-metric problems use the reference's scalarised UCB (gp_bandit.py:214-242): an independent
multi-task GP (one factor, one alpha per metric) scored by the mean over `num_scalarizations`
hyper-volume scalarisations, without a trust region.
`linear_coef` adds the feature-scaled linear kernel and the constant mean of tuned_gp_models.py:203-245
(general launch sequences: no captured graph, explicit K* for the scoring).
`set_priors` trains a stack of residual GPs, one level per prior study plus the current study on top (gp_bandit.py:289-318;
gp/gp_models.py:91-140, :245-300; gp/transfer_learning.py), scored through `vzgp_score_stack` (`gp.StackedGP`).
`scoring_function_factory` (e.g. `acquisitions.bayesian_scoring_function_factory(lambda d: EI(get_best_labels(d.labels)))`
or `AcquisitionTrustRegion.default_ucb_pi`) selects UCB, LCB, EI, PI or a thresholded pair of those; the device
scoring kernels evaluate it (`acquisitions.lower_acquisition`).  Multi-metric problems keep their scalarised UCB.
`scoring_function_is_parallel=True` with a factory returning `QEI`, `QPI` or `QUCB` suggests one set of `count` points
(gp_bandit.py:496-499): Monte Carlo estimates over each set's joint posterior, scored by `vzgp_score_qsets`
(csrc/score_q.cu) inside the n_parallel Eagle loop or the random strategy (`optimizers.optimize_qsets`).
Not implemented (the reference supports them; SURVEY 8f "next"): parallel acquisitions for multi-metric models or
with priors, other acquisition
functions (MaxValueEntropySearch, Sample, user callables), non-independent multi-task kernels, priors for multi-metric or ensemble models; each raises NotImplementedError
instead of silently doing something else.  Categorical parameters ARE supported
end to end.  `padding_schedule` is accepted and has no numerical effect here: the kernels take
explicit sizes (`n_valid`, Dc, Dk) instead of padded shapes + masks, which is what the reference's
padding-invariance tests (gp_bandit_test.py:302-370) assert of its own masked implementation.
"""

from __future__ import annotations

import copy
import datetime
import json
import random
from typing import Any, Optional, Sequence

import numpy as np

from vizier_b200 import acquisitions as acq_lib
from vizier_b200 import ard
from vizier_b200 import converters
from vizier_b200 import gp
from vizier_b200 import optimizers as vb
from vizier_b200 import output_warpers
from vizier_b200 import profiler
from vizier_b200 import vz

# gp_bandit.py:57
_MAX_NUM_FEASIBLE_VALUES_FOR_TRUST_REGION = 1000

# gp_bandit.py:60-66
default_acquisition_optimizer_factory = vb.VectorizedOptimizerFactory(
    strategy_factory=vb.VectorizedEagleStrategyFactory(eagle_config=vb.EagleStrategyConfig()),
    max_evaluations=75_000,
    suggestion_batch_size=25,
)


def _seed_from(rng: Any) -> int:
  """Accepts an int, a NumPy Generator or a JAX-style uint32[2] key."""
  if rng is None:
    return random.getrandbits(32)
  if isinstance(rng, (int, np.integer)):
    return int(rng)
  if isinstance(rng, np.random.Generator):
    return int(rng.integers(2**62))
  arr = np.asarray(rng).reshape(-1)
  return int(arr[-1]) if arr.size else 0


def _halton(index: int, base: int) -> float:
  f, r = 1.0, 0.0
  while index > 0:
    f /= base
    r += f * (index % base)
    index //= base
  return r


_PRIMES = [2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37, 41, 43, 47, 53, 59, 61, 67, 71, 73, 79, 83, 89, 97,
           101, 103, 107, 109, 113, 127, 131, 137, 139, 149, 151, 157, 163, 167, 173, 179, 181, 191, 193,
           197, 199, 211, 223, 227, 229, 233, 239, 241, 251, 257, 263, 269, 271, 277, 281, 283, 293, 307, 311]


class VizierGPBandit(vz.Designer, vz.Predictor):
  """GP-Bandit designer; see module docstring."""

  def __init__(self, problem, *, acquisition_optimizer_factory: vb.VectorizedOptimizerFactory = default_acquisition_optimizer_factory,
               ard_optimizer: Optional[ard.ScipyLbfgsB] = None, ard_random_restarts: int = ard.DEFAULT_RANDOM_RESTARTS,
               num_seed_trials: int = 1, linear_coef: Optional[float] = None, scoring_function_factory=None,
               scoring_function_is_parallel: bool = False, padding_schedule=None, use_trust_region: bool = True,
               rng: Any = None, ensemble_size: Optional[int] = 1, output_warper=None, num_scalarizations: int = 1000,
               ref_scaling: float = 0.01, multitask_type=None, ucb_coefficient: float = acq_lib.DEFAULT_UCB_COEFFICIENT,
               device: int = 0):
    # gp_bandit.py:179-186
    if problem.search_space.is_conditional:
      raise ValueError(f'{type(self)} does not support conditional search.')
    if problem.search_space.num_parameters() == 0:
      raise ValueError('SearchSpace should contain at least one parameter config.')
    self._n_metrics = len(problem.metric_information)
    if self._n_metrics > 8:
      raise NotImplementedError('at most 8 metrics (libvzgp kMaxMetrics).')
    if self._n_metrics > 1 and multitask_type not in (None, 'INDEPENDENT') and getattr(multitask_type, 'name', '') != 'INDEPENDENT':
      raise NotImplementedError('only the INDEPENDENT multi-task kernel (the default) is implemented.')
    self._linear_coef = float(linear_coef) if linear_coef else None   # Matern + feature-scaled linear kernel, constant mean
    if self._linear_coef and self._n_metrics > 1:
      raise NotImplementedError('linear_coef with several metrics is not implemented.')
    self._ensemble_size = int(ensemble_size or 1)
    if self._ensemble_size < 1 or self._ensemble_size > ard_random_restarts:
      raise ValueError('ensemble_size must be in [1, ard_random_restarts].')
    # gp_bandit.py:496-499: a parallel scoring function scores sets of `count` points (QEI / QPI / QUCB)
    self._parallel = bool(scoring_function_is_parallel)
    if self._parallel and (self._n_metrics > 1 or scoring_function_factory is None):
      raise NotImplementedError('parallel (q-) scoring functions need a single metric and a scoring_function_factory '
                                'returning QEI, QPI or QUCB.')
    if self._n_metrics > 1 and self._ensemble_size > 1:
      raise NotImplementedError('ensembles of multi-metric models are not implemented.')
    del padding_schedule, multitask_type
    self._num_scalarizations = int(num_scalarizations)
    self._ref_scaling = float(ref_scaling)
    self._problem = problem
    self._acquisition_optimizer_factory = acquisition_optimizer_factory
    self._ard_optimizer = ard_optimizer or ard.ScipyLbfgsB()
    self._ard_random_restarts = ard_random_restarts
    self._num_seed_trials = num_seed_trials
    self._use_trust_region = use_trust_region and self._n_metrics == 1   # gp_bandit.py:241
    # gp_bandit.py:206-260: multi-metric problems override the factory with scalarised UCB; a single-metric one is
    # validated now on empty data, so an acquisition the device cannot evaluate fails at construction.
    self._scoring_function_factory = scoring_function_factory if self._n_metrics == 1 else None
    self._ucb_coefficient = ucb_coefficient
    self._metadata_ns = 'oss_gp_bandit'
    self._output_warper = output_warper or output_warpers.create_default_warper()
    self._rng = np.random.default_rng(_seed_from(rng))
    self._converter = converters.TrialToModelInputConverter.from_problem(problem)
    self._acquisition_optimizer = acquisition_optimizer_factory(self._converter)
    if self._scoring_function_factory is not None:
      empty = acq_lib.ModelData(features=None, labels=acq_lib.PaddedArray.as_padded(np.zeros((0, self._n_metrics))))
      acq_lib.check_supported(self._scoring_function(empty).acquisition_fn, parallel=self._parallel)
    # Scalarisation weights are drawn once per designer (gp_bandit.py:217-222: one weights_rng): |N(0,1)|,
    # rows normalised to unit L2 norm (acquisitions.py:585-589).
    self._scal_weights = None
    if self._n_metrics > 1:
      w = np.abs(np.random.default_rng(int(self._rng.integers(2**62))).standard_normal((self._num_scalarizations, self._n_metrics)))
      self._scal_weights = w / np.linalg.norm(w, axis=-1, keepdims=True)
    self._halton_offset = int(self._rng.integers(0, 2**16))
    self._halton_count = 0
    self._trials: list = []
    self._incorporated_trials_count = 0
    self._device_index = device
    self._dev = None                       # gp.DeviceGP, or gp.EnsembleGP when ensemble_size > 1
    self._ard_dev: Optional[gp.DeviceGP] = None
    self._stack: Optional[gp.StackedGP] = None   # transfer learning: prior levels (+ the current study's level on top)
    self._n_prior_levels = 0
    self._last_params = None               # GPHyperParams (or a list of them for an ensemble)

  # ------------------------------------------------------------------ API
  def update(self, completed, all_active=None) -> None:
    """gp_bandit.py:282-287."""
    del all_active
    self._trials.extend(copy.deepcopy(list(completed.trials)))

  def set_priors(self, prior_studies) -> None:
    """gp_bandit.py:289-318: one prior GP per study, stacked in the order received - the first on its study's (warped)
    labels, each further one on the residuals of its study against the stack below (gp/gp_models.py:245-300).  The
    current study's GP is later trained on ITS residuals against the whole prior stack (`_update_gp`).  Each call
    retrains the prior stack from scratch on what it is given."""
    if self._n_metrics != 1 or self._ensemble_size != 1 or self._linear_coef or self._parallel:
      raise NotImplementedError('transfer-learning priors: single-metric, single-model Matern GPs with pointwise '
                                'acquisitions only.')
    if self._stack is not None:
      self._stack.close()
    self._stack = gp.StackedGP(self._device_index)
    for study in prior_studies:
      trials = list(study.trials)
      if not trials:
        continue
      (cont, cat), labels = self._converter.to_xy(trials)
      labels = self._warp_labels(labels)
      self._push_level(cont, cat, labels[:, 0])
    self._n_prior_levels = len(self._stack.levels)
    if self._n_prior_levels == 0:
      self._stack = None
    self._last_params = None               # the top level must be retrained against the new priors
    self._incorporated_trials_count = -1

  def _push_level(self, cont, cat, y):
    """Trains one more level of the stack on the residuals of (cont, cat, y) against the levels below."""
    z = cat if cat.shape[1] else None
    resid = y - self._stack.mean(cont, z)
    level = self._stack.new_level()
    ard_rng = np.random.default_rng(int(self._rng.integers(2**62)))
    best, _ = ard.train_gp(level, cont, resid, z, rng=ard_rng, random_restarts=self._ard_random_restarts,
                           ensemble_size=1, optimizer=self._ard_optimizer)
    level.fit(cont, resid, best[0], z=z)
    self._stack.push(level, cont.shape[0])
    return best[0]

  @classmethod
  def from_problem(cls, problem, seed: Optional[int] = None, **kwargs) -> 'VizierGPBandit':
    """gp_bandit.py:629-641."""
    return cls(problem, rng=random.getrandbits(32) if seed is None else seed, **kwargs)

  # ------------------------------------------------------------------ internals
  def _device(self):
    if self._dev is None:
      if self._ensemble_size > 1:
        self._dev = gp.EnsembleGP(self._device_index, self._ensemble_size)
        self._ard_dev = self._dev.members[0]
      else:
        self._dev = gp.DeviceGP(self._device_index)
        self._ard_dev = self._dev
    return self._dev

  @profiler.record_runtime
  def _generate_seed_trials(self, count: int) -> Sequence[Any]:
    """gp_bandit.py:326-364: search-space centre first, quasi-random afterwards."""
    out = []
    dc, dk = self._converter.n_continuous, self._converter.n_categorical
    if not self._trials:
      params = self._converter.to_parameters(0.5 * np.ones((1, dc)), np.zeros((1, dk), np.int32))[0]
      out.append(vz.TrialSuggestion(params, metadata=vz.Metadata({'seeded': 'center'})))
    with profiler.timeit('quasi_random_sampler_seed_trials'):
      while len(out) < count:
        self._halton_count += 1
        idx = self._halton_offset + self._halton_count
        cont = np.array([[_halton(idx, _PRIMES[j % len(_PRIMES)]) for j in range(dc)]])
        cat = np.array([[min(int(_halton(idx, _PRIMES[(dc + j) % len(_PRIMES)]) * s), s - 1) for j, s in enumerate(self._converter.categorical_sizes)]], np.int32).reshape(1, dk)
        out.append(vz.TrialSuggestion(self._converter.to_parameters(cont, cat)[0]))
    return out

  def _warp_labels(self, labels: np.ndarray) -> np.ndarray:
    return np.concatenate([self._output_warper.warp(labels[:, i:i + 1]) for i in range(labels.shape[1])], axis=-1)

  @profiler.record_runtime
  def _trials_to_data(self, trials):
    (cont, cat), labels = self._converter.to_xy_cached(trials)   # completed trials: owned deep copies
    return cont, cat, self._warp_labels(labels)

  @profiler.record_runtime
  def _update_gp(self, cont, cat, labels) -> gp.DeviceGP:
    """gp_bandit.py:449-479: ARD + precompute, skipped when no new trial arrived."""
    if self._stack is not None:
      # transfer learning (gp_bandit.py:470-476): the current study's GP on the residuals against the prior stack
      if len(self._trials) == self._incorporated_trials_count and self._last_params is not None:
        return self._stack
      self._incorporated_trials_count = len(self._trials)
      self._stack.truncate(self._n_prior_levels)
      self._last_params = self._push_level(cont, cat, labels[:, 0])
      return self._stack
    dev = self._device()
    if len(self._trials) == self._incorporated_trials_count and self._last_params is not None:
      return dev
    self._incorporated_trials_count = len(self._trials)
    ard_rng = np.random.default_rng(int(self._rng.integers(2**62)))
    z = cat if cat.shape[1] else None
    y = labels[:, 0] if self._n_metrics == 1 else labels     # [N] or [N, M]
    best, _ = ard.train_gp(self._ard_dev, cont, y, z, rng=ard_rng, random_restarts=self._ard_random_restarts,
                           ensemble_size=self._ensemble_size, optimizer=self._ard_optimizer, linear_coef=self._linear_coef)
    if self._ensemble_size > 1:
      # the E best restarts become the members of a uniform mixture (gp_models.py:200-223)
      self._last_params = list(best)
      dev.fit(cont, y, self._last_params, z=z)
    else:
      self._last_params = best[0]
      dev.fit(cont, y, self._last_params, z=z)
    return dev

  def _scoring_function(self, data):
    sf = self._scoring_function_factory(
        data, None, self._converter.continuous_feasible_values(_MAX_NUM_FEASIBLE_VALUES_FOR_TRUST_REGION),
        self._use_trust_region)
    if not isinstance(sf, acq_lib.BayesianScoringFunction):
      raise NotImplementedError(f'scoring function {type(sf).__name__} is not implemented on the device '
                                '(use acquisitions.bayesian_scoring_function_factory)')
    return sf

  def _acquisition(self, n_obs: int, labels: Optional[np.ndarray] = None, features=None):
    if self._n_metrics > 1:
      # gp_bandit.py:217-239: HV scalarisation around the reference point of the (warped) labels, floored
      # at the best scalarised value observed so far
      ref = acq_lib.hv_reference_point(labels, self._ref_scaling)
      best = acq_lib.hv_scalarize(labels, self._scal_weights, ref).max(axis=-1)
      return gp.ScalarizedUcbAcquisition(self._scal_weights, ref, best, self._ucb_coefficient)
    acq = acq_lib.make_acquisition(
        n_obs, self._converter.continuous_feasible_values(_MAX_NUM_FEASIBLE_VALUES_FOR_TRUST_REGION),
        self._converter.n_continuous, self._converter.n_categorical, use_trust_region=self._use_trust_region,
        ucb_coefficient=self._ucb_coefficient)
    if self._scoring_function_factory is not None:
      # gp_bandit.py:497-505: the factory sees the (warped) labels of this suggest
      data = acq_lib.ModelData(features=features, labels=acq_lib.PaddedArray.as_padded(labels))
      acq.acq_fn = acq_lib.lower_acquisition(self._scoring_function(data).acquisition_fn)
    return acq

  @profiler.record_runtime
  def _optimize_acquisition(self, dev: gp.DeviceGP, acq: gp.Acquisition, count: int, features=None):
    """gp_bandit.py:482-521 + vectorized_base.best_candidates_to_trials (:591-651)."""
    prior = converters.trials_to_sorted_features(self._trials, self._converter, features)
    seed = int(self._rng.integers(2**62))
    res = self._acquisition_optimizer(dev, acq, count=count, prior_features=None if prior is None else prior[0],
                                      prior_categorical=None if prior is None else prior[1], seed=seed)
    order = np.argsort(-res.rewards, kind='stable')
    return [self._result_trial(dev, res, ind) for ind in order]

  def _result_trial(self, dev, res: vb.VectorizedStrategyResults, ind: int):
    """Row `ind` of the optimiser's result as a completed trial carrying its acquisition value and aux arrays."""
    params = self._converter.to_parameters(
        res.features[ind:ind + 1], None if res.categorical is None else res.categorical[ind:ind + 1])[0]
    trial = vz.Trial(parameters=params)
    md = trial.metadata.ns('devinfo')
    aux = {k: float(v[ind]) for k, v in res.aux.items()}
    md['acquisition_optimization'] = json.dumps({'acquisition': float(res.rewards[ind])} | aux)
    failed_fit = any(getattr(m, 'cholesky_failed', False) for m in getattr(dev, 'members', [dev]))
    if failed_fit or np.isnan([res.rewards[ind], *aux.values()]).any():
      md['acquisition_optimization_warning'] = (
          'NaNs encountered in acquisition optimization. See the "acquisition_optimization" field in the '
          'metadata for more details.')
    trial.complete(vz.Measurement({'acquisition': float(res.rewards[ind])}))
    return trial

  @profiler.record_runtime
  def _optimize_parallel_acquisition(self, dev, count: int, labels: np.ndarray, features):
    """gp_bandit.py:482-521 with a parallel scoring function: n_parallel = count, count = 1.  The best set's q points
    become q trials, each carrying the set's acquisition value (vectorized_base.py:591-651)."""
    prior = converters.trials_to_sorted_features(self._trials, self._converter, features)
    seed = int(self._rng.integers(2**62))
    acq_seed = int(self._rng.integers(2**62))   # one acquisition seed per optimiser run (vectorized_base.py:382-404)
    data = acq_lib.ModelData(features=features, labels=acq_lib.PaddedArray.as_padded(labels))
    sf = self._scoring_function(data)
    region = acq_lib.make_acquisition(
        labels.shape[0], self._converter.continuous_feasible_values(_MAX_NUM_FEASIBLE_VALUES_FOR_TRUST_REGION),
        self._converter.n_continuous, self._converter.n_categorical, use_trust_region=self._use_trust_region)
    qacq = acq_lib.lower_parallel_acquisition(sf.acquisition_fn, use_trust_region=region.use_trust_region,
                                              trust_radius=region.trust_radius, tr_dim_mask=region.tr_dim_mask)
    res = self._acquisition_optimizer.optimize_qsets(
        dev, qacq, n_parallel=count, prior_features=None if prior is None else prior[0],
        prior_categorical=None if prior is None else prior[1], seed=seed, acq_seed=acq_seed)
    return [self._result_trial(dev, res, ind) for ind in range(count)]

  # ------------------------------------------------------------------ suggest / predict / sample
  @profiler.record_runtime
  def suggest(self, count: Optional[int] = 1) -> Sequence[Any]:
    """gp_bandit.py:523-559."""
    count = count or 1   # Designer.suggest(count=None) means "as many as you like": one (abstractions.py:118-131)
    if len(self._trials) < self._num_seed_trials:
      return self._generate_seed_trials(count)
    start = datetime.datetime.now()
    cont, cat, labels = self._trials_to_data(self._trials)
    dev = self._update_gp(cont, cat, labels)
    if self._parallel:
      best = self._optimize_parallel_acquisition(dev, count, labels, (cont, cat))
    else:
      acq = self._acquisition(cont.shape[0], labels, features=(cont, cat))
      best = self._optimize_acquisition(dev, acq, count, features=(cont, cat))
    out = []
    for t in best:
      t.metadata.ns(self._metadata_ns).ns('devinfo')['time_spent'] = f'{datetime.datetime.now() - start}'
      out.append(vz.TrialSuggestion(parameters=t.parameters, metadata=t.metadata))
    return out

  @profiler.record_runtime
  def sample(self, trials: Sequence[Any], rng: Any = None, num_samples: int = 1000) -> np.ndarray:
    """gp_bandit.py:561-602: unwarped joint posterior samples, shape (num_samples, num_trials)."""
    if not trials:
      return np.zeros((num_samples, 0))
    cont, cat, labels = self._trials_to_data(self._trials)
    dev = self._update_gp(cont, cat, labels)
    xs, zs = self._converter.to_features(trials)
    xs = np.nan_to_num(xs, nan=0.0)
    g = np.random.default_rng(_seed_from(rng) if rng is not None else 0)
    zq = zs if zs.shape[1] else None
    if self._n_metrics > 1:
      return self._sample_multi(dev, xs, zq, g, num_samples)
    if self._stack is not None:
      # the combined prediction is a diagonal normal (gp/transfer_learning.py:150-152)
      out = dev.score(xs, gp.Acquisition(0.0, False, 1.0), zs=zq, with_aux=True)
      dev.synchronize()
      mean, sd = out['mean'].cpu().numpy(), out['stddev'].cpu().numpy()
      samples = mean[None, :] + g.standard_normal((num_samples, mean.shape[0])) * sd[None, :]
      return self._output_warper.unwarp(samples.reshape(-1, 1)).reshape(samples.shape)
    comps = dev.posterior(xs, zq, add_noise=True) if self._ensemble_size > 1 else [dev.posterior(xs, zq, add_noise=True)]
    # Cholesky of each (small) posterior covariance on the device as well; the retry adds a tiny
    # jitter only if round-off made it indefinite.
    factors = []
    for mean, cov in comps:
      chol, _, _ = self._ard_dev.cholesky_retry(cov, jitter=1e-10, max_iters=8)
      factors.append((mean.cpu().numpy(), chol.cpu().numpy()))
    m = factors[0][0].shape[0]
    normals = g.standard_normal((num_samples, m))
    # equal-weight mixture: every sample is a joint draw from one uniformly chosen member
    member = g.integers(0, len(factors), size=num_samples) if len(factors) > 1 else np.zeros(num_samples, int)
    samples = np.stack([factors[e][0] + normals[i] @ factors[e][1].T for i, e in enumerate(member)])
    # one vectorised unwarp of all num_samples x num_trials values (the warpers act element-wise)
    return self._output_warper.unwarp(samples.reshape(-1, 1)).reshape(samples.shape)

  def _sample_multi(self, dev, xs, zq, g, num_samples: int) -> np.ndarray:
    """Independent multi-task GP: the metrics share the posterior covariance and differ in the mean.
    Returns unwarped samples [num_samples, num_trials, num_metrics]."""
    mean, cov = dev.posterior(xs, zq, add_noise=True)          # mean [M, n]
    chol, _, _ = self._ard_dev.cholesky_retry(cov, jitter=1e-10, max_iters=8)
    mean, chol = mean.cpu().numpy(), chol.cpu().numpy()
    out = np.empty((num_samples, mean.shape[1], self._n_metrics))
    for m in range(self._n_metrics):
      z = g.standard_normal((num_samples, mean.shape[1]))
      warped = mean[m][None, :] + z @ chol.T
      out[:, :, m] = self._output_warper.unwarp(warped.reshape(-1, 1)).reshape(num_samples, -1)
    return out

  @profiler.record_runtime
  def predict(self, trials: Sequence[Any], rng: Any = None, num_samples: Optional[int] = 1000):
    """gp_bandit.py:604-627: empirical mean / stddev of unwarped samples."""
    s = self.sample(trials, rng, num_samples or 1000)
    return vz.Prediction(mean=np.mean(s, axis=0), stddev=np.std(s, axis=0))
