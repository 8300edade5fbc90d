"""`VizierGPUCBPEBandit`: GP-UCB with Pure Exploration, the Vizier service's DEFAULT algorithm.

Mirrors vizier/_src/algorithms/designers/gp_ucb_pe.py:609-1445 on the single-metric default
configuration (`UCBPEConfig()` with `optimize_set_acquisition_for_exploration=False`):

  * ARD: 4 random + 1 fixed initialisation (:828-838), L-BFGS-B maxiter=500, tol=1e-5 (:596-604), or, with
    `ard_optimizer=ard.OptaxTrain(ard.adam(lr), epochs=T)`, Adam in SoftClip-unconstrained coordinates from the same
    initial points (one kernel launch for single-metric studies of up to 64 trials without `mixes_linear_kernel`, one
    device evaluation per epoch otherwise; ard.py);
  * model A = GP on the completed trials (mean, stddev); model B = same hyper-parameters on
    completed + pending trials (stddev_from_all; noise forced to 1e-10 when the signal-to-noise
    ratio is low, :996-1004);
  * per suggestion: UCB (mean_A + 1.8 stddev_B) when trials completed after the newest active
    trial was created, else PE (stddev_B + 10 min(mean_A + 0.5 stddev_A - threshold, 0)), with the
    random overwrites of :1017-1046; strict trust region over completed + initially active trials;
  * batches: every suggestion joins the pending set before the next one is optimised (:1429-1445);
  * acquisition optimiser: Eagle with the tuned UCB-PE config and RANDOM force normalisation
    (:678-698).

Everything numeric runs in libvzgp (two handles, or two ensembles, on one stream, `vzgp_score_pe`,
`vzgp_eagle_run_pe`); `sample` / `predict` (:1262-1354) draw from the device-computed joint posterior
like `VizierGPBandit`.  `prior_acquisition` (a callable on NumPy features) is added to both acquisitions through the
host-stepped Eagle loop (`gp.SteppedEagle`); `optimize_set_acquisition_for_exploration=True` optimises the rest of a
batch as ONE set for the set-PE acquisition (`vzgp_score_set_pe`, the optimiser's n_parallel form; continuous search
spaces with count <= 16 and count * Dc <= 1024); `mixes_linear_kernel=True` uses the Matern + linear kernel with a constant mean
(`linear_coef = 1`, libvzgp's general scoring path).

Multi-metric studies (up to 8 metrics, gp_ucb_pe.py:344-381, :434-492, :701-722, :917-942) use one default output
warper per metric and model A is the independent multi-task GP (one factor, one alpha per metric; ARD on the summed
losses).  UCB is the hyper-volume scalarisation of mean_A,m + 1.8 stddev_B over 1000 weight rows drawn afresh for
each UCB suggestion, floored at the best scalarised label and averaged; PE is stddev_B plus the per-metric penalties
(thresholds per metric) combined by `multimetric_promising_region_penalty_type` (AVERAGE / UNION / INTERSECTION).
The strict trust region stays on.  Both run in `vzgp_score_pe_multi` / `vzgp_eagle_run_pe_multi`; `sample` returns
[num_samples, n, num_metrics] and the prediction metadata holds per-metric vectors.

Ensembles (`ensemble_size = E > 1`, single metric; stochastic_process_model.py:835-878): the E best of the 1 fixed +
`ard_random_restarts` ARD initialisations (the first E initial points before any trial completes) give E members of
model A (completed trials) and E of model B (completed + pending trials, the real labels on completed rows and 0 on
pending rows); every prediction is the members' equal-weight mixture (two-pass variance), UCB / PE / the threshold
are taken on the mixtures and model B's noise is forced to 1e-10 when every member's signal-to-noise ratio is low.
Scoring and Eagle run in `vzgp_score_pe_ensemble` / `vzgp_eagle_run_pe_ensemble`; `sample` draws each joint sample
from one uniformly chosen member.  The set-PE batch path raises ValueError with E > 1 (the reference cannot run it:
its `if noise_is_high:` meets a per-member array there).

Not implemented: ensembles with several metrics (NotImplementedError); with several metrics also
`mixes_linear_kernel`, task kernels other than INDEPENDENT (NotImplementedError) and
`optimize_set_acquisition_for_exploration` (ValueError, as in the reference).
"""

from __future__ import annotations

import copy
import dataclasses
import datetime
import enum
import json
import random
from typing import Any, Optional, Sequence

import numpy as np

from vizier_b200 import _lib
from vizier_b200 import acquisitions as acq_lib
from vizier_b200 import ard
from vizier_b200 import converters
from vizier_b200 import gp
from vizier_b200 import optimizers as vb
from vizier_b200 import output_warpers
from vizier_b200 import profiler
from vizier_b200 import vz
from vizier_b200.designers import gp_bandit as _gpb

_MAX_NUM_FEASIBLE_VALUES_FOR_TRUST_REGION = 1000


class MultimetricPromisingRegionPenaltyType(enum.Enum):
  """gp_ucb_pe.py:63-78: how the PE penalties of the metrics' promising regions combine."""

  UNION = 'union'                  # max over the metrics: penalised outside the union of the regions
  INTERSECTION = 'intersection'    # min over the metrics: penalised outside any of the regions
  AVERAGE = 'average'              # mean over the metrics


_REGION_PENALTY_CODE = {
    MultimetricPromisingRegionPenaltyType.AVERAGE: _lib.REGION_AVERAGE,
    MultimetricPromisingRegionPenaltyType.UNION: _lib.REGION_UNION,
    MultimetricPromisingRegionPenaltyType.INTERSECTION: _lib.REGION_INTERSECTION,
}
_NUM_SCALARIZATIONS = 1000   # UCBScoreFunction's default (gp_ucb_pe.py:282-340)


@dataclasses.dataclass(frozen=True)
class UCBPEConfig:
  """gp_ucb_pe.py:80-135.  `multitask_type`: only the INDEPENDENT multi-task kernel (a name or an enum member with
  that name) is implemented for several metrics."""

  ucb_coefficient: float = 1.8
  explore_region_ucb_coefficient: float = 0.5
  cb_violation_penalty_coefficient: float = 10.0
  ucb_overwrite_probability: float = 0.25
  pe_overwrite_probability: float = 0.1
  pe_overwrite_probability_in_high_noise: float = 0.7
  signal_to_noise_threshold: float = 0.7
  optimize_set_acquisition_for_exploration: bool = False
  multimetric_promising_region_penalty_type: MultimetricPromisingRegionPenaltyType = (
      MultimetricPromisingRegionPenaltyType.AVERAGE)
  multitask_type: Any = 'INDEPENDENT'


# gp_ucb_pe.py:678-698
default_eagle_config = vb.EagleStrategyConfig(
    visibility=3.6782451729470043,
    gravity=3.028167342024462,
    negative_gravity=0.03036267153343141,
    perturbation=0.23337470891647027,
    categorical_perturbation_factor=9.587350648631066,
    pure_categorical_perturbation_factor=28.636337967676518,
    prob_same_category_without_perturbation=0.9744882009359648,
    perturbation_lower_bound=7.376256294543107e-4,
    penalize_factor=0.7817632796830948,
    pool_size_exponent=2.0494446726436744,
    mutate_normalization_type=1,  # RANDOM
    normalization_scale=1.9893618760239418,
    prior_trials_pool_pct=0.423499384081575,
)
default_acquisition_optimizer_factory = vb.VectorizedOptimizerFactory(
    strategy_factory=vb.VectorizedEagleStrategyFactory(eagle_config=default_eagle_config),
    max_evaluations=75000,
    suggestion_batch_size=25,
)


def default_ard_optimizer() -> ard.ScipyLbfgsB:
  """gp_ucb_pe.py:596-604 (the 40-minute wall-clock guard is not needed at GPU speed)."""
  return ard.ScipyLbfgsB(ard.LbfgsBOptions(num_line_search_steps=20, tol=1e-5, maxiter=500))


def _json_value(v):
  """A scalar, or the per-metric vector of a multi-metric aux entry, as a JSON value."""
  a = np.asarray(v, np.float64)
  return float(a) if a.ndim == 0 else [float(x) for x in a]


def _has_new_completed_trials(completed: Sequence[Any], active: Sequence[Any]) -> bool:
  """gp_ucb_pe.py:142-172."""
  if not completed:
    return False
  if not active:
    return True
  done = [t.completion_time for t in completed]
  made = [t.creation_time for t in active]
  if not all(done):
    raise ValueError('All completed trials must have completion times.')
  if not all(made):
    raise ValueError('All active trials must have creation times.')
  return max(done) > max(made)


class VizierGPUCBPEBandit(vz.Designer, vz.Predictor):
  """GP-UCB-PE designer; see module docstring."""

  def __init__(self, problem, *, acquisition_optimizer_factory: vb.VectorizedOptimizerFactory = default_acquisition_optimizer_factory,
               ensemble_size: Optional[int] = 1, ard_optimizer=None,
               ard_random_restarts: int = 4, use_trust_region: bool = True, num_seed_trials: int = 1,
               config: UCBPEConfig = UCBPEConfig(), rng: Any = None, clear_jax_cache: bool = False,
               padding_schedule=None, prior_acquisition=None, mixes_linear_kernel: bool = False,
               metadata_ns: str = 'google_gp_ucb_pe_bandit', device: int = 0):
    if problem.search_space.is_conditional:
      raise ValueError(f'{type(self)} does not support conditional search.')
    if isinstance(acquisition_optimizer_factory, vb.LBFGSBOptimizerFactory):
      raise NotImplementedError('GP-UCB-PE with the L-BFGS-B acquisition optimiser is not implemented.')
    self._n_metrics = len(problem.metric_information)
    if self._n_metrics > 1:
      # gp_ucb_pe.py:701-722
      if config.optimize_set_acquisition_for_exploration:
        raise ValueError(f'{type(self)} works with exactly one metric when '
                         '`optimize_set_acquisition_for_exploration` is enabled.')
      if self._n_metrics > 8:
        raise NotImplementedError('at most 8 metrics (libvzgp kMaxMetrics).')
      mt = config.multitask_type
      if mt not in (None, 'INDEPENDENT') and getattr(mt, 'name', '') != 'INDEPENDENT':
        raise NotImplementedError('only the INDEPENDENT multi-task kernel (the default) is implemented.')
      if mixes_linear_kernel:
        raise NotImplementedError('mixes_linear_kernel with several metrics is not implemented.')
      if not isinstance(config.multimetric_promising_region_penalty_type, MultimetricPromisingRegionPenaltyType):
        raise ValueError('Unsupported multimetric promising region penalty type: '
                         f'{config.multimetric_promising_region_penalty_type}')
    self._ensemble_size = int(ensemble_size or 1)
    if self._n_metrics > 1 and self._ensemble_size != 1:
      raise NotImplementedError('ensembles of multi-metric models are not implemented for GP-UCB-PE.')
    if self._ensemble_size < 1 or self._ensemble_size > ard_random_restarts + 1:
      raise ValueError('ensemble_size must be in [1, ard_random_restarts + 1].')
    # mixes_linear_kernel: the Matern + feature-scaled linear kernel with a constant mean, linear_coef = 1
    # (gp_ucb_pe.py:805-809, :844-853; tuned_gp_models.py:203-245)
    self._linear_coef = 1.0 if mixes_linear_kernel else None
    del clear_jax_cache, padding_schedule
    # prior_acquisition(continuous [m, Dc], categorical [m, Dk]) -> [m]: added to the UCB / PE acquisition
    # (gp_ucb_pe.py:286-381, :487-490); NumPy arrays instead of the reference's JAX ModelInput.
    self._prior_acquisition = prior_acquisition
    self._problem = problem
    self._acquisition_optimizer_factory = acquisition_optimizer_factory
    self._ard_optimizer = ard_optimizer or default_ard_optimizer()
    self._ard_random_restarts = ard_random_restarts
    self._use_trust_region = use_trust_region
    self._num_seed_trials = num_seed_trials
    self._config = config
    self._metadata_ns = metadata_ns
    self._rng = np.random.default_rng(_gpb._seed_from(rng))
    self._converter = converters.TrialToModelInputConverter.from_problem(problem)
    self._halton_offset = int(self._rng.integers(0, 2**16))
    self._halton_count = 0
    self._all_completed_trials: list = []
    self._all_active_trials: Sequence[Any] = []
    self._output_warper = None
    self._output_warpers: list = []        # one per metric (gp_ucb_pe.py:917-942)
    self._device_index = device
    self._dev_a = None    # gp.DeviceGP, or gp.EnsembleGP when ensemble_size > 1
    self._dev_b = None

  # ------------------------------------------------------------------ API
  def update(self, completed, all_active) -> None:
    """gp_ucb_pe.py:740-744."""
    self._all_completed_trials.extend(copy.deepcopy(list(completed.trials)))
    self._all_active_trials = copy.deepcopy(list(all_active.trials))

  @classmethod
  def from_problem(cls, problem, seed: Optional[int] = None, **kwargs) -> 'VizierGPUCBPEBandit':
    return cls(problem, rng=random.getrandbits(32) if seed is None else seed, **kwargs)

  # ------------------------------------------------------------------ internals
  def _devices(self):
    if self._dev_a is None:
      if self._ensemble_size > 1:
        self._dev_a = gp.EnsembleGP(self._device_index, self._ensemble_size)
        self._dev_b = gp.EnsembleGP(self._device_index, self._ensemble_size, stream=self._dev_a.stream)
      else:
        self._dev_a = gp.DeviceGP(self._device_index)
        self._dev_b = gp.DeviceGP(self._device_index, stream=self._dev_a.stream)  # same stream: ordered launches
    return self._dev_a, self._dev_b

  def _ard_dev(self) -> gp.DeviceGP:
    dev_a, _ = self._devices()
    return dev_a.members[0] if self._ensemble_size > 1 else dev_a

  def _params_out(self, vectors, dc: int, dk: int):
    """GPHyperParams of the kept ARD results: one, or the list of E ensemble members."""
    ps = [gp.GPHyperParams.from_vector(v, dc, dk, self._linear_coef) for v in vectors[:self._ensemble_size]]
    return ps[0] if self._ensemble_size == 1 else ps

  def _noise_is_high(self, params) -> bool:
    """gp_ucb_pe.py:1018-1021: the signal-to-noise ratio is below the threshold (for every ensemble member)."""
    members = params if isinstance(params, list) else [params]
    return all(p.signal_variance / max(p.observation_noise_variance, 1e-12) < self._config.signal_to_noise_threshold
               for p in members)

  def _generate_seed_trials(self, count: int):
    """gp_ucb_pe.py:750-787: centre first (if nothing exists yet), quasi-random afterwards."""
    out = []
    dc, dk = self._converter.n_continuous, self._converter.n_categorical
    if not self._all_completed_trials and not self._all_active_trials:
      params = self._converter.to_parameters(0.5 * np.ones((1, dc)), np.zeros((1, dk), np.int32))[0]
      out.append(vz.TrialSuggestion(params, metadata=vz.Metadata({'seeded': 'center'})))
    while len(out) < count:
      self._halton_count += 1
      idx = self._halton_offset + self._halton_count
      cont = np.array([[_gpb._halton(idx, _gpb._PRIMES[j % len(_gpb._PRIMES)]) for j in range(dc)]])
      cat = np.array([[min(int(_gpb._halton(idx, _gpb._PRIMES[(dc + j) % len(_gpb._PRIMES)]) * s), s - 1)
                       for j, s in enumerate(self._converter.categorical_sizes)]], np.int32).reshape(1, dk)
      out.append(vz.TrialSuggestion(self._converter.to_parameters(cont, cat)[0]))
    return out

  @profiler.record_runtime
  def _trials_to_data(self, trials):
    """gp_ucb_pe.py:917-942: a fresh default warper per metric and call; labels [N, n_metrics]."""
    (cont, cat), labels = self._converter.to_xy_cached(trials)   # completed trials: owned deep copies
    self._output_warpers = [output_warpers.create_default_warper() for _ in range(self._n_metrics)]
    self._output_warper = self._output_warpers[0]
    if not labels.shape[0]:
      return cont, cat, labels[:, :self._n_metrics]
    warped = [w.warp(labels[:, i:i + 1]) for i, w in enumerate(self._output_warpers)]
    return cont, cat, warped[0] if self._n_metrics == 1 else np.concatenate(warped, axis=-1)

  @profiler.record_runtime
  def _build_gp_model_and_optimize_parameters(self, cont, cat, labels):
    """gp_ucb_pe.py:789-894: one fixed + `ard_random_restarts` random initialisations; the best one, or the E best
    (a list) for an ensemble (:867-878)."""
    dc, dk = cont.shape[1], cat.shape[1]
    rng = np.random.default_rng(int(self._rng.integers(2**62)))
    lin = self._linear_coef
    random_inits = ard.log_uniform_init(rng, dc, dk, self._ard_random_restarts, linear=bool(lin))
    fixed = gp.GPHyperParams(0.039, np.ones(dc), 0.0039, np.ones(dk), linear_coef=lin, linear_slope_amplitude=0.0,
                             linear_shift=0.0, mean_constant=0.0).to_vector()[None, :]    # :833-853
    inits = np.concatenate([fixed, random_inits], axis=0)
    if cont.shape[0] == 0:
      # no completed trial yet: the dummy loss makes every loss equal, so the optimiser returns its first initial
      # point(s)
      return self._params_out(inits, dc, dk)
    dev_a = self._ard_dev()
    import torch  # device-memory handles only
    xt = torch.from_numpy(np.ascontiguousarray(cont)).to(dev_a.device)
    # [N], or [N, n_metrics] for the independent multi-task GP (the losses sum over the metrics)
    y = labels[:, 0] if self._n_metrics == 1 else labels
    yt = torch.from_numpy(np.ascontiguousarray(y)).to(dev_a.device)
    zt = torch.from_numpy(np.ascontiguousarray(cat)).to(dev_a.device) if dk else None
    lo, hi = gp.param_bounds(dc, dk, bool(lin))
    if lin:
      inits = np.clip(inits, lo, hi)     # the fixed slope 0 sits below its lower bound: L-BFGS-B starts from the projection
    if isinstance(self._ard_optimizer, ard.OptaxTrain):
      try:
        best, _ = self._ard_optimizer.fit(dev_a, xt, yt, zt, inits, lo, hi, best_n=self._ensemble_size, linear_coef=lin)
      finally:
        dev_a.set_int('dataflow_ctas', 0)
      return self._params_out(best, dc, dk)

    # all initial points advance in lock step, one CUDA-graph launch per round (ard.batch_loss_function); small
    # studies (one fused kernel per evaluation) keep one host thread per point
    if not lin and ard.BATCHED_ARD and ard._setulb is not None and xt.shape[0] > 64 and inits.shape[0] <= 16:   # pylint: disable=protected-access
      fns = ard.batch_loss_function(dev_a, xt, yt, zt, inits.shape[0])
    else:
      fns = ard.loss_functions(dev_a, xt, yt, zt, dc, dk, workers=min(ard.MAX_ARD_WORKERS, inits.shape[0]), linear_coef=lin)
    try:
      best, _ = self._ard_optimizer(inits, fns, list(zip(lo, hi)), best_n=self._ensemble_size)
    finally:
      dev_a.set_int('dataflow_ctas', 0)
    return self._params_out(best, dc, dk)

  def _fit_all_features(self, params, cont, cat, labels, pend_c, pend_z, noise_is_high: bool):
    """_get_predictive_all_features (:944-1004): model B on completed + pending trials, the real labels on completed
    rows and 0 on pending rows.  A single model's stddev does not depend on the labels, so a multi-metric study fits B
    as one metric on zeros; an ensemble's mixture stddev does (the spread of the members' means)."""
    _, dev_b = self._devices()
    xc = np.concatenate([cont, pend_c], axis=0)
    xz = np.concatenate([cat, pend_z], axis=0)
    if self._n_metrics == 1:
      y = np.concatenate([labels[:, 0], np.zeros(pend_c.shape[0])])
    else:
      y = np.zeros(xc.shape[0])
    p = params
    if noise_is_high:
      p = ([dataclasses.replace(q, observation_noise_variance=1e-10) for q in params] if isinstance(params, list)
           else dataclasses.replace(params, observation_noise_variance=1e-10))
    dev_b.fit(xc, y, p, z=xz if xz.shape[1] else None)
    return xc, xz

  def _fit_labels(self, labels):
    """Labels for DeviceGP.fit: [N] for one metric, [N, n_metrics] for the independent multi-task GP."""
    return labels[:, 0] if self._n_metrics == 1 else labels

  def _prediction_str(self, v) -> str:
    """A prediction metadata value: repr of the float, or np.array2string of the per-metric vector (:1134-1144; the
    stddev shared by the metrics of the independent multi-task GP is repeated per metric)."""
    if self._n_metrics == 1:
      return repr(float(v))
    return np.array2string(np.broadcast_to(np.asarray(v, np.float64), (self._n_metrics,)), separator=',')

  def _multi_metric_acquisition(self, use_ucb: bool, labels, xc_all, xz_all, mask, radius, n_tr_rows):
    """UCBScoreFunction / PEScoreFunction of a multi-metric study (gp_ucb_pe.py:282-381, :434-492)."""
    cfg = self._config
    dev_a, _ = self._devices()
    nm = self._n_metrics
    common = dict(n_metrics=nm, ucb_coefficient=cfg.ucb_coefficient, explore_coefficient=cfg.explore_region_ucb_coefficient,
                  penalty_coefficient=cfg.cb_violation_penalty_coefficient, use_trust_region=self._use_trust_region,
                  trust_radius=radius, tr_dim_mask=mask, tr_rows=n_tr_rows)
    if use_ucb:
      # fresh HV scalarisation weights per UCB suggestion (:1057; acquisitions.create_hv_scalarization): |N(0, 1)|,
      # rows of unit L2 norm, the reference point of the warped labels, floored at the best scalarised label
      g = np.random.default_rng(int(self._rng.integers(2**62)))
      w = np.abs(g.standard_normal((_NUM_SCALARIZATIONS, nm)))
      w = w / np.linalg.norm(w, axis=-1, keepdims=True)
      ref = acq_lib.hv_reference_point(labels, 0.01)
      best = acq_lib.hv_scalarize(labels, w, ref).max(axis=-1)
      sc = gp.ScalarizedUcbAcquisition(w, ref, best, cfg.ucb_coefficient)
      return gp.UcbPeMultiAcquisition(mode=0, scalarization=sc, **common)
    # _compute_ucb_threshold (:175-218) per metric: mean_m of A at B's feature with the largest UCB_A of metric m.  The
    # means and the shared stddev come from the scalarised scorer's aux outputs (its score is not used).
    probe = gp.ScalarizedUcbAcquisition(np.full((1, nm), 1.0 / np.sqrt(nm)), np.zeros(nm), None, 0.0)
    out = dev_a.score_multi(xc_all, probe, zs=xz_all, with_aux=True)
    dev_a.synchronize()
    mu = out['mean'].cpu().numpy()
    sd = out['stddev'].cpu().numpy()
    best_idx = np.argmax(mu + cfg.ucb_coefficient * sd[None, :], axis=1)
    thresholds = mu[np.arange(nm), best_idx]
    return gp.UcbPeMultiAcquisition(
        mode=1, thresholds=thresholds, region_penalty=_REGION_PENALTY_CODE[cfg.multimetric_promising_region_penalty_type],
        **common)

  def _ucb_threshold(self, xc_all, xz_all) -> float:
    """_compute_ucb_threshold (:175-218): mean of A at B's feature with the largest UCB_A; an ensemble takes the mixture
    of A's members, which score_pe reports as its aux."""
    cfg = self._config
    dev_a, dev_b = self._devices()
    if self._ensemble_size > 1:
      out = dev_a.score_pe(dev_b, xc_all, gp.UcbPeAcquisition(use_trust_region=False), zs=xz_all)
    else:
      out = dev_a.score(xc_all, gp.Acquisition(cfg.ucb_coefficient, False, 1.0), zs=xz_all, with_aux=True)
    dev_a.synchronize()
    mu = out['mean'].cpu().numpy(); sd = out['stddev'].cpu().numpy()
    return float(mu[int(np.argmax(mu + cfg.ucb_coefficient * sd))])

  @profiler.record_runtime
  def _suggest_one(self, active_trials, cont, cat, labels, params, mask, radius, n_tr_rows):
    """gp_ucb_pe.py:1006-1155."""
    start = datetime.datetime.now()
    cfg = self._config
    dev_a, dev_b = self._devices()
    noise_is_high = self._noise_is_high(params)
    pe_overwrite = cfg.pe_overwrite_probability_in_high_noise if noise_is_high else cfg.pe_overwrite_probability
    u = float(self._rng.uniform())
    if _has_new_completed_trials(self._all_completed_trials, active_trials):
      use_ucb = not (u < pe_overwrite)
    else:
      use_ucb = len(self._all_completed_trials) > 0 and (u < cfg.ucb_overwrite_probability)

    pend_c, pend_z = self._converter.to_features(active_trials)
    pend_c = np.nan_to_num(pend_c, nan=0.0)
    has_model = cont.shape[0] + pend_c.shape[0] > 0
    xc_all, xz_all = self._fit_all_features(params, cont, cat, labels, pend_c, pend_z, noise_is_high) if has_model else (cont, cat)
    dk = cat.shape[1]
    if self._n_metrics > 1:
      pe = self._multi_metric_acquisition(use_ucb, labels, xc_all, xz_all if dk else None, mask, radius, n_tr_rows)
    else:
      threshold = 0.0
      if not use_ucb and cont.shape[0] > 0:
        threshold = self._ucb_threshold(xc_all, xz_all if dk else None)
      pe = gp.UcbPeAcquisition(
          mode=0 if use_ucb else 1, ucb_coefficient=cfg.ucb_coefficient,
          explore_coefficient=cfg.explore_region_ucb_coefficient,
          penalty_coefficient=cfg.cb_violation_penalty_coefficient, threshold=threshold,
          use_trust_region=self._use_trust_region, trust_radius=radius, tr_dim_mask=mask, tr_rows=n_tr_rows)
    optimizer = self._acquisition_optimizer_factory(self._converter)
    prior = converters.trials_to_sorted_features(self._all_completed_trials, self._converter, (cont, cat))
    seed = int(self._rng.integers(2**62))
    res = optimizer(dev_a, pe, count=1, prior_features=None if prior is None else prior[0],
                    prior_categorical=None if prior is None else prior[1], seed=seed, other=dev_b,
                    prior_acquisition=self._prior_acquisition)
    params_dict = self._converter.to_parameters(res.features[0:1], None if res.categorical is None else res.categorical[0:1])[0]
    md = vz.Metadata()
    md.ns('devinfo')['acquisition_optimization'] = json.dumps(
        {'acquisition': float(res.rewards[0])} | {k: _json_value(v[0]) for k, v in res.aux.items()})
    pred = md.ns(self._metadata_ns).ns('prediction_in_warped_y_space')
    pred['mean'] = self._prediction_str(res.aux['mean'][0])
    pred['stddev'] = self._prediction_str(res.aux['stddev'][0])
    pred['stddev_from_all'] = self._prediction_str(res.aux['stddev_from_all'][0])
    pred['acquisition'] = f'{float(res.rewards[0])}'
    pred['use_ucb'] = f'{use_ucb}'
    pred['trust_radius'] = f'{radius}'
    pred['params'] = f'{params}'
    if 'prior_acq_values' in res.aux:
      md.ns(self._metadata_ns).ns('prior_acquisition')['value'] = f'{float(res.aux["prior_acq_values"][0])}'
    md.ns(self._metadata_ns).ns('timing')['time'] = f'{datetime.datetime.now() - start}'
    return vz.TrialSuggestion(params_dict, metadata=md)

  @profiler.record_runtime
  def _suggest_batch_with_exploration(self, count, active_trials, cont, cat, labels, params, mask, radius, n_tr_rows):
    """gp_ucb_pe.py:1157-1260: `count` suggestions as one set maximising the set-PE acquisition (log-determinant of
    the joint predictive covariance given completed + pending trials, penalised below the UCB threshold)."""
    start = datetime.datetime.now()
    cfg = self._config
    dev_a, dev_b = self._devices()
    noise_is_high = self._noise_is_high(params)
    pend_c, pend_z = self._converter.to_features(active_trials)
    pend_c = np.nan_to_num(pend_c, nan=0.0)
    xc_all, xz_all = self._fit_all_features(params, cont, cat, labels, pend_c, pend_z, noise_is_high)
    dk = cat.shape[1]
    out = dev_a.score(xc_all, gp.Acquisition(cfg.ucb_coefficient, False, 1.0), zs=xz_all if dk else None, with_aux=True)
    dev_a.synchronize()
    mu = out['mean'].cpu().numpy(); sd = out['stddev'].cpu().numpy()
    threshold = float(mu[int(np.argmax(mu + cfg.ucb_coefficient * sd))])
    pe = gp.UcbPeAcquisition(
        mode=1, ucb_coefficient=cfg.ucb_coefficient, explore_coefficient=cfg.explore_region_ucb_coefficient,
        penalty_coefficient=cfg.cb_violation_penalty_coefficient, threshold=threshold,
        use_trust_region=self._use_trust_region, trust_radius=radius, tr_dim_mask=mask, tr_rows=n_tr_rows)
    optimizer = self._acquisition_optimizer_factory(self._converter)
    prior = converters.trials_to_sorted_features(self._all_completed_trials, self._converter, (cont, cat))
    res = optimizer.optimize_sets(dev_a, dev_b, pe, n_parallel=count, prior_features=None if prior is None else prior[0],
                                  seed=int(self._rng.integers(2**62)), prior_acquisition=self._prior_acquisition)
    params_list = self._converter.to_parameters(res.features, None)
    end = datetime.datetime.now()
    suggestions = []
    for i, params_dict in enumerate(params_list):
      md = vz.Metadata()
      pred = md.ns(self._metadata_ns).ns('prediction_in_warped_y_space')
      pred['mean'] = repr(float(res.aux['mean'][i]))
      pred['stddev'] = repr(float(res.aux['stddev'][i]))
      pred['stddev_from_all'] = repr(float(res.aux['stddev_from_all'][i]))
      pred['acquisition'] = f'{float(res.rewards[0])}'
      pred['use_ucb'] = 'False'
      pred['trust_radius'] = f'{radius}'
      pred['params'] = f'{params}'
      if 'prior_acq_values' in res.aux:
        md.ns(self._metadata_ns).ns('prior_acquisition')['value'] = f'{float(res.aux["prior_acq_values"][0])}'
      md.ns(self._metadata_ns).ns('timing')['time'] = f'{end - start}'
      suggestions.append(vz.TrialSuggestion(params_dict, metadata=md))
    return suggestions

  # ------------------------------------------------------------------ suggest
  @profiler.record_runtime
  def suggest(self, count: Optional[int] = None):
    """gp_ucb_pe.py:1356-1445."""
    count = count or 1
    if len(self._all_completed_trials) + len(self._all_active_trials) < self._num_seed_trials:
      return self._generate_seed_trials(count)
    cont, cat, labels = self._trials_to_data(self._all_completed_trials)
    params = self._build_gp_model_and_optimize_parameters(cont, cat, labels)
    dev_a, _ = self._devices()
    prior_only = cont.shape[0] == 0          # only ACTIVE trials so far (parallel workers at study start)
    if not prior_only:
      dev_a.fit(cont, self._fit_labels(labels), params, z=cat if cat.shape[1] else None)
    act_c, _ = self._converter.to_features(self._all_active_trials)
    n_tr = cont.shape[0] + act_c.shape[0]   # trust region: completed + initially active trials (:1377-1403)
    mask = acq_lib.trust_region_dim_mask(self._converter.continuous_feasible_values(_MAX_NUM_FEASIBLE_VALUES_FOR_TRUST_REGION))
    radius = acq_lib.trust_radius(n_tr, int(mask.sum()), self._converter.n_categorical)
    active = list(self._all_active_trials)
    out = []
    if count > 1 and self._config.optimize_set_acquisition_for_exploration and not prior_only:
      # gp_ucb_pe.py:1423-1434: one UCB / PE suggestion if trials completed since the newest active one, then the
      # rest of the batch as ONE set optimised for the set-PE acquisition
      if self._ensemble_size > 1:
        # the reference's set path tests `if noise_is_high:` on the per-member array (:996, :1168-1177) and fails
        raise ValueError('optimize_set_acquisition_for_exploration does not support ensemble_size > 1.')
      if _has_new_completed_trials(self._all_completed_trials, active):
        out.append(self._suggest_one(active, cont, cat, labels, params, mask, radius, n_tr))
        active.append(out[-1].to_trial())
      return out + self._suggest_batch_with_exploration(count - len(out), active, cont, cat, labels, params, mask, radius, n_tr)
    for _ in range(count):
      if prior_only:
        s = self._suggest_one_prior_only(active, params, mask, radius, n_tr)
      else:
        s = self._suggest_one(active, cont, cat, labels, params, mask, radius, n_tr)
      out.append(s)
      active.append(s.to_trial())
    return out

  @profiler.record_runtime
  def _suggest_one_prior_only(self, active_trials, params, mask, radius, n_tr_rows):
    """No completed trial yet, only pending ones.  The reference then runs the same code on an empty
    data set (:1006-1155): model A is the GP prior (mean 0, stddev sqrt(sf2 + sn2)), the UCB threshold
    degenerates to the prior mean 0 (_compute_ucb_threshold over no valid point, :175-218), so both the
    PE acquisition  stddev_B + 10 min(0 + 0.5 stddev_A - 0, 0)  and the UCB acquisition  0 + 1.8 stddev_B
    are maximised by the stddev of model B = the GP conditioned on the pending points with dummy labels.
    That is `vzgp_eagle_run` on model B with a unit UCB coefficient (its mean is exactly 0; an ensemble: every member's
    mean is 0, so `vzgp_eagle_run_ensemble` maximises the mixture stddev)."""
    start = datetime.datetime.now()
    _, dev_b = self._devices()
    noise_is_high = self._noise_is_high(params)
    pend_c, pend_z = self._converter.to_features(active_trials)
    pend_c = np.nan_to_num(pend_c, nan=0.0)
    empty_c = np.zeros((0, pend_c.shape[1])); empty_z = np.zeros((0, pend_z.shape[1]), np.int32)
    self._fit_all_features(params, empty_c, empty_z, np.zeros((0, 1)), pend_c, pend_z, noise_is_high)
    acq = gp.Acquisition(1.0, self._use_trust_region, radius, mask, tr_rows=n_tr_rows, tr_strict=True)
    optimizer = self._acquisition_optimizer_factory(self._converter)
    res = optimizer(dev_b, acq, count=1, prior_features=None, prior_categorical=None, seed=int(self._rng.integers(2**62)))
    params_dict = self._converter.to_parameters(res.features[0:1], None if res.categorical is None else res.categorical[0:1])[0]
    members = params if isinstance(params, list) else [params]   # an ensemble: the mixture of the members' priors
    prior_sd = float(np.sqrt(np.mean([p.signal_variance + p.observation_noise_variance for p in members])))
    sd_all = float(res.aux['stddev'][0]) if 'stddev' in res.aux else float(res.rewards[0])
    md = vz.Metadata()
    md.ns('devinfo')['acquisition_optimization'] = json.dumps(
        {'acquisition': float(res.rewards[0]), 'mean': 0.0, 'stddev': prior_sd, 'stddev_from_all': sd_all})
    pred = md.ns(self._metadata_ns).ns('prediction_in_warped_y_space')
    pred['mean'] = self._prediction_str(0.0)
    pred['stddev'] = self._prediction_str(prior_sd)
    pred['stddev_from_all'] = self._prediction_str(sd_all)
    pred['acquisition'] = f'{float(res.rewards[0])}'
    pred['use_ucb'] = 'False'
    pred['trust_radius'] = f'{radius}'
    pred['params'] = f'{params}'
    md.ns(self._metadata_ns).ns('timing')['time'] = f'{datetime.datetime.now() - start}'
    return vz.TrialSuggestion(params_dict, metadata=md)

  # ------------------------------------------------------------------ sample / predict
  @profiler.record_runtime
  def sample(self, trials: Sequence[Any], rng: Any = None, num_samples: int = 1000) -> np.ndarray:
    """gp_ucb_pe.py:1262-1329: unwarped joint posterior samples of the model on the COMPLETED trials
    (re-trained like the reference does), shape (num_samples, num_trials), or (num_samples, num_trials,
    num_metrics) for a multi-metric study."""
    if not trials:
      return np.zeros((num_samples, 0) if self._n_metrics == 1 else (num_samples, 0, self._n_metrics))
    cont, cat, labels = self._trials_to_data(self._all_completed_trials)
    if cont.shape[0] == 0:
      raise NotImplementedError('sample() before any completed trial is not implemented (prior-only GP).')
    params = self._build_gp_model_and_optimize_parameters(cont, cat, labels)
    dev_a, _ = self._devices()
    dev_a.fit(cont, self._fit_labels(labels), params, z=cat if cat.shape[1] else None)
    xs, zs = self._converter.to_features(trials)
    xs = np.nan_to_num(xs, nan=0.0)
    if self._ensemble_size > 1:
      # the uniform mixture: each joint sample from one uniformly drawn member (as VizierGPBandit)
      g = np.random.default_rng(_gpb._seed_from(rng) if rng is not None else 0)
      comps = dev_a.posterior(xs, zs if zs.shape[1] else None, add_noise=True)
      samples = _gpb.mixture_samples(comps, dev_a.members[0], g, num_samples)
      return self._output_warper.unwarp(samples.reshape(-1, 1)).reshape(samples.shape)
    mean, cov = dev_a.posterior(xs, zs if zs.shape[1] else None, add_noise=True)
    chol, _, _ = dev_a.cholesky_retry(cov, jitter=1e-10, max_iters=8)
    g = np.random.default_rng(_gpb._seed_from(rng) if rng is not None else 0)
    if self._n_metrics > 1:
      # independent multi-task GP: one shared covariance, a mean [n_metrics, n]; each metric unwarped by its own warper
      mean, chol = mean.cpu().numpy(), chol.cpu().numpy()
      out = np.empty((num_samples, mean.shape[1], self._n_metrics))
      for m, warper in enumerate(self._output_warpers):
        warped = mean[m][None, :] + g.standard_normal((num_samples, mean.shape[1])) @ chol.T
        out[:, :, m] = warper.unwarp(warped.reshape(-1, 1)).reshape(num_samples, -1)
      return out
    samples = mean.cpu().numpy()[None, :] + g.standard_normal((num_samples, mean.shape[0])) @ chol.cpu().numpy().T
    return self._output_warper.unwarp(samples.reshape(-1, 1)).reshape(samples.shape)

  @profiler.record_runtime
  def predict(self, trials: Sequence[Any], rng: Any = None, num_samples: Optional[int] = 1000):
    """gp_ucb_pe.py:1331-1354: empirical mean / stddev of the unwarped samples."""
    s = self.sample(trials, rng, num_samples or 1000)
    return vz.Prediction(mean=np.mean(s, axis=0), stddev=np.std(s, axis=0))

