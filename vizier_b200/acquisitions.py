"""Host-side acquisition parameters: the acquisition function and the trust region's scalar state.

Mirrors vizier/_src/algorithms/designers/gp/acquisitions.py: `UCB` / `LCB` / `EI` / `PI` (:213-274),
`AcquisitionTrustRegion` (:390-492), `get_best_labels` (:92-109), `bayesian_scoring_function_factory`
(:368-387), `TrustRegion.__post_init__` (:734-749, which dimensions take part), `TrustRegion.trust_radius`
(:757-777).  The per-candidate work (the acquisition of (mean, stddev), its thresholding, the min L-inf distance
and the -1e4 - distance penalty) runs inside the CUDA scoring kernels; `lower_acquisition` turns an acquisition
object into the O(1) scalars they take.  The parallel acquisitions `QEI` / `QPI` / `QUCB` (:495-568) score sets of
points; `lower_parallel_acquisition` turns them into the `gp.QAcquisition` of the set scorer (csrc/score_q.cu).
"""

from __future__ import annotations

import dataclasses
import warnings
from typing import Any, Callable, Optional, Sequence

import numpy as np

from vizier_b200 import _lib
from vizier_b200 import gp

EI_EXPLORATION = 0.01      # tfp_bo GaussianProcessExpectedImprovement default exploration
PI_EXPLORATION = 0.0       # tfp_bo GaussianProcessProbabilityOfImprovement default exploration


class PaddedArray:
  """The part of vizier's `types.PaddedArray` the acquisitions use.  Arrays here are never padded: every row is
  an observation, so `replace_fill_value` has nothing to replace."""

  def __init__(self, array, fill_value=np.nan):
    self.padded_array = np.asarray(array, np.float64)
    self.fill_value = fill_value
    self._original_shape = self.padded_array.shape

  @classmethod
  def as_padded(cls, array) -> 'PaddedArray':
    return cls(array)

  def replace_fill_value(self, fill_value) -> 'PaddedArray':
    return PaddedArray(self.padded_array, fill_value)


@dataclasses.dataclass
class ModelData:
  """types.ModelData: `features` as the converter produces them, `labels` [num_observations, num_metrics]."""

  features: Any
  labels: PaddedArray


def get_best_labels(labels: PaddedArray) -> np.ndarray:
  """Maximum label per metric; -inf without observations (acquisitions.py:92-109)."""
  if np.size(labels.padded_array) == 0:
    return np.asarray(-np.inf)
  return np.max(labels.replace_fill_value(-np.inf).padded_array, axis=-2)


@dataclasses.dataclass
class UCB:
  coefficient: float = 1.8


@dataclasses.dataclass
class LCB:
  coefficient: float = 1.8


@dataclasses.dataclass
class EI:
  best_labels: Any


@dataclasses.dataclass
class PI:
  best_labels: Any


@dataclasses.dataclass
class QEI:
  """Parallel expected improvement of a set of points (acquisitions.py:495-518), estimated from `num_samples`
  joint posterior draws."""

  best_labels: Any
  num_samples: int = 100


@dataclasses.dataclass
class QPI:
  """Parallel probability of improvement (acquisitions.py:521-544)."""

  best_labels: Any
  num_samples: int = 100


@dataclasses.dataclass
class QUCB:
  """Parallel upper confidence bound (acquisitions.py:547-568); QUCB(c * sqrt(pi / 2)) equals UCB(c) for one point."""

  coefficient: float = 1.8
  num_samples: int = 100


_PARALLEL = (QEI, QPI, QUCB)


@dataclasses.dataclass
class AcquisitionTrustRegion:
  """`main_acquisition` where `thresholding_acquisition` >= threshold, else bad_acq_value - thresholding value.
  threshold defaults to min(nanmean, nanmedian) of `labels`; with at most `apply_tr_after` labels the main
  acquisition applies everywhere."""

  main_acquisition: Any
  thresholding_acquisition: Any
  bad_acq_value: float = dataclasses.field(kw_only=True)
  labels: Optional[PaddedArray] = dataclasses.field(kw_only=True)
  threshold: Optional[float] = dataclasses.field(kw_only=True, default=None)
  apply_tr_after: Optional[int] = dataclasses.field(kw_only=True, default=0)

  @classmethod
  def default_ucb_pi(cls, data: ModelData) -> 'AcquisitionTrustRegion':
    return cls(UCB(1.8), PI(get_best_labels(data.labels)), bad_acq_value=-1e4, labels=data.labels, threshold=0.3,
               apply_tr_after=0)

  @classmethod
  def default_ucb_lcb(cls, data: ModelData) -> 'AcquisitionTrustRegion':
    return cls(UCB(1.8), LCB(1.8), labels=data.labels, bad_acq_value=-1e4, threshold=None, apply_tr_after=0)

  @classmethod
  def default_ucb_lcb_wide(cls, data: ModelData) -> 'AcquisitionTrustRegion':
    return cls(UCB(1.8), LCB(2.5), labels=data.labels, bad_acq_value=-1e4, threshold=None, apply_tr_after=0)

  @classmethod
  def default_ucb_lcb_delay_tr(cls, data: ModelData) -> 'AcquisitionTrustRegion':
    return cls(UCB(1.8), LCB(1.8), labels=data.labels, bad_acq_value=-1e4, threshold=None, apply_tr_after=5)


@dataclasses.dataclass
class BayesianScoringFunction:
  """What a scoring-function factory returns: the acquisition function and whether the trust region applies.
  The designer lowers `acquisition_fn` and scores on the device."""

  predictive: Any
  acquisition_fn: Any
  use_trust_region: bool = False


def bayesian_scoring_function_factory(acquisition_fn_factory: Callable[[ModelData], Any]) -> Callable:
  """acquisitions.py:368-387: (data, predictive, continuous_feasible_values, use_trust_region) -> scoring function."""

  def f(data: ModelData, predictive, continuous_feasible_values, use_trust_region: bool = False):
    del continuous_feasible_values
    return BayesianScoringFunction(predictive, acquisition_fn_factory(data), use_trust_region)

  return f


def _num_categorical(features) -> int:
  """Categorical feature dimensions of `ModelData.features`: a (continuous, categorical) pair as the designer passes
  it, or an object with a `categorical` array (vizier's ModelInput)."""
  if features is None:
    return 0
  cat = features[1] if isinstance(features, tuple) else getattr(features, 'categorical', None)
  cat = getattr(cat, 'padded_array', cat)
  return 0 if cat is None else int(np.shape(cat)[-1])


@dataclasses.dataclass
class MaxValueEntropySearch:
  """MaxValueEntropySearch scoring function (acquisitions.py:293-365): the MES of Wang & Jegelka (ICML 2017) over
  `num_max_value_samples` Gumbel-fitted max values seeded by `seed`, then the trust region.  The designer draws the
  max values on the device after each fit (`gp.DeviceGP.mes_fit`) from its model and `best_label`, the best warped
  label (-inf without observations).  Continuous features only."""

  best_label: float
  use_trust_region: bool = False
  num_max_value_samples: int = 100
  seed: int = 123

  @classmethod
  def scoring_fn_factory(cls, data: ModelData, predictive, continuous_feasible_values,
                         use_trust_region: bool = False) -> 'MaxValueEntropySearch':
    """acquisitions.py:299-344: raises ValueError for categorical features."""
    del predictive, continuous_feasible_values
    if _num_categorical(data.features) > 0:
      raise ValueError('Categorical data is not supported.')
    labels = np.asarray(data.labels.padded_array, np.float64)
    best = float(np.max(labels)) if labels.size else -np.inf
    return cls(best, bool(use_trust_region))


def _best_label(best_labels) -> float:
  b = np.asarray(best_labels, np.float64).reshape(-1)
  if b.size != 1:
    raise NotImplementedError(f'EI / PI with {b.size} best labels (one metric only)')
  return float(b[0])


def _lower_term(fn) -> gp.AcqTermSpec:
  if isinstance(fn, UCB):
    return gp.AcqTermSpec(_lib.ACQ_UCB, coefficient=float(fn.coefficient))
  if isinstance(fn, LCB):
    return gp.AcqTermSpec(_lib.ACQ_LCB, coefficient=float(fn.coefficient))
  if isinstance(fn, (EI, PI)):
    best = _best_label(fn.best_labels)
    if not np.isfinite(best):
      # No observation yet (best label -inf): EI is +inf and PI is 1 everywhere.  Score the posterior mean
      # instead, the order EI approaches as the best label goes to -inf.
      return gp.AcqTermSpec(_lib.ACQ_UCB, coefficient=0.0)
    if isinstance(fn, EI):
      return gp.AcqTermSpec(_lib.ACQ_EI, best_label=best, exploration=EI_EXPLORATION)
    return gp.AcqTermSpec(_lib.ACQ_PI, best_label=best, exploration=PI_EXPLORATION)
  raise NotImplementedError(
      f'acquisition function {type(fn).__name__} is not implemented on the device (UCB, LCB, EI, PI and '
      'AcquisitionTrustRegion of those are)')


def check_supported(fn, *, parallel: bool = False) -> None:
  """Raises NotImplementedError unless `lower_acquisition` (or, with parallel=True, `lower_parallel_acquisition`)
  can lower `fn` (any labels)."""
  if parallel:
    if not isinstance(fn, _PARALLEL):
      raise NotImplementedError(
          f'acquisition function {type(fn).__name__} is not a parallel acquisition (QEI, QPI and QUCB are); '
          'scoring_function_is_parallel=True needs one of those')
    return
  if isinstance(fn, _PARALLEL):
    raise NotImplementedError(f'{type(fn).__name__} scores sets of points: use scoring_function_is_parallel=True')
  if isinstance(fn, AcquisitionTrustRegion):
    check_supported(fn.main_acquisition)
    check_supported(fn.thresholding_acquisition)
  elif not isinstance(fn, (UCB, LCB, EI, PI)):
    _lower_term(fn)


def lower_acquisition(fn) -> gp.AcqFnSpec:
  """An acquisition function object -> the `gp.AcqFnSpec` the scoring kernels evaluate.  AcquisitionTrustRegion:
  threshold = its `threshold`, else min(nanmean, nanmedian) of its labels; a NaN threshold, or at most
  `apply_tr_after` labels, leaves the main acquisition alone (acquisitions.py:466-492)."""
  if not isinstance(fn, AcquisitionTrustRegion):
    return gp.AcqFnSpec(_lower_term(fn))
  main = _lower_term(fn.main_acquisition)
  thr = _lower_term(fn.thresholding_acquisition)
  threshold, main_only = -np.inf, False
  if fn.labels is not None:
    labels = fn.labels.replace_fill_value(np.nan).padded_array
    with warnings.catch_warnings():           # all-NaN labels: NaN threshold, no warning
      warnings.simplefilter('ignore', RuntimeWarning)
      threshold = float(np.minimum(np.nanmean(labels), np.nanmedian(labels))) if labels.size else np.nan
    main_only = fn.labels._original_shape[0] <= fn.apply_tr_after
  if fn.threshold is not None:
    threshold = float(fn.threshold)
  if np.isnan(threshold) or main_only:
    return gp.AcqFnSpec(main)
  return gp.AcqFnSpec(main, thresholding=thr, threshold=threshold, bad_acq_value=float(fn.bad_acq_value))


def lower_parallel_acquisition(fn, *, use_trust_region: bool = False, trust_radius: float = 1.0,
                               tr_dim_mask: Optional[np.ndarray] = None) -> gp.QAcquisition:
  """QEI / QPI / QUCB -> the `gp.QAcquisition` the set scorer evaluates.  A best label of -inf (no observation) makes
  QEI and QPI score the expected maximum of the set.  The trust region is the set rule of gp_ucb_pe.py:245-269."""
  check_supported(fn, parallel=True)
  common = dict(num_samples=int(fn.num_samples), use_trust_region=bool(use_trust_region),
                trust_radius=float(trust_radius), tr_dim_mask=tr_dim_mask)
  if isinstance(fn, QUCB):
    return gp.QAcquisition(_lib.QACQ_QUCB, coefficient=float(fn.coefficient), **common)
  kind = _lib.QACQ_QEI if isinstance(fn, QEI) else _lib.QACQ_QPI
  return gp.QAcquisition(kind, best_label=_best_label(fn.best_labels), **common)


TR_MIN_RADIUS = 0.2        # TrustRegion.min_radius (acquisitions.py:751-754)
TR_DIMENSION_FACTOR = 5.0  # acquisitions.py:760
DEFAULT_UCB_COEFFICIENT = 1.8


def trust_region_dim_mask(continuous_feasible_values: Sequence[np.ndarray]) -> np.ndarray:
  """True for dimensions used in the L-inf distance.

  Continuous parameters (empty feasible list) always take part; a discrete parameter takes part
  only if its scaled feasible values have no gap larger than min_radius; single-valued ones never.
  """
  mask = []
  for fv in continuous_feasible_values:
    fv = np.asarray(fv, dtype=np.float64).reshape(-1)
    if fv.size == 0:
      mask.append(True)
    elif fv.size == 1:
      mask.append(False)
    else:
      mask.append(bool(np.max(np.diff(np.sort(fv))) <= TR_MIN_RADIUS))
  return np.asarray(mask, dtype=bool)


def trust_radius(num_obs: int, continuous_dof: int, categorical_dof: int = 0) -> float:
  """0.2 + 0.3 * num_obs / (5 * (dof + 1)); 1.0 with no observations."""
  if num_obs == 0:
    return 1.0
  dof = continuous_dof + categorical_dof
  trust_level = (0.1 * num_obs + 0.9 * num_obs) / (TR_DIMENSION_FACTOR * (dof + 1))
  return TR_MIN_RADIUS + (0.5 - TR_MIN_RADIUS) * trust_level


def make_acquisition(num_obs: int, continuous_feasible_values: Optional[Sequence[np.ndarray]],
                     n_continuous: int, n_categorical: int = 0, *, use_trust_region: bool = True,
                     ucb_coefficient: float = DEFAULT_UCB_COEFFICIENT) -> gp.Acquisition:
  """What `bayesian_scoring_function_factory` (acquisitions.py:368-387) builds, as kernel params."""
  if continuous_feasible_values is None:
    mask = np.ones(n_continuous, dtype=bool)
  else:
    mask = trust_region_dim_mask(continuous_feasible_values)
    if mask.shape[0] != n_continuous:
      raise ValueError(f'{mask.shape[0]} feasible-value lists for {n_continuous} continuous features')
  radius = trust_radius(num_obs, int(mask.sum()), n_categorical)
  return gp.Acquisition(ucb_coefficient, use_trust_region, radius, mask)


def hv_reference_point(labels: np.ndarray, scale: float = 0.01) -> np.ndarray:
  """worst - scale * (best - worst) per metric (acquisitions.py:132-149; labels are maximised)."""
  labels = np.asarray(labels, np.float64)
  best, worst = labels.max(axis=0), labels.min(axis=0)
  return worst - scale * (best - worst)


def hv_scalarize(objectives: np.ndarray, weights: np.ndarray, reference_point=None) -> np.ndarray:
  """HyperVolumeScalarization (scalarization.py:95-111): objectives [N, M], weights [S, M] -> [S, N]:
  min_m(max(obj_m - ref_m, 0) / w_sm) ** M.  Host NumPy: only the observed labels go through here, the
  candidates are scalarised on the device (csrc/multi.cu)."""
  obj = np.asarray(objectives, np.float64)
  if reference_point is not None:
    obj = obj - reference_point
  obj = np.maximum(obj, 0.0)
  prod = obj[None, :, :] / np.asarray(weights, np.float64)[:, None, :]
  return np.min(prod, axis=-1) ** obj.shape[-1]
