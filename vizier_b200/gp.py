"""Device GP: thin Python object over a libvzgp handle.

Mirrors the pieces of the reference's GP stack that `VizierGPBandit` touches:
  * `GPHyperParams`  <-> the parameter dict of `VizierGaussianProcess`
    (vizier/_src/jax/models/tuned_gp_models.py:161-271),
  * `DeviceGP.fit`   <-> `StochasticProcessWithCoroutine.precompute_predictive`
    (vizier/_src/jax/stochastic_process_model.py:968-997),
  * `DeviceGP.loss_and_grad` <-> `loss_with_aux` + autodiff (:940-966),
  * `DeviceGP.score` <-> `BayesianScoringFunction.score_with_aux`
    (vizier/_src/algorithms/designers/gp/acquisitions.py:177-207).
All arithmetic runs in the CUDA library; torch tensors are device-memory handles.
"""

from __future__ import annotations

import ctypes as C
import dataclasses
from typing import Optional, Sequence

import numpy as np
import torch

from vizier_b200 import _lib

# Bounds / regulariser centres of the reference model (tuned_gp_models.py:147-159).
BOUNDARY_EPS = 1e-12
SIGNAL_VARIANCE_BOUNDS = (1e-3 - BOUNDARY_EPS, 10.0 + BOUNDARY_EPS)
LENGTH_SCALE_SQUARED_BOUNDS = (1e-2 - BOUNDARY_EPS, 1e2 + BOUNDARY_EPS)
NOISE_VARIANCE_BOUNDS = (1e-10 - BOUNDARY_EPS, 1.0 + BOUNDARY_EPS)
CHOLESKY_MAX_RETRIES = 5   # retrying_cholesky(jitter=1e-4, max_iters=5), tuned_gp_models.py:272-280


@dataclasses.dataclass
class GPHyperParams:
  signal_variance: float
  continuous_length_scale_squared: np.ndarray
  observation_noise_variance: float
  categorical_length_scale_squared: Optional[np.ndarray] = None
  # `linear_coef` variant (tuned_gp_models.py:203-245): None = plain Matern model.  With it the kernel gains
  # (coef*slope)^2 sum_d (x_d/l_d - coef*shift)(x'_d/l_d - coef*shift) and the GP the mean coef*mean_constant.
  linear_coef: Optional[float] = None
  linear_slope_amplitude: float = 1.0
  linear_shift: float = 0.0
  mean_constant: float = 0.0

  def __post_init__(self):
    self.continuous_length_scale_squared = np.ascontiguousarray(
        np.asarray(self.continuous_length_scale_squared, np.float64).reshape(-1))
    if self.categorical_length_scale_squared is None:
      self.categorical_length_scale_squared = np.zeros((0,), np.float64)
    self.categorical_length_scale_squared = np.ascontiguousarray(
        np.asarray(self.categorical_length_scale_squared, np.float64).reshape(-1))

  # jaxopt's sorted-key flattening: categorical ls2, continuous ls2, noise, signal.
  def to_vector(self) -> np.ndarray:
    lin = [] if not self.linear_coef else [self.linear_shift, self.linear_slope_amplitude, self.mean_constant]
    return np.concatenate([
        self.categorical_length_scale_squared, self.continuous_length_scale_squared, lin,
        [self.observation_noise_variance], [self.signal_variance]])

  @classmethod
  def from_vector(cls, v: np.ndarray, dc: int, dk: int, linear_coef: Optional[float] = None) -> 'GPHyperParams':
    v = np.asarray(v, np.float64)
    if linear_coef:   # sorted keys: ..., linear_shift, linear_slope_amplitude, mean_fn, noise, signal
      o = dk + dc
      return cls(signal_variance=float(v[o + 4]), continuous_length_scale_squared=v[dk:o].copy(),
                 observation_noise_variance=float(v[o + 3]), categorical_length_scale_squared=v[:dk].copy(),
                 linear_coef=float(linear_coef), linear_slope_amplitude=float(v[o + 1]), linear_shift=float(v[o]),
                 mean_constant=float(v[o + 2]))
    return cls(signal_variance=float(v[dk + dc + 1]),
               continuous_length_scale_squared=v[dk:dk + dc].copy(),
               observation_noise_variance=float(v[dk + dc]),
               categorical_length_scale_squared=v[:dk].copy())

  def _c(self) -> _lib.Params:
    p = _lib.Params()
    p.signal_variance = float(self.signal_variance)
    p.observation_noise_variance = float(self.observation_noise_variance)
    p.continuous_length_scale_squared = self.continuous_length_scale_squared.ctypes.data_as(
        C.POINTER(C.c_double))
    p.categorical_length_scale_squared = (
        self.categorical_length_scale_squared.ctypes.data_as(C.POINTER(C.c_double))
        if self.categorical_length_scale_squared.size else None)
    p.linear_coef = float(self.linear_coef or 0.0)
    p.linear_slope_amplitude = float(self.linear_slope_amplitude)
    p.linear_shift = float(self.linear_shift)
    p.mean_constant = float(self.mean_constant)
    return p


def param_bounds(dc: int, dk: int, linear: bool = False) -> tuple[np.ndarray, np.ndarray]:
  if linear:   # shift and mean are unconstrained (+-inf, jaxopt_wrappers._get_bounds), the slope has the amplitude bounds
    lo, hi = param_bounds(dc, dk)
    o = dk + dc
    return (np.concatenate([lo[:o], [-np.inf, SIGNAL_VARIANCE_BOUNDS[0], -np.inf], lo[o:]]),
            np.concatenate([hi[:o], [np.inf, SIGNAL_VARIANCE_BOUNDS[1], np.inf], hi[o:]]))
  lo = np.concatenate([np.full(dk, LENGTH_SCALE_SQUARED_BOUNDS[0]), np.full(dc, LENGTH_SCALE_SQUARED_BOUNDS[0]),
                       [NOISE_VARIANCE_BOUNDS[0]], [SIGNAL_VARIANCE_BOUNDS[0]]])
  hi = np.concatenate([np.full(dk, LENGTH_SCALE_SQUARED_BOUNDS[1]), np.full(dc, LENGTH_SCALE_SQUARED_BOUNDS[1]),
                       [NOISE_VARIANCE_BOUNDS[1]], [SIGNAL_VARIANCE_BOUNDS[1]]])
  return lo, hi


@dataclasses.dataclass(frozen=True)
class AcqTermSpec:
  """One pointwise acquisition of (mean, stddev); see vzgp_acq_term in include/vzgp.h."""

  kind: int                    # _lib.ACQ_UCB / ACQ_LCB / ACQ_EI / ACQ_PI
  coefficient: float = 0.0     # UCB / LCB
  best_label: float = 0.0      # EI / PI
  exploration: float = 0.0     # EI / PI

  def _c(self) -> '_lib.AcqTerm':
    return _lib.AcqTerm(int(self.kind), float(self.coefficient), float(self.best_label), float(self.exploration))


@dataclasses.dataclass(frozen=True)
class AcqFnSpec:
  """Acquisition function a handle scores with (vzgp_set_acquisition): `main`, or with `thresholding` set the
  AcquisitionTrustRegion rule (acquisitions.py:466-492): bad_acq_value - t where t = thresholding < threshold."""

  main: AcqTermSpec
  thresholding: Optional[AcqTermSpec] = None
  threshold: float = 0.0
  bad_acq_value: float = -1e4

  def _c(self) -> '_lib.AcqFn':
    f = _lib.AcqFn()
    f.main = self.main._c()
    f.use_threshold = 1 if self.thresholding is not None else 0
    f.thresholding = (self.thresholding or self.main)._c()
    f.threshold = float(self.threshold)
    f.bad_acq_value = float(self.bad_acq_value)
    return f


@dataclasses.dataclass
class Acquisition:
  """UCB coefficient + trust region (acquisitions.py:213-225, :691-820).  `acq_fn` (acquisitions.lower_acquisition)
  replaces UCB by another acquisition function of (mean, stddev); None scores UCB with `ucb_coefficient`."""

  ucb_coefficient: float = 1.8
  use_trust_region: bool = True
  trust_radius: float = 1.0
  tr_dim_mask: Optional[np.ndarray] = None  # bool [Dc]
  tr_rows: int = 0          # trusted points = first tr_rows rows of the model's X (0 = all)
  tr_strict: bool = False   # dist < radius (gp_ucb_pe.py) instead of dist <= radius (acquisitions.py)
  acq_fn: Optional[AcqFnSpec] = None

  def _c(self):
    a = _lib.Acq()
    a.ucb_coefficient = float(self.ucb_coefficient)
    a.use_trust_region = 1 if self.use_trust_region else 0
    a.trust_radius = float(self.trust_radius)
    a.tr_rows = int(self.tr_rows)
    a.tr_strict = 1 if self.tr_strict else 0
    keep = None
    if self.tr_dim_mask is not None:
      keep = np.ascontiguousarray(np.asarray(self.tr_dim_mask).astype(np.uint8))
      a.tr_dim_mask = keep.ctypes.data_as(C.POINTER(C.c_uint8))
    else:
      a.tr_dim_mask = None
    return a, keep


@dataclasses.dataclass
class UcbPeAcquisition:
  """GP-UCB-PE acquisition parameters (gp_ucb_pe.py:282-492); see vzgp_pe_params in include/vzgp.h."""

  mode: int = 0                      # 0 = UCB (mean_A + c * stddev_B), 1 = PE
  ucb_coefficient: float = 1.8
  explore_coefficient: float = 0.5
  penalty_coefficient: float = 10.0
  threshold: float = 0.0
  use_trust_region: bool = True
  trust_radius: float = 1.0
  tr_dim_mask: Optional[np.ndarray] = None
  tr_rows: int = 0

  def _c(self):
    p = _lib.PeParams()
    p.mode = int(self.mode)
    p.ucb_coefficient = float(self.ucb_coefficient)
    p.explore_coefficient = float(self.explore_coefficient)
    p.penalty_coefficient = float(self.penalty_coefficient)
    p.threshold = float(self.threshold)
    p.use_trust_region = 1 if self.use_trust_region else 0
    p.trust_radius = float(self.trust_radius)
    p.tr_rows = int(self.tr_rows)
    keep = None
    if self.tr_dim_mask is not None:
      keep = np.ascontiguousarray(np.asarray(self.tr_dim_mask).astype(np.uint8))
      p.tr_dim_mask = keep.ctypes.data_as(C.POINTER(C.c_uint8))
    else:
      p.tr_dim_mask = None
    return p, keep


@dataclasses.dataclass
class QAcquisition:
  """Parallel acquisition of sets of q points (QEI / QPI / QUCB, acquisitions.py:495-568) with the set trust region
  of gp_ucb_pe.py:245-269; see vzgp_qacq in include/vzgp.h."""

  kind: int                          # _lib.QACQ_QEI / QACQ_QPI / QACQ_QUCB
  best_label: float = -np.inf        # QEI / QPI; -inf (no observation): E[max f]
  coefficient: float = 1.8           # QUCB
  num_samples: int = 100
  use_trust_region: bool = False
  trust_radius: float = 1.0
  tr_dim_mask: Optional[np.ndarray] = None
  tr_rows: int = 0

  def _c(self, period: int = 0, cov_out: Optional[torch.Tensor] = None):
    a = _lib.QAcq()
    a.kind = int(self.kind)
    a.best_label = float(self.best_label)
    a.coefficient = float(self.coefficient)
    a.num_samples = int(self.num_samples)
    a.period = int(period)
    a.use_trust_region = 1 if self.use_trust_region else 0
    a.trust_radius = float(self.trust_radius)
    a.tr_rows = int(self.tr_rows)
    a.cov_out = None if cov_out is None else cov_out.data_ptr()
    keep = None
    if self.tr_dim_mask is not None:
      keep = np.ascontiguousarray(np.asarray(self.tr_dim_mask).astype(np.uint8))
      a.tr_dim_mask = keep.ctypes.data_as(C.POINTER(C.c_uint8))
    else:
      a.tr_dim_mask = None
    return a, keep


def _score_qsets(devs: Sequence['DeviceGP'], xs_sets, q: int, qacq: QAcquisition, seed: int, zs=None,
                 period: int = 0, with_aux: bool = False, with_cov: bool = False) -> dict:
  """`vzgp_score_qsets` over the uniform mixture of `devs` (one model: a list of one)."""
  f = devs[0]
  xst = f._dev(xs_sets, torch.float64).reshape(-1, f.dc)
  zst = f._dev(zs, torch.int32).reshape(-1, f.dk) if (zs is not None and f.dk > 0) else None
  m = xst.shape[0]
  assert m % q == 0, 'xs_sets must hold whole sets of q points'
  n_sets = m // q
  res = {'score': torch.empty((n_sets,), dtype=torch.float64, device=f.device)}
  if with_aux:
    for k in ('mean', 'stddev', 'linf_distance'):
      res[k] = torch.empty((m,), dtype=torch.float64, device=f.device)
  if with_cov:
    res['cov'] = torch.empty((len(devs), n_sets, q, q), dtype=torch.float64, device=f.device)
  f._stream.wait_stream(torch.cuda.current_stream(f.device))
  a, keep = qacq._c(period, res.get('cov'))
  hs = (C.c_void_p * len(devs))(*[d._h for d in devs])
  _lib.check('vzgp_score_qsets', f._lib.vzgp_score_qsets(
      hs, len(devs), _ptr(xst), _ptr(zst), n_sets, int(q), C.byref(a), C.c_uint64(int(seed) & (2**64 - 1)),
      _ptr(res['score']), _ptr(res.get('mean')), _ptr(res.get('stddev')), _ptr(res.get('linf_distance'))))
  res['_inputs'] = (xst, zst, keep)
  return res


@dataclasses.dataclass
class ScalarizedUcbAcquisition:
  """Hyper-volume scalarised UCB for multi-metric problems (gp_bandit.py:214-242); see vzgp_scalarization
  in include/vzgp.h.  weights [S, M] positive with unit-norm rows, reference_point [M], max_scalarized [S]."""

  weights: np.ndarray
  reference_point: np.ndarray
  max_scalarized: Optional[np.ndarray] = None
  ucb_coefficient: float = 1.8

  def _c(self):
    w = np.ascontiguousarray(np.asarray(self.weights, np.float64))
    r = np.ascontiguousarray(np.asarray(self.reference_point, np.float64).reshape(-1))
    b = None if self.max_scalarized is None else np.ascontiguousarray(np.asarray(self.max_scalarized, np.float64).reshape(-1))
    s = _lib.Scalarization()
    s.n_scalarizations, s.n_metrics = w.shape
    s.weights = w.ctypes.data_as(C.POINTER(C.c_double))
    s.reference_point = r.ctypes.data_as(C.POINTER(C.c_double))
    s.max_scalarized = b.ctypes.data_as(C.POINTER(C.c_double)) if b is not None else None
    s.ucb_coefficient = float(self.ucb_coefficient)
    return s, (w, r, b)


@dataclasses.dataclass
class UcbPeMultiAcquisition:
  """Multi-metric GP-UCB-PE acquisition (gp_ucb_pe.py:344-381, :434-492); see vzgp_pe_multi_params in
  include/vzgp.h.  Mode 0 needs `scalarization` (its ucb_coefficient is not used: `ucb_coefficient` is), mode 1
  the per-metric `thresholds` [n_metrics] and `region_penalty` (_lib.REGION_AVERAGE / UNION / INTERSECTION)."""

  n_metrics: int
  mode: int = 0                      # 0 = scalarised UCB (mean_A + c * stddev_B), 1 = PE
  ucb_coefficient: float = 1.8
  explore_coefficient: float = 0.5
  penalty_coefficient: float = 10.0
  thresholds: Optional[np.ndarray] = None
  region_penalty: int = 0
  scalarization: Optional[ScalarizedUcbAcquisition] = None
  use_trust_region: bool = True
  trust_radius: float = 1.0
  tr_dim_mask: Optional[np.ndarray] = None
  tr_rows: int = 0

  def _c(self):
    p = _lib.PeMultiParams()
    p.mode = int(self.mode)
    p.ucb_coefficient = float(self.ucb_coefficient)
    p.explore_coefficient = float(self.explore_coefficient)
    p.penalty_coefficient = float(self.penalty_coefficient)
    p.use_trust_region = 1 if self.use_trust_region else 0
    p.trust_radius = float(self.trust_radius)
    p.tr_rows = int(self.tr_rows)
    p.n_metrics = int(self.n_metrics)
    p.region_penalty = int(self.region_penalty)
    keep = []
    if self.tr_dim_mask is not None:
      mask = np.ascontiguousarray(np.asarray(self.tr_dim_mask).astype(np.uint8))
      p.tr_dim_mask = mask.ctypes.data_as(C.POINTER(C.c_uint8))
      keep.append(mask)
    else:
      p.tr_dim_mask = None
    if self.thresholds is not None:
      thr = np.ascontiguousarray(np.asarray(self.thresholds, np.float64).reshape(-1))
      p.thresholds = thr.ctypes.data_as(C.POINTER(C.c_double))
      keep.append(thr)
    else:
      p.thresholds = None
    if self.scalarization is not None:
      s, skeep = self.scalarization._c()
      p.scalarization = C.pointer(s)
      keep += [s, skeep]
    else:
      p.scalarization = None
    return p, keep


def _ptr(t: Optional[torch.Tensor]):
  return None if t is None else C.c_void_p(t.data_ptr())


class DeviceGP:
  """One libvzgp handle = one study's GP on one GPU."""

  def __init__(self, device: int = 0, stream: Optional[torch.cuda.Stream] = None):
    self._lib = _lib.load()
    if not torch.cuda.is_available():
      raise RuntimeError('vizier_b200 needs a CUDA device; there is no CPU fallback.')
    self.device = torch.device('cuda', device)
    torch.cuda.init()
    with torch.cuda.device(self.device):
      torch.zeros(1, device=self.device)  # make sure the primary context exists
    self._stream = stream if stream is not None else torch.cuda.Stream(device=self.device)
    h = C.c_void_p()
    _lib.check('vzgp_create', self._lib.vzgp_create(device, C.c_void_p(self._stream.cuda_stream), C.byref(h)))
    self._h = h
    self.dc = self.dk = self.n = 0
    self.n_metrics = 1
    self.cholesky_failed = False
    self._acq_fn: Optional[AcqFnSpec] = None   # what vzgp_set_acquisition last gave the handle

  def set_acquisition(self, fn: Optional[AcqFnSpec]) -> None:
    """Acquisition function of the later scoring and Eagle calls on this handle (None: UCB)."""
    c = fn._c() if fn is not None else None
    _lib.check('vzgp_set_acquisition', self._lib.vzgp_set_acquisition(self._h, C.byref(c) if c is not None else None))
    self._acq_fn = fn

  def _use_acq(self, acq) -> None:
    fn = acq.acq_fn if isinstance(acq, Acquisition) else None
    if fn != self._acq_fn:
      self.set_acquisition(fn)

  def close(self):
    if getattr(self, '_h', None):
      self._lib.vzgp_destroy(self._h)
      self._h = None

  def __del__(self):
    try:
      self.close()
    except Exception:  # pylint: disable=broad-except
      pass

  @property
  def stream(self) -> torch.cuda.Stream:
    return self._stream

  def synchronize(self):
    _lib.check('vzgp_synchronize', self._lib.vzgp_synchronize(self._h))

  @property
  def launch_count(self) -> int:
    return int(self._lib.vzgp_launch_count(self._h))

  def set_int(self, key: str, value: int) -> None:
    _lib.check('vzgp_set_int', self._lib.vzgp_set_int(self._h, key.encode(), int(value)))

  def get_int(self, key: str) -> int:
    v = C.c_int64(0)
    _lib.check('vzgp_get_int', self._lib.vzgp_get_int(self._h, key.encode(), C.byref(v)))
    return int(v.value)

  # -- helpers -------------------------------------------------------------
  def _dev(self, a, dtype) -> Optional[torch.Tensor]:
    if a is None:
      return None
    if isinstance(a, torch.Tensor):
      t = a.to(device=self.device, dtype=dtype).contiguous()
    else:
      t = torch.from_numpy(np.ascontiguousarray(np.asarray(a), dtype={torch.float64: np.float64, torch.int32: np.int32}[dtype])).to(self.device)
    # tensors created on torch's current stream must be complete before our stream reads them
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    return t

  def _xz(self, x, z):
    xt = self._dev(x, torch.float64)
    zt = self._dev(z, torch.int32) if z is not None and np.prod(tuple(z.shape)) > 0 else None
    if zt is not None and zt.shape[1] == 0:
      zt = None
    return xt, zt

  # -- stage-wise entry points -------------------------------------------------
  def kernel_matrix(self, x, params: GPHyperParams, z=None, n_valid=None, diag_add=0.0) -> torch.Tensor:
    xt, zt = self._xz(x, z)
    n, dc = xt.shape
    dk = 0 if zt is None else zt.shape[1]
    out = torch.empty((n, n), dtype=torch.float64, device=self.device)
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    p = params._c()
    _lib.check('vzgp_kernel_matrix', self._lib.vzgp_kernel_matrix(
        self._h, _ptr(xt), _ptr(zt), n, dc, dk, n if n_valid is None else n_valid, C.byref(p),
        float(diag_add), _ptr(out), n))
    self.synchronize()
    return out

  def cross_kernel(self, xs, x, params: GPHyperParams, zs=None, z=None) -> torch.Tensor:
    xst, zst = self._xz(xs, zs)
    xt, zt = self._xz(x, z)
    m, dc = xst.shape
    n = xt.shape[0]
    dk = 0 if zt is None else zt.shape[1]
    out = torch.empty((m, n), dtype=torch.float64, device=self.device)
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    p = params._c()
    _lib.check('vzgp_cross_kernel', self._lib.vzgp_cross_kernel(
        self._h, _ptr(xst), _ptr(zst), m, _ptr(xt), _ptr(zt), n, dc, dk, C.byref(p), _ptr(out), n))
    self.synchronize()
    return out

  def cholesky_retry(self, a, jitter: float = 1e-4, max_iters: int = 5):
    at = self._dev(a, torch.float64)
    n = at.shape[0]
    out = torch.empty((n, n), dtype=torch.float64, device=self.device)
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    shift = C.c_double(0.0)
    retries = _lib.check('vzgp_cholesky_retry', self._lib.vzgp_cholesky_retry(
        self._h, _ptr(at), n, n, float(jitter), int(max_iters), _ptr(out), n, C.byref(shift)))
    return out, float(shift.value), retries

  def factor_inverse(self, a, with_kinv: bool = True):
    """L = chol(a), L^-1 and (optionally) the lower triangle of a^-1 (vzgp_factor_inverse); device tensors."""
    at = self._dev(a, torch.float64)
    n = at.shape[0]
    outs = [torch.zeros((n, n), dtype=torch.float64, device=self.device) for _ in range(3 if with_kinv else 2)]
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    bad = _lib.check('vzgp_factor_inverse', self._lib.vzgp_factor_inverse(
        self._h, _ptr(at), n, n, _ptr(outs[0]), _ptr(outs[1]), _ptr(outs[2]) if with_kinv else None, n))
    return outs, bad

  def tri_inverse(self, l) -> torch.Tensor:
    lt = self._dev(l, torch.float64)
    n = lt.shape[0]
    out = torch.empty((n, n), dtype=torch.float64, device=self.device)
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    _lib.check('vzgp_tri_inverse', self._lib.vzgp_tri_inverse(self._h, _ptr(lt), n, n, _ptr(out), n))
    self.synchronize()
    return out

  # -- model ---------------------------------------------------------------
  def _labels(self, y, n: int):
    """Labels as a metric-major device tensor [M, N] (the layout of vzgp_fit_multi); y is [N] or [N, M]."""
    if isinstance(y, torch.Tensor):
      y2 = y.reshape(n, -1)
      yt = y2.t().contiguous().to(device=self.device, dtype=torch.float64)
    else:
      y2 = np.asarray(y, np.float64).reshape(n, -1)
      yt = torch.from_numpy(np.ascontiguousarray(y2.T)).to(self.device)
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    return yt, y2.shape[1]

  def fit(self, x, y, params: GPHyperParams, z=None, n_valid=None) -> int:
    """y [N] or, for a multi-metric study, [N, M] (independent multi-task GP: one factor, M alphas)."""
    xt, zt = self._xz(x, z)
    n, dc = xt.shape
    yt, n_metrics = self._labels(y, n)
    dk = 0 if zt is None else zt.shape[1]
    p = params._c()
    retries = _lib.check('vzgp_fit_multi', self._lib.vzgp_fit_multi(
        self._h, _ptr(xt), _ptr(zt), _ptr(yt), n, dc, dk, n if n_valid is None else n_valid, n_metrics, C.byref(p)))
    self.n_metrics = n_metrics
    self.synchronize()  # inputs may be freed by the caller after return
    self.n, self.dc, self.dk = n, dc, dk
    # retrying_cholesky(max_iters=5) exhausted (tuned_gp_models.py:272-280): the factor holds NaN exactly
    # like the reference's, every score is NaN and top-k treats it as -inf.  Do not stay silent about it.
    self.cholesky_failed = retries > CHOLESKY_MAX_RETRIES
    if self.cholesky_failed:
      import warnings
      warnings.warn('vzgp_fit: the kernel matrix could not be factored after %d jitter retries; posterior '
                    'and acquisition values are NaN' % CHOLESKY_MAX_RETRIES, RuntimeWarning)
    return retries

  def cholesky(self) -> torch.Tensor:
    out = torch.empty((self.n, self.n), dtype=torch.float64, device=self.device)
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    _lib.check('vzgp_get_cholesky', self._lib.vzgp_get_cholesky(self._h, _ptr(out), self.n))
    self.synchronize()
    return out

  def alpha(self) -> torch.Tensor:
    out = torch.empty((self.n,), dtype=torch.float64, device=self.device)
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    _lib.check('vzgp_get_alpha', self._lib.vzgp_get_alpha(self._h, _ptr(out)))
    self.synchronize()
    return out

  def loss_and_grad(self, x, y, params: GPHyperParams, z=None, n_valid=None):
    """x, y (and z) should be device tensors kept alive by the caller across ARD iterations."""
    xt, zt = self._xz(x, z)
    n, dc = xt.shape
    yt, n_metrics = self._labels(y, n)
    dk = 0 if zt is None else zt.shape[1]
    p = params._c()
    loss = C.c_double(0.0)
    grad = np.zeros(dc + dk + 2 + (3 if params.linear_coef else 0), np.float64)
    retries = _lib.check('vzgp_nll_grad_multi', self._lib.vzgp_nll_grad_multi(
        self._h, _ptr(xt), _ptr(zt), _ptr(yt), n, dc, dk, n if n_valid is None else n_valid, n_metrics,
        C.byref(p), C.byref(loss), grad.ctypes.data_as(C.POINTER(C.c_double))))
    return float(loss.value), grad, retries

  def make_loss_fn(self, x, y, z=None, n_valid=None, linear_coef: Optional[float] = None):
    """theta -> (loss, grad) closure for the ARD driver: the device tensors are resolved once and the
    parameter struct / output buffers are reused, so one evaluation costs a ctypes call (tens of
    microseconds of host time) instead of a dozen torch calls.  theta is in `GPHyperParams.to_vector`
    order (categorical ls2, continuous ls2, noise, signal).  Non-finite losses return (1e300, 0)."""
    xt, zt = self._xz(x, z)
    n, dc = xt.shape
    yt, n_metrics = self._labels(y, n)
    dk = 0 if zt is None else zt.shape[1]
    nv = n if n_valid is None else n_valid
    ls_k = np.zeros(max(dk, 1), np.float64)
    ls_c = np.zeros(max(dc, 1), np.float64)
    lin = 3 if linear_coef else 0
    grad = np.zeros(dc + dk + 2 + lin, np.float64)
    loss = C.c_double(0.0)
    p = _lib.Params()
    p.linear_coef = float(linear_coef or 0.0)
    p.continuous_length_scale_squared = ls_c.ctypes.data_as(C.POINTER(C.c_double))
    p.categorical_length_scale_squared = ls_k.ctypes.data_as(C.POINTER(C.c_double)) if dk else None
    fn, h = self._lib.vzgp_nll_grad_multi, self._h
    px, pz, py = _ptr(xt), _ptr(zt), _ptr(yt)
    pp, pl, pg = C.byref(p), C.byref(loss), grad.ctypes.data_as(C.POINTER(C.c_double))
    keep = (xt, zt, yt, ls_k, ls_c, grad, loss, p)   # referenced by the closure: stays alive with it

    def f(theta, _keep=keep):
      theta = np.asarray(theta, np.float64)
      ls_k[:dk] = theta[:dk]
      ls_c[:dc] = theta[dk:dk + dc]
      if lin:
        p.linear_shift, p.linear_slope_amplitude, p.mean_constant = (float(t) for t in theta[dk + dc:dk + dc + 3])
      p.observation_noise_variance = float(theta[dk + dc + lin])
      p.signal_variance = float(theta[dk + dc + lin + 1])
      _lib.check('vzgp_nll_grad_multi', fn(h, px, pz, py, n, dc, dk, nv, n_metrics, pp, pl, pg))
      v = loss.value
      if not np.isfinite(v):
        return 1e300, np.zeros_like(theta)
      return v, grad.copy()

    return f

  @staticmethod
  def make_batch_loss_fn(devs: Sequence['DeviceGP'], x, y, z=None, n_valid=None):
    """(indices, thetas) -> (losses, grads) for the restarts of one ARD fit: restart i is evaluated on
    `devs[i]`, all of them in ONE graph launch (`vzgp_nll_grad_batch`).  `indices` are the restarts still
    running, `thetas[k]` the point of restart indices[k] (to_vector order).  Non-finite losses come back as
    (1e300, 0) like `make_loss_fn`."""
    lead = devs[0]
    r_all = len(devs)
    xt, zt = lead._xz(x, z)
    n, dc = xt.shape
    yt, n_metrics = lead._labels(y, n)
    for d in devs[1:]:   # the inputs were produced on torch's current stream: every branch stream waits for them
      d._stream.wait_stream(torch.cuda.current_stream(d.device))
    dk = 0 if zt is None else zt.shape[1]
    nv = n if n_valid is None else n_valid
    nq = dc + dk + 2
    ls_c = np.zeros((r_all, max(dc, 1)), np.float64)
    ls_k = np.zeros((r_all, max(dk, 1)), np.float64)
    params = (_lib.Params * r_all)()
    for r in range(r_all):
      params[r].continuous_length_scale_squared = ls_c[r].ctypes.data_as(C.POINTER(C.c_double))
      params[r].categorical_length_scale_squared = ls_k[r].ctypes.data_as(C.POINTER(C.c_double)) if dk else None
      params[r].signal_variance = 1.0
      params[r].observation_noise_variance = 1.0
      ls_c[r, :] = 1.0
      ls_k[r, :] = 1.0
    handles = (C.c_void_p * r_all)(*[d._h for d in devs])
    active = np.zeros(r_all, np.uint8)
    losses = np.zeros(r_all, np.float64)
    grads = np.zeros((r_all, nq), np.float64)
    status = (C.c_int * r_all)()
    fn = lead._lib.vzgp_nll_grad_batch
    keep = (xt, zt, yt, ls_c, ls_k, params, handles, active, losses, grads, status, list(devs))

    def f(indices, thetas, _keep=keep):
      active[:] = 0
      for i, theta in zip(indices, thetas):
        theta = np.asarray(theta, np.float64)
        ls_k[i, :dk] = theta[:dk]
        ls_c[i, :dc] = theta[dk:dk + dc]
        params[i].observation_noise_variance = float(theta[dk + dc])
        params[i].signal_variance = float(theta[dk + dc + 1])
        active[i] = 1
      _lib.check('vzgp_nll_grad_batch', fn(
          handles, r_all, _ptr(xt), _ptr(zt), _ptr(yt), n, dc, dk, nv, n_metrics, params,
          active.ctypes.data_as(C.POINTER(C.c_uint8)), losses.ctypes.data_as(C.POINTER(C.c_double)),
          grads.ctypes.data_as(C.POINTER(C.c_double)), status))
      out_l, out_g = [], []
      for i in indices:
        if np.isfinite(losses[i]):
          out_l.append(float(losses[i])); out_g.append(grads[i].copy())
        else:
          out_l.append(1e300); out_g.append(np.zeros(nq))
      return out_l, out_g

    f.n_restarts = r_all
    f.status = status   # per restart, of the last call: Cholesky retries of a restart that took the retry path
    return f

  def score(self, xs, acq: Acquisition, zs=None, with_aux: bool = False, out: Optional[dict] = None) -> dict:
    """Asynchronous on self.stream; returns device tensors {'score', ['mean','stddev','linf_distance']}."""
    xst, zst = self._xz(xs, zs)
    m = xst.shape[0]
    res = out if out is not None else {}
    if 'score' not in res:
      res['score'] = torch.empty((m,), dtype=torch.float64, device=self.device)
      if with_aux:
        for k in ('mean', 'stddev', 'linf_distance'):
          res[k] = torch.empty((m,), dtype=torch.float64, device=self.device)
      self._stream.wait_stream(torch.cuda.current_stream(self.device))
    self._use_acq(acq)
    a, keep = acq._c()
    _lib.check('vzgp_score', self._lib.vzgp_score(
        self._h, _ptr(xst), _ptr(zst), m, C.byref(a), _ptr(res['score']), _ptr(res.get('mean')),
        _ptr(res.get('stddev')), _ptr(res.get('linf_distance'))))
    res['_inputs'] = (xst, zst, keep)  # keep alive until the caller synchronises
    return res

  def score_multi(self, xs, acq: ScalarizedUcbAcquisition, zs=None, with_aux: bool = False) -> dict:
    """Multi-metric scalarised UCB; returns device tensors {'score' [M], ['mean' [n_metrics, M], 'stddev' [M]]}."""
    xst, zst = self._xz(xs, zs)
    m = xst.shape[0]
    res = {'score': torch.empty((m,), dtype=torch.float64, device=self.device)}
    if with_aux:
      res['mean'] = torch.empty((self.n_metrics, m), dtype=torch.float64, device=self.device)
      res['stddev'] = torch.empty((m,), dtype=torch.float64, device=self.device)
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    sc, keep = acq._c()
    _lib.check('vzgp_score_multi', self._lib.vzgp_score_multi(
        self._h, _ptr(xst), _ptr(zst), m, C.byref(sc), _ptr(res['score']), _ptr(res.get('mean')), _ptr(res.get('stddev'))))
    res['_inputs'] = (xst, zst, keep)
    return res

  def clamped_count(self) -> int:
    c = C.c_int64(0)
    _lib.check('vzgp_clamped_count', self._lib.vzgp_clamped_count(self._h, C.byref(c)))
    return int(c.value)

  def score_host(self, xs: np.ndarray, acq: Acquisition, *, score_out: np.ndarray,
                 zs: Optional[np.ndarray] = None, mean_out=None, stddev_out=None, linf_out=None):
    """HOST buffers in, HOST buffers out (pinned memory recommended).  Synchronous."""
    self._use_acq(acq)
    a, keep = acq._c()
    m = xs.shape[0]

    def hp(arr):
      if arr is None:
        return None
      if isinstance(arr, torch.Tensor):
        return C.c_void_p(arr.data_ptr())
      return C.c_void_p(arr.ctypes.data)

    _lib.check('vzgp_score_host', self._lib.vzgp_score_host(
        self._h, hp(xs), hp(zs), m, C.byref(a), hp(score_out), hp(mean_out), hp(stddev_out), hp(linf_out)))
    del keep

  def posterior(self, xs, zs=None, add_noise: bool = True):
    """Joint posterior mean [M] and covariance [M, M] (device tensors)."""
    xst, zst = self._xz(xs, zs)
    m = xst.shape[0]
    mean = torch.empty((self.n_metrics, m), dtype=torch.float64, device=self.device)
    cov = torch.empty((m, m), dtype=torch.float64, device=self.device)
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    _lib.check('vzgp_posterior_multi', self._lib.vzgp_posterior_multi(
        self._h, _ptr(xst), _ptr(zst), m, 1 if add_noise else 0, _ptr(mean), _ptr(cov), m))
    self.synchronize()
    return (mean[0] if self.n_metrics == 1 else mean), cov

  def topk(self, score: torch.Tensor, count: int):
    idx = np.zeros(count, np.int64)
    val = np.zeros(count, np.float64)
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    _lib.check('vzgp_topk', self._lib.vzgp_topk(
        self._h, _ptr(score), score.numel(), count, idx.ctypes.data_as(C.POINTER(C.c_int64)),
        val.ctypes.data_as(C.POINTER(C.c_double))))
    return idx, val

  def score_topk(self, xs: torch.Tensor, acq: Acquisition, count: int, score_out: Optional[torch.Tensor] = None):
    """Score device candidates, select the top `count`, return (features, scores, indices) on the host."""
    self._use_acq(acq)
    a, keep = acq._c()
    m = xs.shape[0]
    bx = np.zeros((count, self.dc), np.float64)
    bs = np.zeros(count, np.float64)
    bi = np.zeros(count, np.int64)
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    _lib.check('vzgp_score_topk', self._lib.vzgp_score_topk(
        self._h, _ptr(xs), None, m, C.byref(a), count, _ptr(score_out),
        bx.ctypes.data_as(C.POINTER(C.c_double)), bs.ctypes.data_as(C.POINTER(C.c_double)),
        bi.ctypes.data_as(C.POINTER(C.c_int64))))
    del keep
    return bx, bs, bi

  def suggest_host(self, xs_host, acq: Acquisition, count: int, index_base: int = 0, *, exchange=None,
                   score_out=None):
    """`vzgp_suggest_host`: one sharded suggest from HOST candidates (torch CPU tensor, ideally pinned, or
    a NumPy array) in one synchronous C call; `exchange` is a `multi_gpu.PeerExchange` (None = this rank
    alone).  Returns (global indices [count] i64, scores [count], features [count, Dc]) - the same on
    every rank."""
    self._use_acq(acq)
    a, keep = acq._c()
    m = xs_host.shape[0]
    rows = np.zeros((count, self.dc + 2), np.float64)

    def hp(arr):
      if arr is None:
        return None
      return C.c_void_p(arr.data_ptr()) if isinstance(arr, torch.Tensor) else C.c_void_p(arr.ctypes.data)

    use_nccl = 1 if (exchange is not None and exchange.transport == 'nccl' and exchange.world > 1) else 0
    _lib.check('vzgp_suggest_host', self._lib.vzgp_suggest_host(
        self._h, exchange._x if exchange is not None else None, use_nccl, hp(xs_host), m, C.byref(a), count,
        int(index_base), hp(score_out), C.c_void_p(rows.ctypes.data)))
    del keep
    return rows[:, 1].astype(np.int64), rows[:, 0].copy(), rows[:, 2:].copy()

  def score_topk_pack(self, xs: torch.Tensor, acq: Acquisition, count: int, index_base: int,
                      payload: torch.Tensor, score_out: Optional[torch.Tensor] = None) -> None:
    """Asynchronous shard step: score, local top-`count`, rows [score, global index, features] into the
    device tensor `payload` [count, Dc+2].  No host synchronisation (multi_gpu.TopkExchange)."""
    self._use_acq(acq)
    a, keep = acq._c()
    assert payload.is_cuda and payload.dtype == torch.float64 and payload.shape == (count, self.dc + 2)
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    _lib.check('vzgp_score_topk_pack', self._lib.vzgp_score_topk_pack(
        self._h, _ptr(xs), None, xs.shape[0], C.byref(a), count, int(index_base), _ptr(score_out), _ptr(payload)))
    del keep

  def merge_topk(self, rows: torch.Tensor, count: int, out: torch.Tensor, host_out: Optional[torch.Tensor] = None) -> None:
    """Device merge of gathered winner rows [n_rows, width] into out [count, width] (+ async copy to the
    pinned host tensor `host_out`); runs on the handle's stream, no host synchronisation."""
    assert rows.is_cuda and rows.dtype == torch.float64 and rows.is_contiguous()
    assert out.shape == (count, rows.shape[1])
    if host_out is not None:
      assert not host_out.is_cuda and host_out.is_pinned() and host_out.shape == out.shape
    _lib.check('vzgp_merge_topk', self._lib.vzgp_merge_topk(
        self._h, _ptr(rows), rows.shape[0], rows.shape[1], count, _ptr(out),
        C.c_void_p(host_out.data_ptr()) if host_out is not None else None))

  def random_pool(self, m: int, dc: int, seed: int, index_base: int = 0) -> torch.Tensor:
    out = torch.empty((m, dc), dtype=torch.float64, device=self.device)
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    _lib.check('vzgp_random_pool', self._lib.vzgp_random_pool(self._h, m, dc, index_base, seed, _ptr(out)))
    self.synchronize()
    return out

  def random_pool_cat(self, m: int, cat_sizes, seed: int, index_base: int = 0) -> torch.Tensor:
    sizes = np.ascontiguousarray(np.asarray(cat_sizes, np.int32))
    out = torch.empty((m, sizes.shape[0]), dtype=torch.int32, device=self.device)
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    _lib.check('vzgp_random_pool_cat', self._lib.vzgp_random_pool_cat(
        self._h, m, sizes.shape[0], sizes.ctypes.data_as(C.POINTER(C.c_int32)), index_base, seed, _ptr(out)))
    self.synchronize()
    return out

  def random_search(self, m: int, acq: Acquisition, count: int, seed: int, index_base: int = 0, cat_sizes=None):
    """Returns (best_x [count,Dc], best_z [count,Dk], best_score [count], best_index [count])."""
    self._use_acq(acq)
    a, keep = acq._c()
    bx = np.zeros((count, self.dc), np.float64)
    bz = np.zeros((count, self.dk), np.int32)
    bs = np.zeros(count, np.float64)
    bi = np.zeros(count, np.int64)
    sizes = np.ascontiguousarray(np.asarray(cat_sizes if cat_sizes is not None else [], np.int32))
    _lib.check('vzgp_random_search', self._lib.vzgp_random_search(
        self._h, m, index_base, C.byref(a), sizes.ctypes.data_as(C.POINTER(C.c_int32)) if sizes.size else None,
        count, seed, bx.ctypes.data_as(C.POINTER(C.c_double)), bz.ctypes.data_as(C.POINTER(C.c_int32)),
        bs.ctypes.data_as(C.POINTER(C.c_double)), bi.ctypes.data_as(C.POINTER(C.c_int64))))
    del keep
    return bx, bz, bs, bi

  def score_pe(self, other: 'DeviceGP', xs, pe: UcbPeAcquisition, zs=None) -> dict:
    """GP-UCB-PE score with self = model on completed trials, other = model on completed+pending.
    Returns device tensors {'score','mean','stddev','stddev_from_all'}; synchronous."""
    xst, zst = self._xz(xs, zs)
    m = xst.shape[0]
    res = {k: torch.empty((m,), dtype=torch.float64, device=self.device) for k in ('score', 'mean', 'stddev', 'stddev_from_all')}
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    p, keep = pe._c()
    _lib.check('vzgp_score_pe', self._lib.vzgp_score_pe(
        self._h, other._h, _ptr(xst), _ptr(zst), m, C.byref(p), _ptr(res['score']), _ptr(res['mean']),
        _ptr(res['stddev']), _ptr(res['stddev_from_all'])))
    self.synchronize()
    del keep
    return res

  def score_pe_multi(self, other: 'DeviceGP', xs, pe: UcbPeMultiAcquisition, zs=None) -> dict:
    """Multi-metric GP-UCB-PE score with self = multi-metric model on completed trials, other = model on
    completed + pending trials.  Returns device tensors {'score' [M], 'mean' [n_metrics, M], 'stddev' [M],
    'stddev_from_all' [M]}; synchronous."""
    xst, zst = self._xz(xs, zs)
    m = xst.shape[0]
    res = {k: torch.empty((m,), dtype=torch.float64, device=self.device) for k in ('score', 'stddev', 'stddev_from_all')}
    res['mean'] = torch.empty((self.n_metrics, m), dtype=torch.float64, device=self.device)
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    p, keep = pe._c()
    _lib.check('vzgp_score_pe_multi', self._lib.vzgp_score_pe_multi(
        self._h, other._h, _ptr(xst), _ptr(zst), m, C.byref(p), _ptr(res['score']), _ptr(res['mean']),
        _ptr(res['stddev']), _ptr(res['stddev_from_all'])))
    self.synchronize()
    del keep
    return res

  def score_set_pe(self, other: 'DeviceGP', xs_sets, q: int, pe: UcbPeAcquisition) -> dict:
    """Set-PE acquisition (gp_ucb_pe.py:510-594) of n_sets sets of q points: xs_sets [n_sets * q, Dc] (or
    [n_sets, q * Dc]).  self = model on completed trials, other = model on completed + pending trials.  Returns
    device tensors {'score' [n_sets], 'mean', 'stddev', 'stddev_from_all' [n_sets * q]}; asynchronous."""
    xst = self._dev(xs_sets, torch.float64).reshape(-1, self.dc)
    m = xst.shape[0]
    assert m % q == 0
    n_sets = m // q
    res = {'score': torch.empty((n_sets,), dtype=torch.float64, device=self.device)}
    for k in ('mean', 'stddev', 'stddev_from_all'):
      res[k] = torch.empty((m,), dtype=torch.float64, device=self.device)
    self._stream.wait_stream(torch.cuda.current_stream(self.device))
    p, keep = pe._c()
    _lib.check('vzgp_score_set_pe', self._lib.vzgp_score_set_pe(
        self._h, other._h, _ptr(xst), n_sets, int(q), C.byref(p), _ptr(res['score']), _ptr(res['mean']),
        _ptr(res['stddev']), _ptr(res['stddev_from_all'])))
    res['_inputs'] = (xst, keep)
    return res

  def score_qsets(self, xs_sets, q: int, qacq: QAcquisition, seed: int, zs=None, period: int = 0,
                  with_aux: bool = False, with_cov: bool = False) -> dict:
    """q-acquisition of n_sets sets of q points: xs_sets [n_sets * q, Dc] (or [n_sets, q * Dc]), zs [n_sets * q, Dk].
    The draws of a set depend on its position (index mod `period`; 0: n_sets) and `seed`.  Returns device tensors
    {'score' [n_sets], ['mean', 'stddev', 'linf_distance' [n_sets * q]], ['cov' [1, n_sets, q, q]]}; asynchronous."""
    return _score_qsets([self], xs_sets, q, qacq, seed, zs, period, with_aux, with_cov)

  def qacq_from_moments(self, mean, cov, qacq: QAcquisition, seed: int, period: int = 0) -> torch.Tensor:
    """The Monte Carlo stage alone: mean [E, n_sets, q], cov [E, n_sets, q, q] -> scores [n_sets] (device)."""
    mt = self._dev(mean, torch.float64)
    ct = self._dev(cov, torch.float64)
    e, n_sets, q = mt.shape
    assert ct.shape == (e, n_sets, q, q)
    out = torch.empty((n_sets,), dtype=torch.float64, device=self.device)
    a, keep = qacq._c(period)
    _lib.check('vzgp_qacq_from_moments', self._lib.vzgp_qacq_from_moments(
        self._h, n_sets, q, e, _ptr(mt), _ptr(ct), C.byref(a), C.c_uint64(int(seed) & (2**64 - 1)), _ptr(out)))
    self.synchronize()
    del keep
    return out

  def eagle_run(self, cfg: '_lib.EagleConfig', acq, count: int, seed: int,
                prior: Optional[Sequence] = None, prior_z: Optional[Sequence] = None, cat_sizes=None,
                other: Optional['DeviceGP'] = None):
    """Returns (best_x [count,Dc], best_z [count,Dk], best_score [count]).  With `other` and a
    UcbPeAcquisition the GP-UCB-PE acquisition is optimised (vzgp_eagle_run_pe), with a UcbPeMultiAcquisition its
    multi-metric form (vzgp_eagle_run_pe_multi)."""
    if isinstance(acq, (UcbPeAcquisition, UcbPeMultiAcquisition)):
      return self._eagle_run_pe(cfg, acq, count, seed, prior, prior_z, cat_sizes, other)
    multi = isinstance(acq, ScalarizedUcbAcquisition)
    if not multi:
      self._use_acq(acq)
    a, keep = acq._c()
    n_prior = 0 if prior is None else len(prior)
    pt = self._dev(prior, torch.float64) if n_prior > 0 and self.dc > 0 else None
    pz = self._dev(prior_z, torch.int32) if n_prior > 0 and self.dk > 0 else None
    bx = np.zeros((count, self.dc), np.float64)
    bz = np.zeros((count, self.dk), np.int32)
    bs = np.zeros(count, np.float64)
    sizes = np.ascontiguousarray(np.asarray(cat_sizes if cat_sizes is not None else [], np.int32))
    fn_name = 'vzgp_eagle_run_multi' if multi else 'vzgp_eagle_run'
    _lib.check(fn_name, getattr(self._lib, fn_name)(
        self._h, C.byref(cfg), C.byref(a), _ptr(pt), _ptr(pz), n_prior,
        sizes.ctypes.data_as(C.POINTER(C.c_int32)) if sizes.size else None, count, seed,
        bx.ctypes.data_as(C.POINTER(C.c_double)), bz.ctypes.data_as(C.POINTER(C.c_int32)),
        bs.ctypes.data_as(C.POINTER(C.c_double))))
    del keep
    return bx, bz, bs

  def _eagle_run_pe(self, cfg, pe, count, seed, prior, prior_z, cat_sizes, other):
    fn_name = 'vzgp_eagle_run_pe_multi' if isinstance(pe, UcbPeMultiAcquisition) else 'vzgp_eagle_run_pe'
    p, keep = pe._c()
    n_prior = 0 if prior is None else len(prior)
    pt = self._dev(prior, torch.float64) if n_prior > 0 and self.dc > 0 else None
    pz = self._dev(prior_z, torch.int32) if n_prior > 0 and self.dk > 0 else None
    bx = np.zeros((count, self.dc), np.float64)
    bz = np.zeros((count, self.dk), np.int32)
    bs = np.zeros(count, np.float64)
    sizes = np.ascontiguousarray(np.asarray(cat_sizes if cat_sizes is not None else [], np.int32))
    _lib.check(fn_name, getattr(self._lib, fn_name)(
        self._h, other._h, C.byref(cfg), C.byref(p), _ptr(pt), _ptr(pz), n_prior,
        sizes.ctypes.data_as(C.POINTER(C.c_int32)) if sizes.size else None, count, seed,
        bx.ctypes.data_as(C.POINTER(C.c_double)), bz.ctypes.data_as(C.POINTER(C.c_int32)),
        bs.ctypes.data_as(C.POINTER(C.c_double))))
    del keep
    return bx, bz, bs

def transfer_dof(n: int, num_hyperparameters: int) -> float:
  """gp/transfer_learning.py:38-59 (_compute_dof)."""
  return max(n - num_hyperparameters, n / (1.0 + num_hyperparameters))


def transfer_alpha(n_top: int, n_base: int, num_hyperparameters: int, expected_base_stddev_mismatch: float = 1.0) -> float:
  """Weight of the top level's stddev in the geometric mean (gp/transfer_learning.py:96-118)."""
  dof_base, dof_top = transfer_dof(n_base, num_hyperparameters), transfer_dof(n_top, num_hyperparameters)
  beta2 = (dof_top / dof_base) * (1.0 + dof_base + expected_base_stddev_mismatch ** 2)
  return beta2 / (1.0 + beta2)


class StackedGP:
  """Stack of residual GPs for transfer learning (`VizierGPBandit.set_priors`, gp_bandit.py:289-318; StackedResidualGP,
  gp/gp_models.py:91-140, :245-300): level 0 is fitted on the first prior study, each further level on the residuals
  of the next study against the stack below it, the last level on the current study.  The levels are libvzgp handles
  on ONE stream; scoring and the Eagle loop run through `vzgp_score_stack` / `vzgp_eagle_run_stack`.  Exposes the
  subset of the `DeviceGP` interface the acquisition optimiser drives."""

  def __init__(self, device: int):
    self._device_index = device
    self.levels: list = []          # DeviceGP per level, base first
    self.counts: list = []          # training points per level
    self.alphas: list = []          # alphas[e]: weight of level e's stddev against the stack below (alphas[0] unused)
    self.device = None
    self.dc = self.dk = self.n = 0

  @property
  def top(self) -> 'DeviceGP':
    return self.levels[-1]

  @property
  def stream(self):
    return self.levels[0].stream

  @property
  def launch_count(self) -> int:
    return sum(m.launch_count for m in self.levels)

  def synchronize(self):
    self.levels[0].synchronize()

  def close(self):
    for m in self.levels:
      m.close()
    self.levels = []

  def truncate(self, n_levels: int) -> None:
    """Keeps the first n_levels levels (the prior stack) and drops the rest (a new top level follows)."""
    for m in self.levels[n_levels:]:
      m.close()
    del self.levels[n_levels:], self.counts[n_levels:], self.alphas[n_levels:]

  def new_level(self) -> 'DeviceGP':
    m = DeviceGP(self._device_index) if not self.levels else DeviceGP(self._device_index, stream=self.levels[0].stream)
    return m

  def mean(self, xs, zs=None) -> np.ndarray:
    """Mean of the stack built so far at xs (0 for an empty stack): the quantity the next level's labels are reduced by
    (`_pred_mean`, gp/gp_models.py:268-283)."""
    n = len(xs)
    if not self.levels:
      return np.zeros(n)
    out = self.score(xs, Acquisition(0.0, False, 1.0), zs=zs, with_aux=True)
    self.synchronize()
    return out['mean'].cpu().numpy()

  def push(self, level: 'DeviceGP', n_points: int) -> None:
    """Adds a fitted level on top of the stack."""
    h = level.dc + level.dk + 2           # GPState.num_hyperparameters (gp/gp_models.py:77-88)
    self.alphas.append(0.0 if not self.levels else transfer_alpha(n_points, self.counts[-1], h))
    self.levels.append(level)
    self.counts.append(int(n_points))
    self.device, self.dc, self.dk, self.n = level.device, level.dc, level.dk, level.n

  def _handles(self):
    return (C.c_void_p * len(self.levels))(*[m._h for m in self.levels])

  def _alphas(self):
    return (C.c_double * len(self.levels))(*self.alphas)

  def score(self, xs, acq: Acquisition, zs=None, with_aux: bool = False) -> dict:
    f = self.levels[-1]
    xst, zst = f._xz(xs, zs)
    m = xst.shape[0]
    res = {'score': torch.empty((m,), dtype=torch.float64, device=f.device)}
    if with_aux:
      for k in ('mean', 'stddev', 'linf_distance'):
        res[k] = torch.empty((m,), dtype=torch.float64, device=f.device)
    f._stream.wait_stream(torch.cuda.current_stream(f.device))
    self.levels[0]._use_acq(acq)          # multi-handle calls take the acquisition of hs[0]
    a, keep = acq._c()
    _lib.check('vzgp_score_stack', f._lib.vzgp_score_stack(
        self._handles(), len(self.levels), self._alphas(), _ptr(xst), _ptr(zst), m, C.byref(a), _ptr(res['score']),
        _ptr(res.get('mean')), _ptr(res.get('stddev')), _ptr(res.get('linf_distance'))))
    res['_inputs'] = (xst, zst, keep)
    return res

  def eagle_run(self, cfg, acq: Acquisition, count: int, seed: int, prior=None, prior_z=None, cat_sizes=None, other=None):
    assert other is None
    f = self.levels[-1]
    self.levels[0]._use_acq(acq)
    a, keep = acq._c()
    n_prior = 0 if prior is None else len(prior)
    pt = f._dev(prior, torch.float64) if n_prior > 0 and self.dc > 0 else None
    pz = f._dev(prior_z, torch.int32) if n_prior > 0 and self.dk > 0 else None
    bx = np.zeros((count, self.dc), np.float64)
    bz = np.zeros((count, self.dk), np.int32)
    bs = np.zeros(count, np.float64)
    sizes = np.ascontiguousarray(np.asarray(cat_sizes if cat_sizes is not None else [], np.int32))
    _lib.check('vzgp_eagle_run_stack', f._lib.vzgp_eagle_run_stack(
        self._handles(), len(self.levels), self._alphas(), C.byref(cfg), C.byref(a), _ptr(pt), _ptr(pz), n_prior,
        sizes.ctypes.data_as(C.POINTER(C.c_int32)) if sizes.size else None, count, seed,
        bx.ctypes.data_as(C.POINTER(C.c_double)), bz.ctypes.data_as(C.POINTER(C.c_int32)),
        bs.ctypes.data_as(C.POINTER(C.c_double))))
    del keep
    return bx, bz, bs

  def random_search(self, m: int, acq: Acquisition, count: int, seed: int, index_base: int = 0, cat_sizes=None):
    """RandomVectorizedStrategy over the stack: Philox pool -> combined score -> device top-k."""
    f = self.levels[-1]
    xs = f.random_pool(m, self.dc, seed, index_base) if self.dc else torch.zeros((m, 0), dtype=torch.float64, device=f.device)
    zs = f.random_pool_cat(m, cat_sizes, seed, index_base) if self.dk else None
    out = self.score(xs, acq, zs=zs)
    idx, val = f.topk(out['score'], count)
    it = torch.from_numpy(np.maximum(idx, 0)).to(f.device)
    bx = xs[it].cpu().numpy()
    bz = zs[it].cpu().numpy() if zs is not None else np.zeros((count, 0), np.int32)
    return bx, bz, val, idx + index_base

  def topk(self, score, count: int):
    return self.levels[-1].topk(score, count)


class _DevView:
  """A raw device pointer as a `__cuda_array_interface__` object (zero-copy torch view of library-owned memory)."""

  def __init__(self, ptr: int, shape, typestr: str):
    self.__cuda_array_interface__ = {'shape': tuple(shape), 'typestr': typestr, 'data': (int(ptr), False), 'version': 2}


class SteppedEagle:
  """Host-stepped Eagle loop (vzgp_eagle_begin / seed / ask / tell / end): the device-resident optimiser state and
  kernels of `DeviceGP.eagle_run`, with the batch scored by the caller - used for acquisitions that include a
  host-side term (`prior_acquisition`, gp_ucb_pe.py:286-381)."""

  def __init__(self, dev: 'DeviceGP', cfg: '_lib.EagleConfig', count: int, seed: int, n_prior: int = 0, cat_sizes=None):
    self.dev, self.count, self.batch_size = dev, count, int(cfg.batch_size)
    self.n_prior = int(n_prior)
    self.q = max(1, int(cfg.n_parallel))          # points per fly (set acquisitions)
    self.fly_dim = dev.dc * self.q
    sizes = np.ascontiguousarray(np.asarray(cat_sizes if cat_sizes is not None else [], np.int32))
    pr = C.c_void_p(0)
    _lib.check('vzgp_eagle_begin', dev._lib.vzgp_eagle_begin(
        dev._h, C.byref(cfg), sizes.ctypes.data_as(C.POINTER(C.c_int32)) if sizes.size else None, count, seed,
        self.n_prior, C.byref(pr)))
    self._prior_rewards = pr.value

  def _view(self, ptr, shape, typestr):
    return torch.as_tensor(_DevView(ptr, shape, typestr), device=self.dev.device)

  def seed(self, prior, prior_z, rewards) -> None:
    """prior [n_prior, Dc] / prior_z [n_prior, Dk] features and their acquisition values [n_prior]."""
    d = self.dev
    with torch.cuda.stream(d._stream):
      self._view(self._prior_rewards, (self.n_prior,), '<f8').copy_(torch.as_tensor(rewards, dtype=torch.float64, device=d.device))
    pt = d._dev(prior, torch.float64).reshape(self.n_prior, self.fly_dim).contiguous() if d.dc > 0 else None
    pz = d._dev(prior_z, torch.int32) if d.dk > 0 else None
    d._stream.wait_stream(torch.cuda.current_stream(d.device))
    _lib.check('vzgp_eagle_seed', d._lib.vzgp_eagle_seed(d._h, _ptr(pt), _ptr(pz)))
    self._keep = (pt, pz)

  def ask(self):
    """Next batch: (xs [B, Dc] device view, zs [B, Dk] device view or None, rewards [B] device view to fill)."""
    d = self.dev
    px, pz, pr = C.c_void_p(0), C.c_void_p(0), C.c_void_p(0)
    _lib.check('vzgp_eagle_ask', d._lib.vzgp_eagle_ask(d._h, C.byref(px), C.byref(pz), C.byref(pr)))
    b = self.batch_size
    xs = self._view(px.value, (b, self.fly_dim), '<f8') if d.dc > 0 else torch.zeros((b, 0), dtype=torch.float64, device=d.device)
    zs = self._view(pz.value, (b, d.dk), '<i4') if d.dk > 0 else None
    return xs, zs, self._view(pr.value, (b,), '<f8')

  def tell(self) -> None:
    _lib.check('vzgp_eagle_tell', self.dev._lib.vzgp_eagle_tell(self.dev._h))

  def end(self):
    d = self.dev
    bx = np.zeros((self.count, self.fly_dim), np.float64)
    bz = np.zeros((self.count, d.dk), np.int32)
    bs = np.zeros(self.count, np.float64)
    _lib.check('vzgp_eagle_end', d._lib.vzgp_eagle_end(
        d._h, bx.ctypes.data_as(C.POINTER(C.c_double)), bz.ctypes.data_as(C.POINTER(C.c_int32)),
        bs.ctypes.data_as(C.POINTER(C.c_double))))
    return bx, bz, bs


class EnsembleGP:
  """Uniform ensemble of E GPs fitted on the same trials with different hyper-parameters
  (`VizierGPBandit(ensemble_size=E)`: the E best ARD restarts, gp_models.py:200-223; predictive =
  UniformEnsemblePredictive, stochastic_process_model.py:836-868).  The members are E libvzgp handles on
  ONE stream; scoring and the Eagle loop run through `vzgp_score_ensemble` / `vzgp_eagle_run_ensemble`.
  Exposes the subset of the `DeviceGP` interface the acquisition optimiser drives."""

  def __init__(self, device: int, size: int):
    first = DeviceGP(device)
    self.members = [first] + [DeviceGP(device, stream=first.stream) for _ in range(size - 1)]
    self.device = first.device
    self._lib = first._lib
    self.n = self.dc = self.dk = 0

  @property
  def stream(self):
    return self.members[0].stream

  @property
  def launch_count(self) -> int:
    return sum(m.launch_count for m in self.members)

  def synchronize(self):
    self.members[0].synchronize()

  def _handles(self):
    arr = (C.c_void_p * len(self.members))(*[m._h for m in self.members])
    return arr

  def fit(self, x, y, params: Sequence[GPHyperParams], z=None, n_valid=None) -> int:
    assert len(params) == len(self.members)
    retries = 0
    for m, p in zip(self.members, params):
      retries = max(retries, m.fit(x, y, p, z=z, n_valid=n_valid))
    f = self.members[0]
    self.n, self.dc, self.dk = f.n, f.dc, f.dk
    return retries

  def score(self, xs, acq: Acquisition, zs=None, with_aux: bool = False) -> dict:
    f = self.members[0]
    xst, zst = f._xz(xs, zs)
    m = xst.shape[0]
    res = {'score': torch.empty((m,), dtype=torch.float64, device=self.device)}
    if with_aux:
      for k in ('mean', 'stddev', 'linf_distance'):
        res[k] = torch.empty((m,), dtype=torch.float64, device=self.device)
    f._use_acq(acq)                       # multi-handle calls take the acquisition of hs[0]
    a, keep = acq._c()
    _lib.check('vzgp_score_ensemble', self._lib.vzgp_score_ensemble(
        self._handles(), len(self.members), _ptr(xst), _ptr(zst), m, C.byref(a), _ptr(res['score']),
        _ptr(res.get('mean')), _ptr(res.get('stddev')), _ptr(res.get('linf_distance'))))
    res['_inputs'] = (xst, zst, keep)
    return res

  def score_qsets(self, xs_sets, q: int, qacq: QAcquisition, seed: int, zs=None, period: int = 0,
                  with_aux: bool = False, with_cov: bool = False) -> dict:
    """`DeviceGP.score_qsets` under the uniform mixture of the members ('cov' [E, n_sets, q, q] per member)."""
    return _score_qsets(self.members, xs_sets, q, qacq, seed, zs, period, with_aux, with_cov)

  def eagle_run(self, cfg, acq: Acquisition, count: int, seed: int, prior=None, prior_z=None, cat_sizes=None,
                other=None):
    assert other is None
    f = self.members[0]
    f._use_acq(acq)
    a, keep = acq._c()
    n_prior = 0 if prior is None else len(prior)
    pt = f._dev(prior, torch.float64) if n_prior > 0 and self.dc > 0 else None
    pz = f._dev(prior_z, torch.int32) if n_prior > 0 and self.dk > 0 else None
    bx = np.zeros((count, self.dc), np.float64)
    bz = np.zeros((count, self.dk), np.int32)
    bs = np.zeros(count, np.float64)
    sizes = np.ascontiguousarray(np.asarray(cat_sizes if cat_sizes is not None else [], np.int32))
    _lib.check('vzgp_eagle_run_ensemble', self._lib.vzgp_eagle_run_ensemble(
        self._handles(), len(self.members), C.byref(cfg), C.byref(a), _ptr(pt), _ptr(pz), n_prior,
        sizes.ctypes.data_as(C.POINTER(C.c_int32)) if sizes.size else None, count, seed,
        bx.ctypes.data_as(C.POINTER(C.c_double)), bz.ctypes.data_as(C.POINTER(C.c_int32)),
        bs.ctypes.data_as(C.POINTER(C.c_double))))
    del keep
    return bx, bz, bs

  def random_search(self, m: int, acq: Acquisition, count: int, seed: int, index_base: int = 0, cat_sizes=None):
    """RandomVectorizedStrategy over the ensemble: Philox pool -> mixture score -> device top-k."""
    f = self.members[0]
    xs = f.random_pool(m, self.dc, seed, index_base) if self.dc else torch.zeros((m, 0), dtype=torch.float64, device=self.device)
    zs = f.random_pool_cat(m, cat_sizes, seed, index_base) if self.dk else None
    out = self.score(xs, acq, zs=zs)
    idx, val = f.topk(out['score'], count)
    it = torch.from_numpy(np.maximum(idx, 0)).to(self.device)
    bx = xs[it].cpu().numpy()
    bz = zs[it].cpu().numpy() if zs is not None else np.zeros((count, 0), np.int32)
    return bx, bz, val, idx + index_base

  def posterior(self, xs, zs=None, add_noise: bool = True):
    """Per-member joint posteriors [(mean [M], cov [M, M])] (the mixture components)."""
    return [m.posterior(xs, zs, add_noise) for m in self.members]
