"""ctypes binding of libvzgp.so (the C ABI in include/vzgp.h).

The product path has NO CPU fallback: if the CUDA library is missing or a call
fails, an exception is raised.  PyTorch is used only as a device-memory handle
(`tensor.data_ptr()`), never for arithmetic on this path.
"""

from __future__ import annotations

import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
# VZGP_LIB: an alternative build of the same library (instrumented debug builds, tools/i8_timing.py)
LIB_PATH = os.environ.get('VZGP_LIB') or os.path.join(_HERE, '_lib', 'libvzgp.so')

VZGP_ERR_ARG = -1
VZGP_ERR_CUDA = -2
VZGP_ERR_STATE = -3
VZGP_ERR_UNSUPPORTED = -4


class VzgpError(RuntimeError):
  """A libvzgp call returned a negative status."""

  def __init__(self, fn: str, status: int, message: str):
    super().__init__(f'{fn} failed with status {status}: {message}')
    self.status = status


class Params(C.Structure):
  _fields_ = [
      ('signal_variance', C.c_double),
      ('observation_noise_variance', C.c_double),
      ('continuous_length_scale_squared', C.POINTER(C.c_double)),
      ('categorical_length_scale_squared', C.POINTER(C.c_double)),
      ('linear_coef', C.c_double),
      ('linear_slope_amplitude', C.c_double),
      ('linear_shift', C.c_double),
      ('mean_constant', C.c_double),
  ]


class Acq(C.Structure):
  _fields_ = [
      ('ucb_coefficient', C.c_double),
      ('use_trust_region', C.c_int),
      ('trust_radius', C.c_double),
      ('tr_dim_mask', C.POINTER(C.c_uint8)),
      ('tr_rows', C.c_int),
      ('tr_strict', C.c_int),
  ]


ACQ_UCB, ACQ_LCB, ACQ_EI, ACQ_PI, ACQ_MES = 0, 1, 2, 3, 4   # vzgp_acq_kind
MES_MAX_SAMPLES = 256


class AcqTerm(C.Structure):
  _fields_ = [
      ('kind', C.c_int),
      ('coefficient', C.c_double),
      ('best_label', C.c_double),
      ('exploration', C.c_double),
  ]


class AcqFn(C.Structure):
  _fields_ = [
      ('main', AcqTerm),
      ('use_threshold', C.c_int),
      ('thresholding', AcqTerm),
      ('threshold', C.c_double),
      ('bad_acq_value', C.c_double),
  ]


QACQ_QEI, QACQ_QPI, QACQ_QUCB = 0, 1, 2   # vzgp_qacq_kind


class QAcq(C.Structure):
  _fields_ = [
      ('kind', C.c_int),
      ('best_label', C.c_double),
      ('coefficient', C.c_double),
      ('num_samples', C.c_int),
      ('period', C.c_int),
      ('use_trust_region', C.c_int),
      ('trust_radius', C.c_double),
      ('tr_dim_mask', C.POINTER(C.c_uint8)),
      ('tr_rows', C.c_int),
      ('cov_out', C.c_void_p),
  ]


class PeParams(C.Structure):
  _fields_ = [
      ('mode', C.c_int),
      ('ucb_coefficient', C.c_double),
      ('explore_coefficient', C.c_double),
      ('penalty_coefficient', C.c_double),
      ('threshold', C.c_double),
      ('use_trust_region', C.c_int),
      ('trust_radius', C.c_double),
      ('tr_dim_mask', C.POINTER(C.c_uint8)),
      ('tr_rows', C.c_int),
  ]


class Scalarization(C.Structure):
  _fields_ = [
      ('n_metrics', C.c_int),
      ('n_scalarizations', C.c_int),
      ('weights', C.POINTER(C.c_double)),
      ('reference_point', C.POINTER(C.c_double)),
      ('max_scalarized', C.POINTER(C.c_double)),
      ('ucb_coefficient', C.c_double),
  ]


REGION_AVERAGE, REGION_UNION, REGION_INTERSECTION = 0, 1, 2   # vzgp_region_penalty


class PeMultiParams(C.Structure):
  _fields_ = [
      ('mode', C.c_int),
      ('ucb_coefficient', C.c_double),
      ('explore_coefficient', C.c_double),
      ('penalty_coefficient', C.c_double),
      ('use_trust_region', C.c_int),
      ('trust_radius', C.c_double),
      ('tr_dim_mask', C.POINTER(C.c_uint8)),
      ('tr_rows', C.c_int),
      ('n_metrics', C.c_int),
      ('thresholds', C.POINTER(C.c_double)),
      ('region_penalty', C.c_int),
      ('scalarization', C.POINTER(Scalarization)),
  ]


class EagleConfig(C.Structure):
  _fields_ = [
      ('visibility', C.c_double),
      ('gravity', C.c_double),
      ('negative_gravity', C.c_double),
      ('perturbation', C.c_double),
      ('perturbation_lower_bound', C.c_double),
      ('penalize_factor', C.c_double),
      ('normalization_scale', C.c_double),
      ('prior_trials_pool_pct', C.c_double),
      ('pool_size', C.c_int),
      ('batch_size', C.c_int),
      ('max_evaluations', C.c_int),
      ('categorical_perturbation_factor', C.c_double),
      ('pure_categorical_perturbation_factor', C.c_double),
      ('prob_same_category_without_perturbation', C.c_double),
      ('mutate_normalization_type', C.c_int),
      ('n_parallel', C.c_int),
  ]

  def __init__(self, *args, **kwargs):
    super().__init__(*args, **kwargs)
    if len(args) < 12 and 'categorical_perturbation_factor' not in kwargs:
      self.categorical_perturbation_factor = 1.0
    if len(args) < 13 and 'pure_categorical_perturbation_factor' not in kwargs:
      self.pure_categorical_perturbation_factor = 30.0
    if len(args) < 14 and 'prob_same_category_without_perturbation' not in kwargs:
      self.prob_same_category_without_perturbation = 0.98


class Adam(C.Structure):
  _fields_ = [
      ('learning_rate', C.c_double),
      ('b1', C.c_double),
      ('b2', C.c_double),
      ('eps', C.c_double),
      ('eps_root', C.c_double),
      ('epochs', C.c_int),
  ]


_vp = C.c_void_p
_i = C.c_int
_i64 = C.c_int64
_u64 = C.c_uint64
_d = C.c_double
_pd = C.POINTER(C.c_double)
_pi64 = C.POINTER(C.c_int64)
_pi32 = C.POINTER(C.c_int32)
_pP = C.POINTER(Params)
_pA = C.POINTER(Acq)
_pE = C.POINTER(EagleConfig)
_pPE = C.POINTER(PeParams)

# name -> (restype, argtypes).  Must list every symbol declared in include/vzgp.h
# (tests/test_abi.py checks this against the header).
SIGNATURES = {
    'vzgp_last_error': (C.c_char_p, []),
    'vzgp_version': (_i, []),
    'vzgp_device_count': (_i, []),
    'vzgp_create': (_i, [_i, _vp, C.POINTER(_vp)]),
    'vzgp_destroy': (_i, [_vp]),
    'vzgp_synchronize': (_i, [_vp]),
    'vzgp_launch_count': (_i64, [_vp]),
    'vzgp_set_int': (_i, [_vp, C.c_char_p, _i]),
    'vzgp_get_int': (_i, [_vp, C.c_char_p, C.POINTER(C.c_int64)]),
    'vzgp_set_acquisition': (_i, [_vp, C.POINTER(AcqFn)]),
    'vzgp_mes_fit': (_i, [_vp, C.c_double, _i, C.c_uint64, _vp]),
    'vzgp_set_mes': (_i, [_vp, _vp, _i]),
    'vzgp_kernel_matrix': (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _pP, _d, _vp, _i]),
    'vzgp_cross_kernel': (_i, [_vp, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _pP, _vp, _i]),
    'vzgp_cholesky_retry': (_i, [_vp, _vp, _i, _i, _d, _i, _vp, _i, _pd]),
    'vzgp_factor_inverse': (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _i]),
    'vzgp_tri_inverse': (_i, [_vp, _vp, _i, _i, _vp, _i]),
    'vzgp_fit': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _pP]),
    'vzgp_fit_multi': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _pP]),
    'vzgp_nll_grad_multi': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _pP, _pd, _pd]),
    'vzgp_nll_grad_batch': (_i, [C.POINTER(_vp), _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, C.POINTER(Params), C.POINTER(C.c_uint8), _pd, _pd, C.POINTER(_i)]),
    'vzgp_ard_adam_small_supported': (_i, [_i, _i, _i]),
    'vzgp_ard_adam_small': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _pd, _pd, _pd, C.POINTER(Adam), _pd, _pd,
                                 C.POINTER(_i), _pd]),
    'vzgp_score_multi': (_i, [_vp, _vp, _vp, _i, C.POINTER(Scalarization), _vp, _vp, _vp]),
    'vzgp_eagle_run_multi': (_i, [_vp, _pE, C.POINTER(Scalarization), _vp, _vp, _i, _pi32, _i, _u64, _pd, _pi32, _pd]),
    'vzgp_fit_separable': (_i, [C.POINTER(_vp), _i, _vp, _vp, _vp, _i, _i, _i, _i, _pP, _pd]),
    'vzgp_nll_grad_separable_batch': (_i, [C.POINTER(_vp), _i, _i, _vp, _vp, _vp, _i, _i, _i, _i, C.POINTER(Params), _pd,
                                           C.POINTER(C.c_uint8), _pd, _pd, _pd, C.POINTER(_i)]),
    'vzgp_score_separable': (_i, [C.POINTER(_vp), _i, _vp, _vp, _i, C.POINTER(Scalarization), _vp, _vp, _vp]),
    'vzgp_eagle_run_separable': (_i, [C.POINTER(_vp), _i, _pE, C.POINTER(Scalarization), _vp, _vp, _i, _pi32, _i, _u64,
                                      _pd, _pi32, _pd]),
    'vzgp_posterior_separable': (_i, [C.POINTER(_vp), _i, _vp, _vp, _i, _i, _vp, _vp, _i]),
    'vzgp_get_cholesky': (_i, [_vp, _vp, _i]),
    'vzgp_get_alpha': (_i, [_vp, _vp]),
    'vzgp_nll_grad': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _pP, _pd, _pd]),
    'vzgp_score': (_i, [_vp, _vp, _vp, _i, _pA, _vp, _vp, _vp, _vp]),
    'vzgp_clamped_count': (_i, [_vp, _pi64]),
    'vzgp_score_host': (_i, [_vp, _vp, _vp, _i, _pA, _vp, _vp, _vp, _vp]),
    'vzgp_posterior': (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _i]),
    'vzgp_posterior_multi': (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _i]),
    'vzgp_topk': (_i, [_vp, _vp, _i64, _i, _pi64, _pd]),
    'vzgp_score_topk': (_i, [_vp, _vp, _vp, _i, _pA, _i, _vp, _pd, _pd, _pi64]),
    'vzgp_score_ensemble': (_i, [C.POINTER(_vp), _i, _vp, _vp, _i, _pA, _vp, _vp, _vp, _vp]),
    'vzgp_score_grad': (_i, [_vp, _vp, _i, _pA, _vp, _vp, _vp, _vp, _vp]),
    'vzgp_score_grad_ensemble': (_i, [C.POINTER(_vp), _i, _vp, _i, _pA, _vp, _vp, _vp, _vp, _vp]),
    'vzgp_eagle_run_ensemble': (_i, [C.POINTER(_vp), _i, C.POINTER(EagleConfig), _pA, _vp, _vp, _i, _pi32, _i, C.c_uint64, _pd, _pi32, _pd]),
    'vzgp_score_topk_pack': (_i, [_vp, _vp, _vp, _i, _pA, _i, _i64, _vp, _vp]),
    'vzgp_merge_topk': (_i, [_vp, _vp, _i, _i, _i, _vp, _vp]),
    'vzgp_exchange_create': (_i, [_vp, _i, _i, _i, _i, C.POINTER(_vp)]),
    'vzgp_exchange_destroy': (_i, [_vp]),
    'vzgp_exchange_ipc_handle': (_i, [_vp, _vp]),
    'vzgp_exchange_open': (_i, [_vp, _vp]),
    'vzgp_exchange_base': (_vp, [_vp]),
    'vzgp_exchange_set_peers': (_i, [_vp, C.POINTER(_vp)]),
    'vzgp_nccl_unique_id': (_i, [_vp]),
    'vzgp_exchange_nccl_init': (_i, [_vp, _vp]),
    'vzgp_allgather_topk': (_i, [_vp, _vp, _vp, _vp, _vp, _i]),
    'vzgp_exchange_status': (_i, [_vp, _vp, C.POINTER(_i)]),
    'vzgp_suggest_host': (_i, [_vp, _vp, _i, _vp, _i, _pA, _i, _i64, _vp, _vp]),
    'vzgp_eagle_run': (_i, [_vp, _pE, _pA, _vp, _vp, _i, _pi32, _i, _u64, _pd, _pi32, _pd]),
    'vzgp_score_pe': (_i, [_vp, _vp, _vp, _vp, _i, _pPE, _vp, _vp, _vp, _vp]),
    'vzgp_eagle_run_pe': (_i, [_vp, _vp, _pE, _pPE, _vp, _vp, _i, _pi32, _i, _u64, _pd, _pi32, _pd]),
    'vzgp_score_pe_ensemble': (_i, [C.POINTER(_vp), C.POINTER(_vp), _i, _vp, _vp, _i, _pPE, _vp, _vp, _vp, _vp]),
    'vzgp_eagle_run_pe_ensemble': (_i, [C.POINTER(_vp), C.POINTER(_vp), _i, _pE, _pPE, _vp, _vp, _i, _pi32, _i, _u64,
                                        _pd, _pi32, _pd]),
    'vzgp_score_pe_multi': (_i, [_vp, _vp, _vp, _vp, _i, C.POINTER(PeMultiParams), _vp, _vp, _vp, _vp]),
    'vzgp_eagle_run_pe_multi': (_i, [_vp, _vp, _pE, C.POINTER(PeMultiParams), _vp, _vp, _i, _pi32, _i, _u64, _pd, _pi32,
                                     _pd]),
    'vzgp_score_stack': (_i, [C.POINTER(C.c_void_p), _i, _pd, _vp, _vp, _i, _pA, _vp, _vp, _vp, _vp]),
    'vzgp_eagle_run_stack': (_i, [C.POINTER(C.c_void_p), _i, _pd, _pE, _pA, _vp, _vp, _i, _pi32, _i, _u64, _pd, _pi32, _pd]),
    'vzgp_score_stack_ensemble': (_i, [C.POINTER(C.c_void_p), _i, _i, _pd, _vp, _vp, _i, _pA, _vp, _vp, _vp, _vp]),
    'vzgp_eagle_run_stack_ensemble': (_i, [C.POINTER(C.c_void_p), _i, _i, _pd, _pE, _pA, _vp, _vp, _i, _pi32, _i, _u64,
                                           _pd, _pi32, _pd]),
    'vzgp_score_stack_multi': (_i, [C.POINTER(C.c_void_p), _i, _pd, _vp, _vp, _i, C.POINTER(Scalarization), _vp, _vp,
                                    _vp]),
    'vzgp_eagle_run_stack_multi': (_i, [C.POINTER(C.c_void_p), _i, _pd, _pE, C.POINTER(Scalarization), _vp, _vp, _i,
                                        _pi32, _i, _u64, _pd, _pi32, _pd]),
    'vzgp_score_set_pe': (_i, [_vp, _vp, _vp, _i, _i, _pPE, _vp, _vp, _vp, _vp]),
    'vzgp_score_qsets': (_i, [C.POINTER(_vp), _i, _vp, _vp, _i, _i, C.POINTER(QAcq), _u64, _vp, _vp, _vp, _vp]),
    'vzgp_qacq_from_moments': (_i, [_vp, _i, _i, _i, _vp, _vp, C.POINTER(QAcq), _u64, _vp]),
    'vzgp_eagle_begin': (_i, [_vp, _pE, _pi32, _i, _u64, _i, C.POINTER(C.c_void_p)]),
    'vzgp_eagle_seed': (_i, [_vp, _vp, _vp]),
    'vzgp_eagle_ask': (_i, [_vp, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]),
    'vzgp_eagle_tell': (_i, [_vp]),
    'vzgp_eagle_end': (_i, [_vp, _pd, _pi32, _pd]),
    'vzgp_random_search': (_i, [_vp, _i64, _i64, _pA, _pi32, _i, _u64, _pd, _pi32, _pd, _pi64]),
    'vzgp_random_pool': (_i, [_vp, _i64, _i, _i64, _u64, _vp]),
    'vzgp_random_pool_cat': (_i, [_vp, _i64, _i, _pi32, _i64, _u64, _vp]),
    'vzgp_pareto_optimal_against': (_i, [_vp, _vp, _i, _vp, _i, _i, _i, _vp]),
    'vzgp_pareto_rank': (_i, [_vp, _vp, _i, _i, _vp]),
    'vzgp_cum_hypervolume_origin': (_i, [_vp, _vp, _i, _i, _vp, _i, _vp]),
}

_lock = threading.Lock()
_lib = None


def load() -> C.CDLL:
  """Loads libvzgp.so (once).  Raises ImportError loudly if it is not built."""
  global _lib
  with _lock:
    if _lib is not None:
      return _lib
    if not os.path.exists(LIB_PATH):
      raise ImportError(
          f'{LIB_PATH} is missing: build it with `python -c "import __graft_entry__ as g; '
          'g.build()"` (or `make -C vizier_b200/csrc`).  vizier_b200 has no CPU fallback.'
      )
    lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    for name, (res, args) in SIGNATURES.items():
      fn = getattr(lib, name)  # AttributeError if the symbol is not exported
      fn.restype = res
      fn.argtypes = args
    _lib = lib
    return lib


def check(fn: str, status: int) -> int:
  """Raises VzgpError for negative statuses; returns non-negative ones."""
  if status < 0:
    msg = load().vzgp_last_error()
    raise VzgpError(fn, status, msg.decode('utf-8', 'replace') if msg else '')
  return status
