"""Pareto frontiers, Pareto ranks and randomized hypervolume of multi-objective studies, computed on the device.

Mirrors the public names of the reference's
  * `vizier/_src/jax/xla_pareto.py`: `is_frontier`, `get_frontier`, `pareto_rank`, `jax_cum_hypervolume_origin` and
    `JaxParetoOptimalAlgorithm` (here `DeviceParetoOptimalAlgorithm`),
  * `vizier/_src/pyvizier/multimetric/hypervolume.py`: `ParetoFrontier`,
with the same argument meaning.  Every metric is maximised: row a dominates row p when all(p <= a), and strictly when
also any(a > p).  A row with a NaN coordinate neither dominates nor is dominated, as in `jnp`.

Inputs may be NumPy arrays (or anything `np.asarray` takes), returned as NumPy, or fp64 CUDA tensors, returned as
tensors on the same device; the kind of the first argument decides.  The comparisons, the ranks and the hypervolume
sums run in libvzgp (`vzgp_pareto_optimal_against`, `vzgp_pareto_rank`, `vzgp_cum_hypervolume_origin`); there is no
CPU fallback.  At most 64 metrics and 2^30 rows per set.  The functions may be called from several threads: they share
one handle per device and take its lock while they enqueue their launches.
"""

from __future__ import annotations

import ctypes as C
import math
import threading
from typing import Callable, Optional

import numpy as np
import torch

from vizier_b200 import _lib
from vizier_b200 import gp

MAX_METRICS = 64

_handles: dict = {}
_handles_lock = threading.Lock()


def _device_gp(device: torch.device):
  """The handle these calls use on `device` (they need no fitted model), and the lock that serialises its use.

  One handle serves every thread of the process, and its hypervolume keeps its partial sums in handle memory between
  two launches; each call therefore enqueues its launches under the lock, so that calls from different threads reach
  the handle's stream one after the other."""
  index = device.index if device.index is not None else torch.cuda.current_device()
  with _handles_lock:
    if index not in _handles:
      _handles[index] = (gp.DeviceGP(index), threading.Lock())
    return _handles[index]


def _points(a, name: str):
  """`a` as a 2-D fp64 array or CUDA tensor [rows, metrics]; raises before any device work."""
  if isinstance(a, torch.Tensor):
    if not a.is_cuda or a.dtype != torch.float64:
      raise TypeError(f'{name}: tensors must be float64 CUDA tensors, got {a.dtype} on {a.device}')
  else:
    a = np.asarray(a, dtype=np.float64)
  if a.ndim != 2:
    raise ValueError(f'{name} must be 2-D [num_points, num_metrics], got shape {tuple(a.shape)}')
  if not 1 <= a.shape[1] <= MAX_METRICS:
    raise ValueError(f'{name} has {a.shape[1]} metrics; 1 to {MAX_METRICS} are supported')
  return a


def _device_of(*arrays) -> torch.device:
  for a in arrays:
    if isinstance(a, torch.Tensor):
      return a.device
  return torch.device('cuda', torch.cuda.current_device())


def _run(first, inputs, out_shape, out_dtype, call):
  """Copies `inputs` to the device, runs `call(dev, *device_inputs, out)` on the handle's stream and returns `out`
  as the kind of `first`."""
  device = _device_of(*inputs)
  dev, lock = _device_gp(device)
  with torch.cuda.device(device):
    with lock:
      ts = [dev._dev(a, torch.float64) for a in inputs]   # pylint: disable=protected-access
      out = torch.empty(out_shape, dtype=out_dtype, device=device)
      dev.stream.wait_stream(torch.cuda.current_stream(device))
      call(dev, *ts, out)
      torch.cuda.current_stream(device).wait_stream(dev.stream)
  if isinstance(first, torch.Tensor):
    return out
  return out.cpu().numpy()


def _ptr(t: torch.Tensor):
  return C.c_void_p(t.data_ptr())


def is_pareto_optimal_against(points, against, *, strict: bool):
  """Boolean [B1]: True where no row of `against` [B2, M] dominates the row of `points` [B1, M] (strictly when
  `strict`).  With B2 = 0 every row is optimal."""
  points = _points(points, 'points')
  against = _points(against, 'against')
  if against.shape[1] != points.shape[1]:
    raise ValueError(f'points have {points.shape[1]} metrics but against has {against.shape[1]}')
  n, m = points.shape

  def call(dev, p, a, out):
    _lib.check('vzgp_pareto_optimal_against', dev._lib.vzgp_pareto_optimal_against(   # pylint: disable=protected-access
        dev._h, _ptr(p), n, _ptr(a), a.shape[0], m, 1 if strict else 0, _ptr(out)))    # pylint: disable=protected-access

  out = _run(points, [points, against], (n,), torch.uint8, call)
  return out.bool() if isinstance(out, torch.Tensor) else out.astype(bool)


def is_frontier(ys, *, num_shards: int = 10, verbose: bool = False):
  """Boolean [B]: the Pareto-optimal rows of `ys` [B, M] (strict dominance), in one pass.  `num_shards` and
  `verbose` are accepted for the reference's signature; the device needs no sharding, and the result does not depend
  on them."""
  del num_shards, verbose
  ys = _points(ys, 'ys')
  return is_pareto_optimal_against(ys, ys, strict=True)


def get_frontier(ys, *, num_shards: int = 10, verbose: bool = True):
  """The Pareto-optimal rows of `ys` [B, M], in their original order (`ys[is_frontier(ys)]`)."""
  ys = _points(ys, 'ys')
  return ys[is_frontier(ys, num_shards=num_shards, verbose=verbose)]


def pareto_rank(ys):
  """int32 [B]: for each row of `ys` [B, M], the number of rows that strictly dominate it."""
  ys = _points(ys, 'ys')
  n, m = ys.shape

  def call(dev, p, out):
    _lib.check('vzgp_pareto_rank', dev._lib.vzgp_pareto_rank(dev._h, _ptr(p), n, m, _ptr(out)))   # pylint: disable=protected-access

  return _run(ys, [ys], (n,), torch.int32, call)


def cum_hypervolume_origin(points, vectors):
  """float64 [B]: out[i] = mean over the rows u of `vectors` [V, M] of (max_{j <= i} min_k points[j, k] / u[k])^M,
  the randomized cumulative hypervolume of `points` [B, M] from the origin (arXiv 2006.04655, Section 3, Lemma 5),
  unnormalised.  NaN propagates as in NumPy; V = 0 gives NaN, the mean of nothing."""
  points = _points(points, 'points')
  vectors = _points(vectors, 'vectors')
  if vectors.shape[1] != points.shape[1]:
    raise ValueError(f'points have {points.shape[1]} metrics but the vectors have {vectors.shape[1]}')
  n, m = points.shape
  v = vectors.shape[0]

  def call(dev, p, u, out):
    if v == 0:
      out.fill_(float('nan'))
      return
    _lib.check('vzgp_cum_hypervolume_origin', dev._lib.vzgp_cum_hypervolume_origin(   # pylint: disable=protected-access
        dev._h, _ptr(p), n, m, _ptr(u), v, _ptr(out)))   # pylint: disable=protected-access

  return _run(points, [points, vectors], (n,), torch.float64, call)


jax_cum_hypervolume_origin = cum_hypervolume_origin


class DeviceParetoOptimalAlgorithm:
  """`pareto_optimal.BaseParetoOptimalAlgorithm` on the device; usable as the `base_algorithm` of the reference's
  `FastParetoOptimalAlgorithm`.  Takes and returns NumPy arrays."""

  def is_pareto_optimal(self, points: np.ndarray) -> np.ndarray:
    return np.asarray(is_frontier(np.asarray(points, dtype=np.float64)), dtype=bool)

  def is_pareto_optimal_against(self, points: np.ndarray, against: np.ndarray, *, strict: bool) -> np.ndarray:
    return np.asarray(is_pareto_optimal_against(np.asarray(points, dtype=np.float64),
                                                np.asarray(against, dtype=np.float64), strict=strict), dtype=bool)

  def update_pareto_optimal(self, current_pareto_optimal: np.ndarray, incremental_points: np.ndarray) -> np.ndarray:
    """Indices of the Pareto-optimal rows of the current frontier followed by the new points."""
    is_optimal = self.is_pareto_optimal(np.append(current_pareto_optimal, incremental_points, axis=0))
    return np.asarray(is_optimal).nonzero()[0]


def _orthant_fraction_of_unit_ball(m: int) -> float:
  """Volume of the part of the unit ball in R^m with every coordinate positive."""
  return math.pi ** (m / 2) / math.gamma(m / 2 + 1) / 2 ** m


class ParetoFrontier:
  """Randomized hypervolume of a set of points above an origin (`hypervolume.ParetoFrontier`), with the
  cumulative hypervolume from the origin computed on the device by default."""

  def __init__(self, points: np.ndarray, origin: np.ndarray, num_vectors: int = 10000,
               cum_hypervolume_base: Callable[[np.ndarray, np.ndarray], np.ndarray] = cum_hypervolume_origin):
    """`points` [N, M], `origin` [M]; `num_vectors` random directions in the positive orthant (NumPy's global
    generator, as in the reference); `cum_hypervolume_base(points, vectors)` is the cumulative hypervolume from the
    origin.  Raises ValueError when the points and the origin differ in dimension."""
    if points.shape[1] != len(origin):
      raise ValueError(f'Dimension mismatch: points have {points.shape[1]} metrics, the origin {len(origin)}')
    self._points = points
    self._origin = origin
    self._cum_hypervolume_base = cum_hypervolume_base
    directions = np.abs(np.random.normal(size=(num_vectors, len(origin))))
    self._vectors = directions / np.linalg.norm(directions, axis=1, keepdims=True)

  def hypervolume(self, additional_points: Optional[np.ndarray] = None, is_cumulative: bool = False,
                  num_shards: int = 10) -> np.ndarray:
    """The dominated hypervolume of the points (and `additional_points`, appended), or with `is_cumulative` its
    running value over the first i points.  The vectors are taken in `num_shards` shards, each shard's curve made
    non-decreasing before the shards are averaged."""
    if additional_points is not None and additional_points.shape[1] != self._points.shape[1]:
      raise ValueError(f'Dimension mismatch: additional points have {additional_points.shape[1]} metrics, the '
                       f'frontier points {self._points.shape[1]}')
    stacked = self._points if additional_points is None else np.concatenate((self._points, additional_points))
    # Measured from the origin; a row not strictly above it in every metric counts as the origin itself.
    shifted = stacked - self._origin
    shifted[~np.all(shifted > 0, axis=1)] = 0
    if shifted.size == 0:
      return np.asarray([0.0])

    scale = _orthant_fraction_of_unit_ball(shifted.shape[1])
    bounds = np.linspace(0, len(self._vectors), num_shards + 1).astype(np.int32)
    total = 0
    for s in reversed(range(num_shards)):   # the reference adds the shards last to first
      curve = np.asarray(self._cum_hypervolume_base(shifted, self._vectors[bounds[s]:bounds[s + 1]]))
      total = total + np.maximum.accumulate(curve * scale)
    mean = total / num_shards
    return np.array(mean) if is_cumulative else np.array(np.max(mean))
