"""NumPy oracle of Pareto dominance, Pareto rank and the randomized cumulative hypervolume from the origin.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE (see oracle/gp_oracle.py).

Definitions (every metric maximised), restated from the reference's documented semantics:
  * row a dominates row p when every p_k <= a_k; strictly, when in addition some a_k > p_k.  Comparisons with NaN are
    false, so a row with a NaN coordinate neither dominates nor is dominated;
  * a point is optimal against a set when no row of the set dominates it; the frontier of a set is the rows optimal
    against the set itself under strict dominance;
  * the Pareto rank of a row is the number of rows of the set that strictly dominate it;
  * the cumulative hypervolume from the origin (arXiv 2006.04655, Section 3, Lemma 5) of points [N, M] over direction
    vectors [V, M] is out[i] = mean_u (max_{j <= i} min_k points[j, k] / u[k])^M, NaN propagating through the min and
    the running max as NumPy's minimum / maximum do.
Work is done in blocks of rows so that no temporary grows past a few tens of MB.
"""

from __future__ import annotations

import numpy as np

_BLOCK_ELEMS = 1 << 22


def _blocks(points: np.ndarray, against: np.ndarray, strict: bool):
  """Yields (first row, bool [b, B2]) blocks of the domination matrix: entry (i, j) is True when row j of `against`
  dominates row i of `points`."""
  points = np.asarray(points, dtype=np.float64)
  against = np.asarray(against, dtype=np.float64)
  b1, m = points.shape
  step = max(1, _BLOCK_ELEMS // max(1, against.shape[0] * m))
  for lo in range(0, b1, step):
    p = points[lo:lo + step, None, :]                 # [b, 1, M]
    a = against[None, :, :]                           # [1, B2, M]
    dominated = np.logical_and.reduce(p <= a, axis=2)
    if strict:
      dominated &= np.logical_or.reduce(a > p, axis=2)
    yield lo, dominated


def domination_matrix(points: np.ndarray, against: np.ndarray, strict: bool) -> np.ndarray:
  """bool [B1, B2]: entry (i, j) is True when row j of `against` dominates row i of `points`."""
  out = np.zeros((len(points), len(against)), dtype=bool)
  for lo, d in _blocks(points, against, strict):
    out[lo:lo + len(d)] = d
  return out


def is_pareto_optimal_against(points: np.ndarray, against: np.ndarray, strict: bool) -> np.ndarray:
  """bool [B1]: True where no row of `against` dominates the row of `points`."""
  out = np.ones(len(points), dtype=bool)
  for lo, d in _blocks(points, against, strict):
    out[lo:lo + len(d)] = ~np.any(d, axis=1)
  return out


def is_frontier(ys: np.ndarray) -> np.ndarray:
  """bool [B]: the rows of `ys` that no row of `ys` strictly dominates (all pairs)."""
  return is_pareto_optimal_against(ys, ys, strict=True)


def pareto_rank(ys: np.ndarray) -> np.ndarray:
  """int32 [B]: how many rows of `ys` strictly dominate each row."""
  out = np.zeros(len(ys), dtype=np.int32)
  for lo, d in _blocks(ys, ys, strict=True):
    out[lo:lo + len(d)] = np.sum(d, axis=1)
  return out


def cum_hypervolume_origin(points: np.ndarray, vectors: np.ndarray) -> np.ndarray:
  """float64 [N]: the randomized cumulative hypervolume of `points` from the origin over `vectors`."""
  points = np.asarray(points, dtype=np.float64)
  vectors = np.asarray(vectors, dtype=np.float64)
  if points.shape[1] != vectors.shape[1]:
    raise ValueError(f'points {points.shape} and vectors {vectors.shape} differ in dimension')
  n, m = points.shape
  total = np.zeros(n)
  step = max(1, _BLOCK_ELEMS // max(1, n * m))
  for lo in range(0, vectors.shape[0], step):
    u = vectors[lo:lo + step]                                   # [v, M]
    ratio = np.min(points[None, :, :] / u[:, None, :], axis=2)  # [v, N]
    running = np.maximum.accumulate(ratio, axis=1)
    total += np.sum(running ** m, axis=0)
  with np.errstate(invalid='ignore', divide='ignore'):
    return total / vectors.shape[0]
