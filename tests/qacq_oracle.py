"""NumPy oracle of the parallel (q-) acquisitions QEI / QPI / QUCB over sets of q points (acquisitions.py:495-568
[R]; TFP ParallelExpectedImprovement, ParallelProbabilityOfImprovement, ParallelUpperConfidenceBound [T]), restating
vizier_b200/csrc/score_q.cu draw for draw.  [R]: read in the reference; [T]: TFP behaviour, not verifiable here.

  * [T] QEI = mean_s max_j max(f_sj - best - 0.01, 0) (default exploration 0.01); QPI = mean_s [max_j f_sj - best > 0];
    QUCB = mean_s max_j (mu_j + c |f_sj - mu_j|).  No observation (best -inf): QEI and QPI score mean_s max_j f_sj.
  * [T] the predictive GPRM samples through the model's retrying_cholesky (jitter 1e-4, 5 retries); a set whose
    factor still fails scores NaN.  Its covariance is K** - V^T V + sn2 I (predictive noise = observation noise).
  * [R] ensembles are the uniform mixture (stochastic_process_model.py:846-868): every (set, sample) draws one member.
  * [R] one acquisition seed per optimiser run (vectorized_base.py:382-404): draws depend on a set's position
    p = index mod period.  Normals: Philox stream 12, uniforms 2e and 2e + 1, e = (p S + s) q + j (Box-Muller);
    member: stream 13, element p S + s.
  * Samples are summed per thread s = t + 256 k in order, then reduced by the device's warp-shuffle tree.

Built on the model oracle (oracle/gp_oracle.py: kernel, predict, L-inf distance) and its Philox
(oracle/eagle_oracle.py: philox4x32)."""
from typing import Optional, Sequence

import numpy as np
import scipy.linalg as sla

from oracle import eagle_oracle as eo
from oracle import gp_oracle as go

STREAM_QACQ_NORMAL = 12      # Monte Carlo normals (Box-Muller pairs); the optimiser's streams are 0-11
STREAM_QACQ_MEMBER = 13      # ensemble member of each (set position, sample)


def philox_uniform_at(seed: int, stream: int, iteration: int, elements) -> np.ndarray:
  """philox_uniform at arbitrary element indices (uint64; the high word goes to counter word 3, as on the device)."""
  e = np.asarray(elements, np.uint64)
  ctr = np.stack([
      (e & np.uint64(0xFFFFFFFF)).astype(np.uint32),
      np.full(e.shape, iteration, np.uint32),
      np.full(e.shape, stream, np.uint32),
      (e >> np.uint64(32)).astype(np.uint32),
  ], axis=-1)
  key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], dtype=np.uint32)
  out = eo.philox4x32(ctr, key)
  a = (out[..., 0] >> np.uint32(5)).astype(np.float64)
  b = (out[..., 1] >> np.uint32(6)).astype(np.float64)
  return (a * 67108864.0 + b) / 9007199254740992.0


def qacq_normals(seed: int, elements) -> np.ndarray:
  """Standard normals of the q-acquisitions (Box-Muller): element e takes uniforms 2e and 2e + 1 of
  STREAM_QACQ_NORMAL, z = sqrt(-2 log(1 - u1)) cos(2 pi u2)."""
  e = np.asarray(elements, np.uint64)
  u1 = philox_uniform_at(seed, STREAM_QACQ_NORMAL, 0, np.uint64(2) * e)
  u2 = philox_uniform_at(seed, STREAM_QACQ_NORMAL, 0, np.uint64(2) * e + np.uint64(1))
  return np.sqrt(-2.0 * np.log(1.0 - u1)) * np.cos(2.0 * np.pi * u2)


def predictive_covariance(pred: go.Predictive, xs, zs=None) -> np.ndarray:
  """Joint posterior predictive covariance at xs [m, D] (zs [m, Dk]): K** - V^T V + sn2 I (the GPRM of
  stochastic_process_model.py:800-868 with predictive noise = observation noise [T])."""
  xs = np.asarray(xs, np.float64)
  ks = go.kernel(pred.params, xs, pred.x, zs, pred.z, pred.cont_dim_valid, pred.cat_dim_valid)
  ks = ks * pred.row_valid[None, :]
  v = sla.solve_triangular(pred.chol, ks.T, lower=True)
  kss = go.kernel(pred.params, xs, xs, zs, zs, pred.cont_dim_valid, pred.cat_dim_valid)
  return kss - v.T @ v + pred.params.observation_noise_variance * np.eye(xs.shape[0])


QACQ_QEI, QACQ_QPI, QACQ_QUCB = 0, 1, 2
QEI_EXPLORATION = 0.01
QACQ_JITTER, QACQ_MAX_RETRIES = 1e-4, 5
QACQ_THREADS = 256


def qacq_cholesky(cov: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
  """cov [n, q, q] -> (L [n, q, q], ok [n]): right-looking Cholesky of cov + shift I with shifts 0, 1e-4, 1e-3, ...
  (QACQ_MAX_RETRIES retries); L is NaN where every shift failed."""
  cov = np.asarray(cov, np.float64)
  n, q, _ = cov.shape
  out = np.full_like(cov, np.nan)
  ok = np.zeros(n, bool)
  shift = 0.0
  with np.errstate(all='ignore'):
    for _ in range(QACQ_MAX_RETRIES + 1):
      todo = np.nonzero(~ok)[0]
      if todo.size == 0:
        break
      c = np.tril(cov[todo]) + shift * np.eye(q)
      good = np.ones(todo.size, bool)
      for k in range(q):
        d = c[:, k, k]
        good &= (d > 0.0) & np.isfinite(d)
        l = np.sqrt(np.where(good, d, 1.0))
        c[:, k, k] = l
        c[:, k + 1:, k] /= l[:, None]
        for i in range(k + 1, q):
          c[:, i, k + 1:i + 1] -= c[:, i, k][:, None] * c[:, k + 1:i + 1, k]
      out[todo[good]] = np.tril(c[good])
      ok[todo[good]] = True
      shift = QACQ_JITTER if shift == 0.0 else shift * 10.0
  return out, ok


def _block_sum(vals: np.ndarray) -> np.ndarray:
  """vals [n, S] -> [n]: the device's per-thread ordered sums and warp-shuffle tree (device.cuh block_sum)."""
  n, s = vals.shape
  k = -(-s // QACQ_THREADS)
  padded = np.zeros((n, k * QACQ_THREADS))
  padded[:, :s] = vals
  padded = padded.reshape(n, k, QACQ_THREADS)
  acc = np.zeros((n, QACQ_THREADS))
  for i in range(k):
    acc = acc + padded[:, i, :]

  def tree(v):   # [n, w, 32] -> [n, w]: lane 0 of __shfl_down_sync by 16, 8, 4, 2, 1
    v = v.copy()
    for o in (16, 8, 4, 2, 1):
      v[..., :o] = v[..., :o] + v[..., o:2 * o]
    return v[..., 0]

  red = tree(acc.reshape(n, QACQ_THREADS // 32, 32))
  lanes = np.zeros((n, 1, 32))
  lanes[:, 0, :red.shape[1]] = red
  return tree(lanes)[:, 0]


def qacq_from_moments(mean, cov, *, kind: int, best_label: float = -np.inf, coefficient: float = 1.8,
                      num_samples: int = 100, seed: int = 0, period: Optional[int] = None):
  """Monte Carlo stage: mean [E, n, q], cov [E, n, q, q] -> (score [n], mixture mean [n, q], mixture stddev [n, q])."""
  mean = np.asarray(mean, np.float64)
  cov = np.asarray(cov, np.float64)
  e_count, n, q = mean.shape
  s_count = int(num_samples)
  period = n if not period or period <= 0 else int(period)
  chol, ok = qacq_cholesky(cov.reshape(e_count * n, q, q))
  chol = chol.reshape(e_count, n, q, q)
  ok = ok.reshape(e_count, n).all(axis=0)
  mix_mean = mean.sum(axis=0) / e_count
  diag = np.diagonal(cov, axis1=-2, axis2=-1)
  mix_var = diag[0] if e_count == 1 else (diag + mean * mean).sum(axis=0) / e_count - mix_mean ** 2
  pos = (np.arange(n, dtype=np.uint64) % np.uint64(period))
  ps = pos[:, None] * np.uint64(s_count) + np.arange(s_count, dtype=np.uint64)[None, :]     # [n, S]
  if e_count > 1:
    u = philox_uniform_at(seed, STREAM_QACQ_MEMBER, 0, ps)
    member = np.minimum((u * e_count).astype(np.int64), e_count - 1)
  else:
    member = np.zeros(ps.shape, np.int64)
  z = qacq_normals(seed, ps[:, :, None] * np.uint64(q) + np.arange(q, dtype=np.uint64))   # [n, S, q]
  sets = np.arange(n)[:, None]
  f = mean[member, sets].copy()                                                            # [n, S, q]
  with np.errstate(all='ignore'):
    for k in range(q):
      lk = chol[member, sets, k:, k]                                                       # [n, S, q - k]
      f[:, :, k:] = f[:, :, k:] + lk * z[:, :, k:k + 1]
    if kind == QACQ_QUCB:
      vals = np.max(mix_mean[:, None, :] + coefficient * np.abs(f - mix_mean[:, None, :]), axis=-1)
    else:
      vals = np.max(f, axis=-1)
      if np.isfinite(best_label):
        vals = np.maximum(vals - best_label - QEI_EXPLORATION, 0.0) if kind == QACQ_QEI else (vals - best_label > 0.0).astype(np.float64)
    score = _block_sum(vals) / s_count
  score = np.where(ok, score, np.nan)
  return score, mix_mean, np.sqrt(np.maximum(mix_var, 0.0))


def set_moments(preds: Sequence[go.Predictive], sets, zs_sets=None):
  """Per-member set moments: sets [n, q, D] (zs_sets [n, q, Dk]) -> mean [E, n, q], cov [E, n, q, q]."""
  sets = np.asarray(sets, np.float64)
  n, q, d = sets.shape
  flat = sets.reshape(n * q, d)
  zflat = None if zs_sets is None else np.asarray(zs_sets).reshape(n * q, -1)
  means, covs = [], []
  for p in preds:
    means.append(go.predict(p, flat, zflat)[0].reshape(n, q))
    covs.append(np.stack([predictive_covariance(p, sets[s], None if zs_sets is None else np.asarray(zs_sets)[s])
                          for s in range(n)]))
  return np.stack(means), np.stack(covs)


def qacq_score(preds: Sequence[go.Predictive], sets, zs_sets=None, *, kind: int, best_label: float = -np.inf,
               coefficient: float = 1.8, num_samples: int = 100, seed: int = 0, period: Optional[int] = None,
               use_trust_region: bool = False, trust_radius_value: float = 1.0, tr_dim_mask=None, tr_rows=None):
  """q-acquisition of sets [n, q, D] under the uniform mixture of `preds` (one model: a list of one), plus the set
  trust-region term of gp_ucb_pe.py:245-269 against the first tr_rows trials of preds[0].  Returns (score [n],
  aux {'mean', 'stddev', 'linf_distance' [n * q], 'cov' [E, n, q, q]})."""
  sets = np.asarray(sets, np.float64)
  n, q, d = sets.shape
  mean, cov = set_moments(preds, sets, zs_sets)
  score, mu, sd = qacq_from_moments(mean, cov, kind=kind, best_label=best_label, coefficient=coefficient,
                                    num_samples=num_samples, seed=seed, period=period)
  if tr_dim_mask is None:
    tr_dim_mask = np.ones(d, bool)
  n_tr = int(np.sum(preds[0].row_valid)) if tr_rows is None else tr_rows
  dist = go.min_linf_distance(sets.reshape(n * q, d), preds[0].x[:n_tr], tr_dim_mask)
  if use_trust_region:
    dq = dist.reshape(n, q)
    score = score + np.sum(((dq > trust_radius_value) & (trust_radius_value <= 0.5)) * (-1e4 - dq), axis=1)
  return score, {'mean': mu.reshape(-1), 'stddev': sd.reshape(-1), 'linf_distance': dist, 'cov': cov}
