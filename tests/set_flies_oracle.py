"""The Eagle optimiser's set form (n_parallel = q points per fly) in both force normalisations, for the tests of set
flies.  No GPU import.

oracle/eagle_oracle.run_eagle_optimizer_sets restates the set form with MEAN normalisation.  GP-UCB-PE's default Eagle
config, which its set-PE batches run, normalises RANDOM (eagle_strategy.py:858-885).  `run_sets` is the same driver
with both modes, built from the oracle's steps:
  * MEAN: eagle_oracle.suggest with the forces normalised over one point's Dc dimensions;
  * RANDOM: the weights of eagle_oracle.force_scale with uniforms from Philox streams 9 and 10 at element b * P + j,
    the numbering of csrc/eagle_dev.cuh;
  * q = 1: the single-point sign perturbation (stream 1), which is what the kernel draws for a one-point fly.
With MEAN and q > 1 it is run_eagle_optimizer_sets; with RANDOM and q = 1 it is run_eagle_optimizer_mixed without
categorical features (tests/test_set_flies_host.py checks both).
"""
from typing import Callable, Optional

import numpy as np

from oracle import eagle_oracle as eo


def random_force_scale(pool, rewards, batch, rewards_batch, cfg: eo.EagleConfig, pull_u, push_u, norm_dim: int):
  """eagle_oracle.force_scale in RANDOM mode with the force exponent normalised by norm_dim (one point's Dc)."""
  dists = eo.features_dist_squared(batch, pool)
  with np.errstate(invalid='ignore'):
    directions = rewards[None, :] - rewards_batch[:, None]
  scaled_dir = np.where(directions >= 0.0, cfg.gravity, -cfg.negative_gravity)
  force = np.exp(-cfg.visibility * dists / norm_dim * 10.0)
  scaled_force = scaled_dir * force * np.isfinite(rewards).astype(np.float64)[None, :]
  pulls = np.maximum(scaled_force, 0.0)
  push = np.minimum(scaled_force, 0.0)
  pos = (pulls > 0.0).astype(np.float64)
  r1, r2 = pull_u * pos, push_u * pos
  s1, s2 = r1.sum(axis=1, keepdims=True), r2.sum(axis=1, keepdims=True)
  w1 = np.where(s1 > 0, r1 / np.where(s1 > 0, s1, 1.0), 0.0)
  w2 = np.where(s2 > 0, r2 / np.where(s2 > 0, s2, 1.0), 0.0)
  return cfg.normalization_scale * pulls * w1 + cfg.normalization_scale * push * w2


def run_sets(score_fn: Callable[[np.ndarray], np.ndarray], *, dim: int, n_parallel: int, pool_size: int,
             batch_size: int, max_evaluations: int, count: int, seed: int, cfg: eo.EagleConfig = eo.EagleConfig(),
             prior_features: Optional[np.ndarray] = None):
  """eagle_oracle.run_eagle_optimizer_sets with cfg.mutate_normalization_type honoured.  score_fn([B, q, D]) -> [B].
  Returns (best sets [count, q, D], rewards [count])."""
  q, width = n_parallel, n_parallel * dim
  prior_sets = prior_rewards = None
  if prior_features is not None and prior_features.shape[0] >= q:
    n_sets = prior_features.shape[0] // q
    prior_sets = prior_features[: n_sets * q].reshape(n_sets, width)
    prior_rewards = score_fn(prior_sets.reshape(n_sets, q, dim))
  random_pool = eo.philox_uniform(seed, eo.STREAM_INIT_POOL, 0, pool_size * width).reshape(pool_size, width)
  state = eo.init_state(random_pool, cfg, prior_sets, prior_rewards)
  best_f = np.zeros((count, width))
  best_r = np.full(count, -np.inf)
  best_id = np.full(count, np.iinfo(np.int64).max, dtype=np.int64)
  nb = pool_size // batch_size
  for t in range((max_evaluations - 1) // batch_size + 1):
    if q == 1:
      dirs = eo.philox_signs(seed, t, batch_size * dim).reshape(batch_size, dim)
    else:
      dirs = eo.set_perturbation_directions(seed, t, batch_size, q, dim)
    if cfg.mutate_normalization_type == 1 and t >= nb:
      sl = slice((t % nb) * batch_size, (t % nb) * batch_size + batch_size)
      pool, fb = state.features, state.features[sl]
      pu = eo.philox_uniform(seed, eo.STREAM_PULL_RAND, t, batch_size * pool_size).reshape(batch_size, pool_size)
      qu = eo.philox_uniform(seed, eo.STREAM_PUSH_RAND, t, batch_size * pool_size).reshape(batch_size, pool_size)
      scale = random_force_scale(pool, state.rewards, fb, state.rewards[sl], cfg, pu, qu, dim)
      change = scale @ pool - fb * np.sum(scale, axis=-1, keepdims=True)
      x = np.clip(fb + change + dirs * state.perturbations[sl][:, None], 0.0, 1.0)
    else:
      x = eo.suggest(state, batch_size, dirs, cfg, norm_dim=dim)
    r = score_fn(x.reshape(batch_size, q, dim))
    rnd = eo.philox_uniform(seed, eo.STREAM_TRIM, t, batch_size * width).reshape(batch_size, width)
    state = eo.update(state, batch_size, x, r, rnd, cfg)
    ids = np.arange(batch_size, dtype=np.int64) + t * batch_size
    best_f, best_r, best_id = eo.update_best(best_f, best_r, best_id, x, r, ids, count)
  return best_f.reshape(count, q, dim), best_r
