"""The Eagle optimiser's remaining strategy options, for the tests of them.  No GPU import.

oracle/eagle_oracle.py restates the strategy with MEAN and RANDOM force normalisation and the ADDITIVE perturbation.
This module adds, from eagle_strategy.py:847-935, the two options the reference has beyond those:
  * mutate_normalization_type = 2 (UNNORMALIZED, :886-891): the raw pulls and pushes, in the continuous move and in
    the categorical logits;
  * ContinuousFeaturePerturbationType.MULTIPLICATIVE (:917-935): the new feature is moved * exp(perturbation)
    instead of moved + perturbation, before the clip to [0, 1].
The runners are eagle_oracle.run_eagle_optimizer_mixed (single points, with or without categorical features) and the
set runner of tests/set_flies_oracle.py with both options honoured; with MEAN or RANDOM and ADDITIVE they retrace
those runners (tests/test_eagle_options_host.py checks it).  `categorical_logits` is eagle_oracle.categorical_logits
with the sum over the pool as one product per feature, so that features of a thousand categories stay cheap.
"""
from typing import Callable, Optional

import numpy as np

from oracle import eagle_oracle as eo

ADDITIVE, MULTIPLICATIVE = 0, 1
MEAN, RANDOM, UNNORMALIZED = 0, 1, 2


def force_scale(pool, rewards, batch, rewards_batch, cfg: eo.EagleConfig, pool_z=None, batch_z=None, pull_u=None,
                push_u=None, norm_dim: Optional[int] = None) -> np.ndarray:
  """The force matrix `scale` [B, P] (eagle_strategy.py:811-899) in all three normalisations.  norm_dim: the feature
  dimensions of one point (set flies), by default every column of pool and pool_z."""
  dk = 0 if pool_z is None else pool_z.shape[1]
  n_features = pool.shape[1] + dk if norm_dim is None else norm_dim
  dists = eo.features_dist_squared_cat(batch, pool, batch_z, pool_z) if dk else eo.features_dist_squared(batch, pool)
  with np.errstate(invalid='ignore'):
    directions = rewards[None, :] - rewards_batch[:, None]
  scaled_dir = np.where(directions >= 0.0, cfg.gravity, -cfg.negative_gravity)
  force = np.exp(-cfg.visibility * dists / n_features * 10.0)
  scaled_force = scaled_dir * force * np.isfinite(rewards).astype(np.float64)[None, :]
  pulls = np.maximum(scaled_force, 0.0)
  push = np.minimum(scaled_force, 0.0)
  norm = cfg.mutate_normalization_type
  if norm == UNNORMALIZED:
    return pulls + push
  if norm == RANDOM:
    pos = (pulls > 0.0).astype(np.float64)
    r1, r2 = pull_u * pos, push_u * pos
    s1, s2 = r1.sum(axis=1, keepdims=True), r2.sum(axis=1, keepdims=True)
    w1 = np.where(s1 > 0, r1 / np.where(s1 > 0, s1, 1.0), 0.0)
    w2 = np.where(s2 > 0, r2 / np.where(s2 > 0, s2, 1.0), 0.0)
    return cfg.normalization_scale * pulls * w1 + cfg.normalization_scale * push * w2
  assert norm == MEAN, norm
  with np.errstate(invalid='ignore', divide='ignore'):
    npull = cfg.normalization_scale * np.nan_to_num(pulls / np.sum(pulls > 0.0, axis=1, keepdims=True), nan=0.0)
    npush = cfg.normalization_scale * np.nan_to_num(push / np.sum(push < 0.0, axis=1, keepdims=True), nan=0.0)
  return npull + npush


def move(pool, batch, scale, perturbations, perturbation_type: int) -> np.ndarray:
  """eagle_strategy.py:907-935: the moved features with the perturbation added, or multiplied in as exp(p)."""
  moved = batch + (scale @ pool - batch * np.sum(scale, axis=-1, keepdims=True))
  if perturbation_type == MULTIPLICATIVE:
    return moved * np.exp(perturbations)
  assert perturbation_type == ADDITIVE, perturbation_type
  return moved + perturbations


def categorical_logits(pool_z, batch_z, scale, sizes, cfg: eo.EagleConfig) -> np.ndarray:
  """eagle_oracle.categorical_logits (_create_logits_vector, :954-985) -> [B, Dk, max_size], any category count."""
  b, dk = batch_z.shape
  max_size = int(max(sizes)) if dk else 0
  out = np.full((b, dk, max_size), -np.inf)
  log_same = np.log(cfg.prob_same_category_without_perturbation)
  cats = np.arange(max_size)
  for k in range(dk):
    s_k = int(sizes[k])
    with np.errstate(divide='ignore'):
      log_diff = np.log((1.0 - cfg.prob_same_category_without_perturbation) / (s_k - 1.0)) if s_k > 1 else np.inf
    onehot = (pool_z[:, k][:, None] == cats[None, :]).astype(np.float64)        # [P, max_size]
    lg = scale @ onehot + log_diff
    lg = np.where(cats[None, :] < s_k, lg, -np.inf)
    with np.errstate(invalid='ignore'):    # a size-1 feature: inf - inf, and its logits are never sampled
      lg[np.arange(b), batch_z[:, k]] += -np.sum(scale, axis=1) + log_same - log_diff
    out[:, k] = lg
  return out


def run_mixed(score_fn, *, dim: int, sizes, pool_size: int, batch_size: int, max_evaluations: int, count: int,
              seed: int, cfg: eo.EagleConfig = eo.EagleConfig(), perturbation_type: int = ADDITIVE, prior_c=None,
              prior_z=None):
  """eagle_oracle.run_eagle_optimizer_mixed with all three normalisations and both perturbation types.
  score_fn(xc [B, Dc], xz [B, Dk]) -> [B].  Returns (best_c, best_z, best_r)."""
  sizes = np.asarray(sizes, np.int64)
  dk = sizes.shape[0]
  smax = int(sizes.max()) if dk else 0
  factor = cfg.categorical_perturbation_factor if dim > 0 else cfg.pure_categorical_perturbation_factor
  pool_c = eo.philox_uniform(seed, eo.STREAM_INIT_POOL, 0, pool_size * dim).reshape(pool_size, dim)
  pool_z = eo.uniform_categories(eo.philox_uniform(seed, eo.STREAM_INIT_CAT, 0, pool_size * dk).reshape(pool_size, dk),
                                 sizes)
  if prior_c is not None and prior_c.shape[0] > 0:
    prior_r = score_fn(prior_c, prior_z)
    order = np.flip(np.arange(prior_r.shape[0]))        # no padded priors here: newest first
    fc, fz, fr = prior_c[order], prior_z[order], prior_r[order]
    n_random = int(pool_size * (1 - cfg.prior_trials_pool_pct))
    left = pool_size - n_random
    cc, cz, cr = fc[:left].copy(), fz[:left].copy(), fr[:left].copy()
    for i in range(left, fr.shape[0]):
      d = eo.features_dist_squared_cat(fc[i][None, :], cc, fz[i][None, :], cz)[0]
      ind = int(np.argmin(d))
      if cr[ind] < fr[i]:
        cc[ind], cz[ind], cr[ind] = fc[i], fz[i], fr[i]
    n = cr.shape[0]
    pool_c[n_random:n_random + n] = cc
    pool_z[n_random:n_random + n] = cz
  rewards = np.full(pool_size, -np.inf)
  perts = np.full(pool_size, cfg.perturbation)
  best_reward = -np.inf
  best_c = np.zeros((count, dim)); best_z = np.zeros((count, dk), np.int32)
  best_r = np.full(count, -np.inf); best_id = np.full(count, np.iinfo(np.int64).max, dtype=np.int64)
  nb = pool_size // batch_size
  for t in range((max_evaluations - 1) // batch_size + 1):
    start = (t % nb) * batch_size
    sl = slice(start, start + batch_size)
    bc, bz = pool_c[sl].copy(), pool_z[sl].copy()
    if t >= nb:
      signs = eo.philox_signs(seed, t, batch_size * dim).reshape(batch_size, dim)
      pu = eo.philox_uniform(seed, eo.STREAM_PULL_RAND, t, batch_size * pool_size).reshape(batch_size, pool_size)
      qu = eo.philox_uniform(seed, eo.STREAM_PUSH_RAND, t, batch_size * pool_size).reshape(batch_size, pool_size)
      scale = force_scale(pool_c, rewards, bc, rewards[sl], cfg, pool_z, bz, pu, qu)
      new_c = move(pool_c, bc, scale, signs * perts[sl][:, None], perturbation_type)
      new_z = bz.copy()
      if dk:
        lap = eo.laplace_from_uniform(eo.philox_uniform(seed, eo.STREAM_CAT_LAPLACE, t, batch_size * dk * smax))
        gum = eo.gumbel_from_uniform(eo.philox_uniform(seed, eo.STREAM_CAT_GUMBEL, t, batch_size * dk * smax))
        logits = (categorical_logits(pool_z, bz, scale, sizes, cfg)
                  + lap.reshape(batch_size, dk, smax) * factor * perts[sl][:, None, None])
        gum = gum.reshape(batch_size, dk, smax)
        for k in range(dk):
          s_k = int(sizes[k])
          new_z[:, k] = 0 if s_k == 1 else np.argmax(logits[:, k, :s_k] + gum[:, k, :s_k], axis=-1)
      bc, bz = new_c, new_z
    bc = np.clip(bc, 0.0, 1.0)
    r = score_fn(bc, bz)
    new_best = eo.batch_best(best_reward, r)
    if t < nb:
      pool_c[sl], pool_z[sl], rewards[sl] = bc, bz, r
    else:
      improve = r > rewards[sl]
      nc = np.where(improve[:, None], bc, pool_c[sl]); nz = np.where(improve[:, None], bz, pool_z[sl])
      nr = np.where(improve, r, rewards[sl]); npert = np.where(improve, perts[sl], perts[sl] * cfg.penalize_factor)
      trim = (npert < cfg.perturbation_lower_bound) & (nr != new_best)
      rc = eo.philox_uniform(seed, eo.STREAM_TRIM, t, batch_size * dim).reshape(batch_size, dim)
      rz = eo.uniform_categories(eo.philox_uniform(seed, eo.STREAM_TRIM_CAT, t, batch_size * dk).reshape(batch_size, dk),
                                 sizes)
      pool_c[sl] = np.where(trim[:, None], rc, nc); pool_z[sl] = np.where(trim[:, None], rz, nz)
      rewards[sl] = np.where(trim, -np.inf, nr); perts[sl] = np.where(trim, cfg.perturbation, npert)
    best_reward = new_best
    ids = np.arange(batch_size, dtype=np.int64) + t * batch_size
    f = np.concatenate([bc, best_c]); z = np.concatenate([bz, best_z]); rr = np.concatenate([r, best_r])
    ii = np.concatenate([ids, best_id])
    order = np.lexsort((ii, -np.where(np.isnan(rr), -np.inf, rr)))[:count]
    best_c, best_z, best_r, best_id = f[order], z[order], rr[order], ii[order]
  return best_c, best_z, best_r


def run_sets(score_fn: Callable[[np.ndarray], np.ndarray], *, dim: int, n_parallel: int, pool_size: int,
             batch_size: int, max_evaluations: int, count: int, seed: int, cfg: eo.EagleConfig = eo.EagleConfig(),
             perturbation_type: int = ADDITIVE, prior_features: Optional[np.ndarray] = None):
  """tests/set_flies_oracle.run_sets with all three normalisations and both perturbation types.
  score_fn([B, q, D]) -> [B].  Returns (best sets [count, q, D], rewards [count])."""
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
    sl = slice((t % nb) * batch_size, (t % nb) * batch_size + batch_size)
    fb = state.features[sl]
    if t < nb:
      x = np.clip(fb, 0.0, 1.0)
    else:
      pu = eo.philox_uniform(seed, eo.STREAM_PULL_RAND, t, batch_size * pool_size).reshape(batch_size, pool_size)
      qu = eo.philox_uniform(seed, eo.STREAM_PUSH_RAND, t, batch_size * pool_size).reshape(batch_size, pool_size)
      scale = force_scale(state.features, state.rewards, fb, state.rewards[sl], cfg, pull_u=pu, push_u=qu, norm_dim=dim)
      x = np.clip(move(state.features, fb, scale, dirs * state.perturbations[sl][:, None], perturbation_type), 0.0, 1.0)
    r = score_fn(x.reshape(batch_size, q, dim))
    rnd = eo.philox_uniform(seed, eo.STREAM_TRIM, t, batch_size * width).reshape(batch_size, width)
    state = eo.update(state, batch_size, x, r, rnd, cfg)
    ids = np.arange(batch_size, dtype=np.int64) + t * batch_size
    best_f, best_r, best_id = eo.update_best(best_f, best_r, best_id, x, r, ids, count)
  return best_f.reshape(count, q, dim), best_r
