"""CPU oracle for the vectorised Eagle/Firefly acquisition optimiser and its driver.

TEST INFRASTRUCTURE ONLY (see oracle/gp_oracle.py header for the rules).

Restates, in NumPy, the continuous-feature path of
  vizier/_src/algorithms/optimizers/eagle_strategy.py   (a12-a14 in SURVEY 8a)
  vizier/_src/algorithms/optimizers/vectorized_base.py  (a11)
  vizier/_src/algorithms/optimizers/random_vectorized_optimizer.py
with n_parallel == 1.

Randomness.  The reference draws from JAX threefry (`jax.random.uniform`,
`laplace`, `split`); bit-matching it is out of scope (SURVEY 8c).  Parity is
stage-wise with INJECTED draws: every function takes its random numbers as
arrays.  For whole-loop comparisons the product and this oracle share one
counter-based generator, Philox4x32-10 (`philox_uniform` below, validated
against the Random123 known-answer vectors in tests/test_philox.py).

With n_parallel == 1 the reference's normalised Laplace noise
(eagle_strategy.py:1033-1044: noise / max|noise| over axis=1) is exactly
sign(noise) = +-1 per coordinate, so only a sign bit per coordinate is drawn.
"""

from __future__ import annotations

import dataclasses
from typing import Callable, Optional

import numpy as np

# EagleStrategyConfig defaults, eagle_strategy.py:139-167.
@dataclasses.dataclass(frozen=True)
class EagleConfig:
  visibility: float = 0.45
  gravity: float = 1.5
  negative_gravity: float = 0.008
  perturbation: float = 0.16
  perturbation_lower_bound: float = 7e-5
  penalize_factor: float = 0.7
  pool_size_exponent: float = 1.2
  pool_size: int = 0
  max_pool_size: int = 100
  normalization_scale: float = 0.5
  prior_trials_pool_pct: float = 0.96
  categorical_perturbation_factor: float = 1.0
  pure_categorical_perturbation_factor: float = 30.0
  prob_same_category_without_perturbation: float = 0.98
  mutate_normalization_type: int = 0   # 0 MEAN, 1 RANDOM (MutateNormalizationType, eagle_strategy.py:86-98)


def default_pool_size(n_features: int, batch_size: Optional[int], cfg: EagleConfig) -> int:
  """eagle_strategy.py:376-386."""
  pool = cfg.pool_size
  if pool == 0:
    pool = 10 + int(0.5 * n_features + n_features**cfg.pool_size_exponent)
    pool = min(pool, cfg.max_pool_size)
    if batch_size is not None:
      pool = int(np.ceil(pool / batch_size) * batch_size)
  return pool


# ----------------------------------------------------------------------------
# Philox4x32-10 (Salmon et al. 2011), shared with vizier_b200/csrc/philox.cuh
# ----------------------------------------------------------------------------
_M0 = np.uint64(0xD2511F53)
_M1 = np.uint64(0xCD9E8D57)
_W0 = np.uint32(0x9E3779B9)
_W1 = np.uint32(0xBB67AE85)

STREAM_INIT_POOL = 0
STREAM_PERTURB_SIGN = 1
STREAM_TRIM = 2
STREAM_RANDOM_POOL = 3  # RandomVectorizedStrategy candidate pool
STREAM_INIT_CAT = 4        # categorical features of the initial pool
STREAM_CAT_LAPLACE = 5     # categorical logit perturbation
STREAM_CAT_GUMBEL = 6      # Gumbel-max sampling of the mutated categories
STREAM_TRIM_CAT = 7        # categorical features of re-seeded flies
STREAM_RANDOM_POOL_CAT = 8
STREAM_PULL_RAND = 9        # RANDOM force normalisation weights (eagle_strategy.py:862-877)
STREAM_PUSH_RAND = 10
STREAM_SET_LAPLACE = 11      # continuous perturbations of set flies (n_parallel > 1)


def philox4x32(counter: np.ndarray, key: np.ndarray) -> np.ndarray:
  """counter [...,4] uint32, key [2] uint32 -> [...,4] uint32 (10 rounds)."""
  c = np.array(counter, dtype=np.uint32, copy=True)
  c0, c1, c2, c3 = (c[..., i].copy() for i in range(4))
  k0 = np.uint32(key[0])
  k1 = np.uint32(key[1])
  with np.errstate(over='ignore'):
    for _ in range(10):
      p0 = _M0 * c0.astype(np.uint64)
      p1 = _M1 * c2.astype(np.uint64)
      hi0 = (p0 >> np.uint64(32)).astype(np.uint32)
      lo0 = (p0 & np.uint64(0xFFFFFFFF)).astype(np.uint32)
      hi1 = (p1 >> np.uint64(32)).astype(np.uint32)
      lo1 = (p1 & np.uint64(0xFFFFFFFF)).astype(np.uint32)
      c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
      k0 = np.uint32(k0 + _W0)
      k1 = np.uint32(k1 + _W1)
  return np.stack([c0, c1, c2, c3], axis=-1)


def philox_uniform(seed: int, stream: int, iteration: int, n: int) -> np.ndarray:
  """n doubles in [0,1): element e uses counter (e, iteration, stream, 0).

  u = ((w0 >> 5) * 2^26 + (w1 >> 6)) / 2^53 from output words w0, w1.
  """
  e = np.arange(n, dtype=np.uint32)
  ctr = np.stack([
      e,
      np.full(n, iteration, np.uint32),
      np.full(n, stream, np.uint32),
      np.zeros(n, np.uint32),
  ], axis=-1)
  key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], dtype=np.uint32)
  out = philox4x32(ctr, key)
  a = (out[..., 0] >> np.uint32(5)).astype(np.float64)
  b = (out[..., 1] >> np.uint32(6)).astype(np.float64)
  return (a * 67108864.0 + b) / 9007199254740992.0


def philox_signs(seed: int, iteration: int, n: int) -> np.ndarray:
  """+-1 per coordinate: +1 if u >= 0.5 else -1."""
  u = philox_uniform(seed, STREAM_PERTURB_SIGN, iteration, n)
  return np.where(u >= 0.5, 1.0, -1.0)


# ----------------------------------------------------------------------------
# Strategy state and steps
# ----------------------------------------------------------------------------
@dataclasses.dataclass
class EagleState:
  iterations: int
  features: np.ndarray  # [P, D]
  rewards: np.ndarray  # [P]
  best_reward: float
  perturbations: np.ndarray  # [P]

  def copy(self) -> 'EagleState':
    return EagleState(self.iterations, self.features.copy(), self.rewards.copy(),
                      self.best_reward, self.perturbations.copy())


def features_dist_squared(batch: np.ndarray, pool: np.ndarray) -> np.ndarray:
  """Direct sum (a-b)^2 as in eagle_strategy_test.py:89-104 (`_create_features_simple`).

  The library code (eagle_strategy.py:451-455) uses |a|^2+|b|^2-2ab; both agree
  to ~1e-15 on [0,1]^D and the reference tests one against the other.
  """
  diff = batch[:, None, :] - pool[None, :, :]
  return np.sum(diff * diff, axis=-1)


def mask_flip(prior_features: np.ndarray, prior_rewards: np.ndarray):
  """eagle_strategy.py:472-496: valid entries newest-first, -inf ones last."""
  mask = ~np.isneginf(prior_rewards)
  idx = np.flip(np.argsort(np.where(mask, np.arange(prior_rewards.shape[0]), -1), kind='stable'))
  return prior_features[idx], prior_rewards[idx]


def populate_pool_with_prior_trials(
    random_pool: np.ndarray, prior_features: np.ndarray, prior_rewards: np.ndarray,
    cfg: EagleConfig,
) -> np.ndarray:
  """eagle_strategy.py:568-713.  random_pool [P, D] are the injected uniform draws."""
  pool_size = random_pool.shape[0]
  flipped_f, flipped_r = mask_flip(prior_features, prior_rewards)
  n_random = int(pool_size * (1 - cfg.prior_trials_pool_pct))
  init_features = random_pool[:n_random]
  left = pool_size - n_random
  random_features = random_pool[n_random:]
  features = flipped_f[:left].copy()
  rewards = flipped_r[:left].copy()
  for i in range(left, prior_rewards.shape[0]):
    d = features_dist_squared(flipped_f[i][None, :], features)[0]
    ind = int(np.argmin(d))
    if rewards[ind] < flipped_r[i]:
      features[ind] = flipped_f[i]
      rewards[ind] = flipped_r[i]
  chosen = rewards.shape[0]
  features = np.where(np.isneginf(rewards)[:, None], random_features[:chosen], features)
  features = np.concatenate([features, random_features[chosen:]], axis=0)
  return np.concatenate([init_features, features], axis=0)


def init_state(
    random_pool: np.ndarray, cfg: EagleConfig,
    prior_features: Optional[np.ndarray] = None, prior_rewards: Optional[np.ndarray] = None,
) -> EagleState:
  """eagle_strategy.py:527-565."""
  pool_size = random_pool.shape[0]
  if prior_features is not None and prior_rewards is not None and prior_features.shape[0] > 0:
    feats = populate_pool_with_prior_trials(random_pool, prior_features, prior_rewards, cfg)
  else:
    feats = random_pool.copy()
  return EagleState(0, feats, np.full(pool_size, -np.inf), -np.inf,
                    np.full(pool_size, cfg.perturbation))


def create_features(
    pool: np.ndarray, rewards: np.ndarray, batch: np.ndarray, rewards_batch: np.ndarray,
    perturbations: np.ndarray, cfg: EagleConfig, norm_dim: Optional[int] = None,
) -> np.ndarray:
  """eagle_strategy.py:784-952, MEAN normalisation, ADDITIVE perturbation.

  perturbations [B, D] already = sign * perturbation_i.  norm_dim: the number of feature dimensions of ONE point
  (eagle_strategy.py:830-837); differs from the flattened width for set flies (n_parallel > 1).
  """
  n_features = pool.shape[1] if norm_dim is None else norm_dim
  dists = features_dist_squared(batch, pool)
  with np.errstate(invalid='ignore'):
    directions = rewards[None, :] - rewards_batch[:, None]
  scaled_dir = np.where(directions >= 0.0, cfg.gravity, -cfg.negative_gravity)
  force = np.exp(-cfg.visibility * dists / n_features * 10.0)
  scaled_force = scaled_dir * force * np.isfinite(rewards).astype(np.float64)[None, :]
  pulls = np.maximum(scaled_force, 0.0)
  push = np.minimum(scaled_force, 0.0)
  with np.errstate(invalid='ignore', divide='ignore'):
    npull = cfg.normalization_scale * np.nan_to_num(
        pulls / np.sum(pulls > 0.0, axis=1, keepdims=True), nan=0.0)
    npush = cfg.normalization_scale * np.nan_to_num(
        push / np.sum(push < 0.0, axis=1, keepdims=True), nan=0.0)
  scale = npull + npush
  change = scale @ pool - batch * np.sum(scale, axis=-1, keepdims=True)
  return batch + change + perturbations


def suggest(state: EagleState, batch_size: int, signs: np.ndarray, cfg: EagleConfig,
            norm_dim: Optional[int] = None) -> np.ndarray:
  """eagle_strategy.py:720-782 incl. DefaultProjection clip to [0,1] (:257-268)."""
  pool_size = state.features.shape[0]
  nb = pool_size // batch_size
  start = (state.iterations % nb) * batch_size
  fb = state.features[start : start + batch_size]
  if state.iterations < nb:
    new = fb.copy()
  else:
    rb = state.rewards[start : start + batch_size]
    pb = state.perturbations[start : start + batch_size]
    new = create_features(state.features, state.rewards, fb, rb, signs * pb[:, None], cfg, norm_dim)
  return np.clip(new, 0.0, 1.0)


def batch_best(best_reward: float, batch_rewards: np.ndarray) -> float:
  """The best reward seen so far after one more batch, a NaN reward counting as -inf.

  Deliberate deviation (DESIGN.md 6b): the reference's `jnp.max` over a batch with a NaN is NaN, which becomes
  `best_reward` for the rest of the run, so `rewards != best_reward` holds for every fly and the best fly loses its
  protection from trimming.  NaN ranks as -inf everywhere else in the optimiser (update_best), and here as well."""
  r = np.where(np.isnan(batch_rewards), -np.inf, batch_rewards)
  return max(best_reward, float(np.max(r)))


def update(
    state: EagleState, batch_size: int, batch_features: np.ndarray, batch_rewards: np.ndarray,
    random_features: np.ndarray, cfg: EagleConfig,
) -> EagleState:
  """eagle_strategy.py:1075-1247 (update, _update_pool_features_and_rewards, _trim_pool)."""
  pool_size = state.features.shape[0]
  nb = pool_size // batch_size
  new_best = batch_best(state.best_reward, batch_rewards)
  start = (state.iterations % nb) * batch_size
  sl = slice(start, start + batch_size)
  pert = state.perturbations[sl]
  if state.iterations < nb:
    nf, nr, npert = batch_features, batch_rewards, pert
  else:
    prev_f, prev_r = state.features[sl], state.rewards[sl]
    improve = batch_rewards > prev_r
    nf = np.where(improve[:, None], batch_features, prev_f)
    nr = np.where(improve, batch_rewards, prev_r)
    npert = np.where(improve, pert, pert * cfg.penalize_factor)
    trim = (npert < cfg.perturbation_lower_bound) & (nr != new_best)
    nf = np.where(trim[:, None], random_features, nf)
    npert = np.where(trim, cfg.perturbation, npert)
    nr = np.where(trim, -np.inf, nr)
  out = state.copy()
  out.iterations = state.iterations + 1
  out.features[sl] = nf
  out.rewards[sl] = nr
  out.perturbations[sl] = npert
  out.best_reward = new_best
  return out


# ----------------------------------------------------------------------------
# Driver (vectorized_base.py:324-587)
# ----------------------------------------------------------------------------
def update_best(best_f, best_r, best_id, new_f, new_r, new_id, count):
  """Top-`count` of (new U best); ties -> smaller evaluation id (earlier)."""
  f = np.concatenate([new_f, best_f], axis=0)
  r = np.concatenate([new_r, best_r], axis=0)
  ids = np.concatenate([new_id, best_id], axis=0)
  rr = np.where(np.isnan(r), -np.inf, r)
  order = np.lexsort((ids, -rr))[:count]
  return f[order], r[order], ids[order]


def run_eagle_optimizer(
    score_fn: Callable[[np.ndarray], np.ndarray], *, dim: int, pool_size: int, batch_size: int,
    max_evaluations: int, count: int, seed: int, cfg: EagleConfig = EagleConfig(),
    prior_features: Optional[np.ndarray] = None, on_step: Optional[Callable[[int, EagleState], None]] = None,
):
  """VectorizedOptimizer.__call__ with the eagle strategy and Philox draws.  on_step(t, state) sees the strategy
  state after the update of step t (tests count trims and protected flies there)."""
  prior_rewards = None
  if prior_features is not None and prior_features.shape[0] > 0:
    prior_rewards = score_fn(prior_features)
  random_pool = philox_uniform(seed, STREAM_INIT_POOL, 0, pool_size * dim).reshape(pool_size, dim)
  state = init_state(random_pool, cfg, prior_features, prior_rewards)
  best_f = np.zeros((count, dim))
  best_r = np.full(count, -np.inf)
  best_id = np.full(count, np.iinfo(np.int64).max, dtype=np.int64)
  n_steps = (max_evaluations - 1) // batch_size + 1
  for t in range(n_steps):
    signs = philox_signs(seed, t, batch_size * dim).reshape(batch_size, dim)
    x = suggest(state, batch_size, signs, cfg)
    r = score_fn(x)
    rnd = philox_uniform(seed, STREAM_TRIM, t, batch_size * dim).reshape(batch_size, dim)
    state = update(state, batch_size, x, r, rnd, cfg)
    if on_step is not None:
      on_step(t, state)
    ids = np.arange(batch_size, dtype=np.int64) + t * batch_size
    best_f, best_r, best_id = update_best(best_f, best_r, best_id, x, r, ids, count)
  return best_f, best_r, state


def run_random_optimizer(score_fn, *, dim: int, num_candidates: int, count: int, seed: int):
  """RandomVectorizedStrategy with batch = max_evaluations = M (SURVEY 8a note)."""
  xs = philox_uniform(seed, STREAM_RANDOM_POOL, 0, num_candidates * dim).reshape(num_candidates, dim)
  r = score_fn(xs)
  rr = np.where(np.isnan(r), -np.inf, r)
  order = np.lexsort((np.arange(num_candidates), -rr))[:count]
  return xs[order], r[order], order


# ----------------------------------------------------------------------------
# Categorical features (eagle_strategy.py:936-1011, :1046-1073, :293-311)
# ----------------------------------------------------------------------------
def laplace_from_uniform(u: np.ndarray) -> np.ndarray:
  """Standard Laplace draw from u in [0,1) (inverse CDF; shared with csrc/eagle.cu)."""
  v = u - 0.5
  return -np.sign(v) * np.log(np.maximum(1.0 - 2.0 * np.abs(v), 1.1102230246251565e-16))


def gumbel_from_uniform(u: np.ndarray) -> np.ndarray:
  return -np.log(-np.log(np.maximum(u, 1e-300)))


def uniform_categories(u: np.ndarray, sizes: np.ndarray) -> np.ndarray:
  """DefaultRandomSampler: uniform over the valid categories of each feature (u [..., Dk])."""
  return np.minimum((u * sizes).astype(np.int32), np.asarray(sizes, np.int32) - 1)


def features_dist_squared_cat(batch, pool, batch_z, pool_z) -> np.ndarray:
  """eagle_strategy.py:458-468: squared distance + unweighted Hamming distance."""
  d = features_dist_squared(batch, pool) if batch.shape[1] else np.zeros((batch_z.shape[0], pool_z.shape[0]))
  if batch_z.shape[1]:
    d = d + np.sum(batch_z[:, None, :] != pool_z[None, :, :], axis=-1)
  return d


def force_scale(pool, rewards, batch, rewards_batch, cfg: EagleConfig, pool_z=None, batch_z=None,
                pull_u=None, push_u=None) -> np.ndarray:
  """The normalised force matrix `scale` [B, P] of _create_features (:811-899).

  MEAN mode, or RANDOM mode (:858-885) with injected uniform draws pull_u / push_u [B, P].  In RANDOM
  mode the reference masks both weight matrices with (pull > 0) - pushes get zero weight - and a
  fly without pulls gets 0/0 = NaN weights; we use zero weights there (deliberate deviation shared
  with the CUDA kernel, DESIGN.md)."""
  dk = 0 if pool_z is None else pool_z.shape[1]
  n_features = pool.shape[1] + dk
  if dk:
    dists = features_dist_squared_cat(batch, pool, batch_z, pool_z)
  else:
    dists = features_dist_squared(batch, pool)
  with np.errstate(invalid='ignore'):
    directions = rewards[None, :] - rewards_batch[:, None]
  scaled_dir = np.where(directions >= 0.0, cfg.gravity, -cfg.negative_gravity)
  force = np.exp(-cfg.visibility * dists / n_features * 10.0)
  scaled_force = scaled_dir * force * np.isfinite(rewards).astype(np.float64)[None, :]
  pulls = np.maximum(scaled_force, 0.0)
  push = np.minimum(scaled_force, 0.0)
  if cfg.mutate_normalization_type == 1:
    pos = (pulls > 0.0).astype(np.float64)
    r1, r2 = pull_u * pos, push_u * pos
    s1, s2 = r1.sum(axis=1, keepdims=True), r2.sum(axis=1, keepdims=True)
    w1 = np.where(s1 > 0, r1 / np.where(s1 > 0, s1, 1.0), 0.0)
    w2 = np.where(s2 > 0, r2 / np.where(s2 > 0, s2, 1.0), 0.0)
    return cfg.normalization_scale * pulls * w1 + cfg.normalization_scale * push * w2
  with np.errstate(invalid='ignore', divide='ignore'):
    npull = cfg.normalization_scale * np.nan_to_num(pulls / np.sum(pulls > 0.0, axis=1, keepdims=True), nan=0.0)
    npush = cfg.normalization_scale * np.nan_to_num(push / np.sum(push < 0.0, axis=1, keepdims=True), nan=0.0)
  return npull + npush


def categorical_logits(pool_z, batch_z, scale, sizes, cfg: EagleConfig) -> np.ndarray:
  """_create_logits_vector (:954-985) for every batch member and feature -> [B, Dk, max_size]."""
  b, dk = batch_z.shape
  max_size = int(max(sizes)) if dk else 0
  out = np.full((b, dk, max_size), -np.inf)
  log_same = np.log(cfg.prob_same_category_without_perturbation)
  for k in range(dk):
    s_k = int(sizes[k])
    with np.errstate(divide='ignore'):
      log_diff = np.log((1.0 - cfg.prob_same_category_without_perturbation) / (s_k - 1.0)) if s_k > 1 else np.inf
    for i in range(b):
      lg = np.array([np.sum(np.where(pool_z[:, k] == c, scale[i], 0.0)) for c in range(max_size)]) + log_diff
      lg = np.where(np.arange(max_size) < s_k, lg, -np.inf)
      with np.errstate(invalid='ignore'):    # a size-1 feature: inf - inf, and its logits are never sampled
        lg[batch_z[i, k]] += -np.sum(scale[i]) + log_same - log_diff
      out[i, k] = lg
  return out


def create_features_mixed(pool, pool_z, rewards, batch, batch_z, rewards_batch, perturbations, cat_noise,
                          gumbel, sizes, cfg: EagleConfig, pull_u=None, push_u=None):
  """_create_features with categorical features.  perturbations [B, Dc] (already scaled),
  cat_noise [B, Dk, max_size] = laplace * factor * perturbation_i, gumbel [B, Dk, max_size]."""
  scale = force_scale(pool, rewards, batch, rewards_batch, cfg, pool_z, batch_z, pull_u, push_u)
  change = scale @ pool - batch * np.sum(scale, axis=-1, keepdims=True)
  new_c = batch + change + perturbations
  logits = categorical_logits(pool_z, batch_z, scale, sizes, cfg) + cat_noise
  new_z = np.zeros_like(batch_z)
  for k in range(batch_z.shape[1]):
    s_k = int(sizes[k])
    if s_k == 1:
      new_z[:, k] = 0
    else:
      new_z[:, k] = np.argmax(logits[:, k, :s_k] + gumbel[:, k, :s_k], axis=-1)  # Gumbel-max = Categorical.sample
  return new_c, new_z


def run_eagle_optimizer_mixed(score_fn, *, dim: int, sizes, pool_size: int, batch_size: int, max_evaluations: int,
                              count: int, seed: int, cfg: EagleConfig = EagleConfig(), prior_c=None, prior_z=None,
                              on_step=None):
  """VectorizedOptimizer + eagle strategy with continuous AND categorical features, Philox draws.

  score_fn(xc [B,Dc], xz [B,Dk]) -> [B].  Element numbering of the draws is the contract shared
  with csrc/eagle.cu (see STREAM_* above): init (p*Dk+k), laplace/gumbel ((b*Dk+k)*Smax+c), trim (b*Dk+k).
  """
  sizes = np.asarray(sizes, np.int64)
  dk = sizes.shape[0]
  smax = int(sizes.max()) if dk else 0
  factor = cfg.categorical_perturbation_factor if dim > 0 else cfg.pure_categorical_perturbation_factor
  pool_c = philox_uniform(seed, STREAM_INIT_POOL, 0, pool_size * dim).reshape(pool_size, dim)
  pool_z = uniform_categories(philox_uniform(seed, STREAM_INIT_CAT, 0, pool_size * dk).reshape(pool_size, dk), sizes)
  if prior_c is not None and prior_c.shape[0] > 0:
    prior_r = score_fn(prior_c, prior_z)
    order = np.flip(np.arange(prior_r.shape[0]))        # no padded priors here: newest first
    fc, fz, fr = prior_c[order], prior_z[order], prior_r[order]
    n_random = int(pool_size * (1 - cfg.prior_trials_pool_pct))
    left = pool_size - n_random
    cc, cz, cr = fc[:left].copy(), fz[:left].copy(), fr[:left].copy()
    for i in range(left, fr.shape[0]):
      d = features_dist_squared_cat(fc[i][None, :], cc, fz[i][None, :], cz)[0]
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
      signs = philox_signs(seed, t, batch_size * dim).reshape(batch_size, dim)
      lap = laplace_from_uniform(philox_uniform(seed, STREAM_CAT_LAPLACE, t, batch_size * dk * smax)).reshape(batch_size, dk, smax)
      gum = gumbel_from_uniform(philox_uniform(seed, STREAM_CAT_GUMBEL, t, batch_size * dk * smax)).reshape(batch_size, dk, smax)
      pu = philox_uniform(seed, STREAM_PULL_RAND, t, batch_size * pool_size).reshape(batch_size, pool_size)
      qu = philox_uniform(seed, STREAM_PUSH_RAND, t, batch_size * pool_size).reshape(batch_size, pool_size)
      bc, bz = create_features_mixed(pool_c, pool_z, rewards, bc, bz, rewards[sl], signs * perts[sl][:, None],
                                     lap * factor * perts[sl][:, None, None], gum, sizes, cfg, pu, qu)
    bc = np.clip(bc, 0.0, 1.0)
    r = score_fn(bc, bz)
    new_best = batch_best(best_reward, r)
    if t < nb:
      pool_c[sl], pool_z[sl], rewards[sl] = bc, bz, r
    else:
      improve = r > rewards[sl]
      nc = np.where(improve[:, None], bc, pool_c[sl]); nz = np.where(improve[:, None], bz, pool_z[sl])
      nr = np.where(improve, r, rewards[sl]); npert = np.where(improve, perts[sl], perts[sl] * cfg.penalize_factor)
      trim = (npert < cfg.perturbation_lower_bound) & (nr != new_best)
      rc = philox_uniform(seed, STREAM_TRIM, t, batch_size * dim).reshape(batch_size, dim)
      rz = uniform_categories(philox_uniform(seed, STREAM_TRIM_CAT, t, batch_size * dk).reshape(batch_size, dk), sizes)
      pool_c[sl] = np.where(trim[:, None], rc, nc); pool_z[sl] = np.where(trim[:, None], rz, nz)
      rewards[sl] = np.where(trim, -np.inf, nr); perts[sl] = np.where(trim, cfg.perturbation, npert)
    best_reward = new_best
    if on_step is not None:     # as in run_eagle_optimizer; the state's features are the continuous ones
      on_step(t, EagleState(t + 1, pool_c, rewards, best_reward, perts).copy())
    ids = np.arange(batch_size, dtype=np.int64) + t * batch_size
    f = np.concatenate([bc, best_c]); z = np.concatenate([bz, best_z]); rr = np.concatenate([r, best_r]); ii = np.concatenate([ids, best_id])
    order = np.lexsort((ii, -np.where(np.isnan(rr), -np.inf, rr)))[:count]
    best_c, best_z, best_r, best_id = f[order], z[order], rr[order], ii[order]
  return best_c, best_z, best_r


# ----------------------------------------------------------------------------
# Set flies (n_parallel > 1): a fly is a set of q points scored together (vectorized_base.py:331-377, :108-122;
# eagle_strategy.py:1013-1046).  Flattened to [*, q * D]; distances and moves over all coordinates, forces normalised
# by D, perturbations = Laplace noise divided by its largest magnitude over the q members of each feature.
# ----------------------------------------------------------------------------
def set_perturbation_directions(seed: int, iteration: int, batch_size: int, q: int, dim: int) -> np.ndarray:
  """[B, q * D] normalised Laplace directions; element numbering b * q * D + m * D + f (shared with csrc/eagle_dev.cuh)."""
  u = philox_uniform(seed, STREAM_SET_LAPLACE, iteration, batch_size * q * dim).reshape(batch_size, q, dim)
  lap = laplace_from_uniform(u)
  big = np.max(np.abs(lap), axis=1, keepdims=True)
  with np.errstate(invalid='ignore', divide='ignore'):
    out = np.where(big > 0.0, lap / big, 0.0)
  return out.reshape(batch_size, q * dim)


def run_eagle_optimizer_sets(
    score_fn: Callable[[np.ndarray], np.ndarray], *, dim: int, n_parallel: int, pool_size: int, batch_size: int,
    max_evaluations: int, count: int, seed: int, cfg: EagleConfig = EagleConfig(),
    prior_features: Optional[np.ndarray] = None, on_step: Optional[Callable[[int, EagleState], None]] = None,
):
  """VectorizedOptimizer.__call__(n_parallel=q) with the eagle strategy and Philox draws.

  score_fn([B, q, D]) -> [B].  prior_features [n, D] are grouped into n // q consecutive sets
  (`_reshape_to_parallel_batches`, vectorized_base.py:108-122).  Returns (best sets [count, q, D], rewards, state).
  """
  q, width = n_parallel, n_parallel * dim
  prior_sets = prior_rewards = None
  if prior_features is not None and prior_features.shape[0] >= q:
    n_sets = prior_features.shape[0] // q
    prior_sets = prior_features[: n_sets * q].reshape(n_sets, width)
    prior_rewards = score_fn(prior_sets.reshape(n_sets, q, dim))
  random_pool = philox_uniform(seed, STREAM_INIT_POOL, 0, pool_size * width).reshape(pool_size, width)
  state = init_state(random_pool, cfg, prior_sets, prior_rewards)
  best_f = np.zeros((count, width))
  best_r = np.full(count, -np.inf)
  best_id = np.full(count, np.iinfo(np.int64).max, dtype=np.int64)
  n_steps = (max_evaluations - 1) // batch_size + 1
  for t in range(n_steps):
    dirs = set_perturbation_directions(seed, t, batch_size, q, dim)
    x = suggest(state, batch_size, dirs, cfg, norm_dim=dim)
    r = score_fn(x.reshape(batch_size, q, dim))
    rnd = philox_uniform(seed, STREAM_TRIM, t, batch_size * width).reshape(batch_size, width)
    state = update(state, batch_size, x, r, rnd, cfg)
    if on_step is not None:
      on_step(t, state)
    ids = np.arange(batch_size, dtype=np.int64) + t * batch_size
    best_f, best_r, best_id = update_best(best_f, best_r, best_id, x, r, ids, count)
  return best_f.reshape(count, q, dim), best_r, state
