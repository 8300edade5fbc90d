"""Lock-step comparison of an Eagle optimiser with oracle/eagle_oracle.py, one batch at a time.  No GPU import.

The oracle's drivers call `score_fn` once for the prior trials and once per batch.  `run` uses that callback as the
lock-step point: it asks the optimiser under test for its batch, requires it to equal the oracle's (continuous
features within 1e-12, categories exactly), computes the rewards ONCE on the host from the oracle's batch and hands the
same numbers to both sides.  Round-off in a scorer therefore cannot separate the two trajectories: any difference is a
difference in the optimiser, and a wrong pool update shows in the batch in which the fly is next visited.

The optimiser under test is any object with
  seed(prior_c [n, q * Dc], prior_z [n, Dk], rewards [n])      only when the case has prior trials
  ask() -> (xc [B, q * Dc], xz [B, Dk])                        NumPy arrays
  tell(rewards [B])
  end() -> (best_c [count, q * Dc], best_z [count, Dk], best_r [count])
(tests/test_gpu_eagle_steps.py wraps vzgp_eagle_begin / seed / ask / tell / end, tests/test_eagle_lockstep_host.py a
NumPy stand-in).  `run(case, None)` runs the oracle alone and checks only the coverage of the case.

Rewards are synthetic and seeded (`Case.schedule`); each schedule asserts, on the oracle's side, that the branch it
exists for was reached, so a case cannot silently stop exercising it:
  decaying   r = f(x) - 2 t: nothing improves after the first pass, every fly but the best is trimmed on its 22nd
             visit with the default config
  quantised  r = f(x) rounded to eighths: ties inside a batch, against the stored winners and against a fly's own
             reward (rb == prev is not an improvement)
  nonfinite  NaN, +inf and -inf planted in chosen slots (a NaN while the pool fills, a whole-NaN batch, a NaN next to
             the run's best reward), cheap trimming: NaN ranks as -inf in the winners AND in best_reward
  improving  r = f(x) + 2 t: every visit improves, nothing is penalised or trimmed
"""
import dataclasses

import numpy as np

from oracle import eagle_oracle as eo

BIG = 50.0      # the planted best reward of the nonfinite schedule: above every f(x) and every f(x) + 2 t used here


@dataclasses.dataclass(frozen=True)
class Case:
  name: str
  schedule: str
  dc: int                 # continuous features of one point
  pool: int
  batch: int
  steps: int
  count: int
  sizes: tuple = ()       # categorical feature sizes
  q: int = 1              # n_parallel: points per fly
  n_prior: int = 0        # prior flies (sets of q points)
  norm: int = 0           # mutate_normalization_type: 0 MEAN, 1 RANDOM
  seed: int = 7

  @property
  def nb(self):
    return self.pool // self.batch

  @property
  def width(self):
    return self.q * self.dc

  @property
  def cfg(self) -> eo.EagleConfig:
    # the nonfinite schedule trims after 4 failed visits (0.16 * 0.7^4 < 0.05), the others keep the default 22
    lower = 0.05 if self.schedule == 'nonfinite' else eo.EagleConfig().perturbation_lower_bound
    return eo.EagleConfig(perturbation_lower_bound=lower, mutate_normalization_type=self.norm)


def decaying_steps(pool, batch):
  """First pass, 22 failed visits, then two more passes over flies that were trimmed."""
  return 25 * (pool // batch)


def nonfinite_steps(pool, batch):
  """The planted best reward arrives at step nb + 2 and its fly is protected from its 4th failed visit on."""
  return 5 * (pool // batch) + 11


def priors(case: Case):
  rng = np.random.default_rng(case.seed + 100)
  pc = rng.uniform(size=(case.n_prior, case.width))
  pz = np.stack([rng.integers(0, s, size=case.n_prior) for s in case.sizes], axis=1).astype(np.int32) \
      if case.sizes else np.zeros((case.n_prior, 0), np.int32)
  return pc, pz


def _f(xc, xz):
  """Smooth in every continuous coordinate, a step in every categorical one; values in [-1.1, 0]."""
  out = np.zeros(xc.shape[0])
  if xc.shape[1]:
    w = 1.0 + np.arange(xc.shape[1]) % 3
    out -= np.sum(w * (xc - 0.3) ** 2, axis=1) / np.sum(w)
  if xz.shape[1]:
    out -= 0.3 * np.mean(xz != 1, axis=1)
  return out


def rewards(case: Case, t: int, xc, xz):
  """Rewards of batch t (t = -1: the prior trials) under the case's schedule."""
  f, tt, nb, b = _f(xc, xz), max(t, 0), case.nb, case.batch
  if case.schedule == 'decaying':
    return f - 2.0 * tt
  if case.schedule == 'improving':
    return f + 2.0 * tt
  if case.schedule == 'quantised':
    return np.round(f * 8.0) / 8.0 + 0.0
  assert case.schedule == 'nonfinite' and b >= 2
  r = f.copy()
  if t == -1:
    r[0] = np.nan
  elif t == min(1, nb - 1):
    r[0] = np.nan                       # while the pool fills: the NaN becomes the fly's stored reward
  elif t == nb + 1:
    r[:] = np.nan
  elif t == nb + 2:
    r[0], r[1] = np.nan, BIG            # the run's best reward arrives in a batch that holds a NaN
  elif t == case.steps - 4:
    r[0] = np.inf
  elif t % 5 == 3:
    r[t % b] = -np.inf
  return r


class Watch:
  """The oracle drivers' on_step observer: counts, from the state after every update, what the cases assert on."""

  def __init__(self, pool, batch, steps, cfg):
    self.nb, self.batch, self.steps, self.cfg, self.prev = pool // batch, batch, steps, cfg, None
    self.trims, self.trim_steps, self.protected, self.neginf_steps, self.big_kept = 0, [], 0, 0, False
    self.nan_fly_visits = 0

  def __call__(self, t, state):
    c, cfg = self, self.cfg
    start = (t % c.nb) * c.batch
    sl = slice(start, start + c.batch)
    if t >= c.nb:
      # a fly leaves an update with the initial perturbation and reward -inf only by being trimmed in it
      n = int(np.sum(np.isneginf(state.rewards[sl]) & (state.perturbations[sl] == cfg.perturbation)
                     & (self.prev.perturbations[sl] < cfg.perturbation)))
      self.trims += n
      self.trim_steps += [t] * n
      # and keeps a perturbation below the bound only because it holds the best reward
      self.protected += int(np.sum(state.perturbations[sl] < cfg.perturbation_lower_bound))
      self.neginf_steps += bool(np.any(np.isneginf(self.prev.rewards)))    # what this step's suggest saw
      # a fly whose own reward is NaN: every direction is NaN, so nobody pulls it (zero weights in RANDOM mode)
      self.nan_fly_visits += int(np.sum(np.isnan(self.prev.rewards[sl])))
    if t == c.steps - 5:      # nonfinite: just before +inf takes over as the best reward
      self.big_kept = bool(np.any((state.rewards == BIG) & (state.perturbations < cfg.perturbation_lower_bound)))
    self.prev, self.last = state, state


def _expected_winners(log_c, log_z, log_r, count):
  """Top-`count` of every evaluation by one global sort: NaN as -inf, ties to the earlier evaluation."""
  c, z, r = np.concatenate(log_c), np.concatenate(log_z), np.concatenate(log_r)
  order = np.lexsort((np.arange(r.shape[0]), -np.where(np.isnan(r), -np.inf, r)))[:count]
  pad = count - order.shape[0]
  return (np.concatenate([c[order], np.zeros((pad, c.shape[1]))]), np.concatenate([z[order], np.zeros((pad, z.shape[1]), z.dtype)]),
          np.concatenate([r[order], np.full(pad, -np.inf)]))


def run(case: Case, opt=None) -> dict:
  """Drives the oracle and `opt` in lock step; raises AssertionError at the first batch that differs."""
  cfg, sizes, dk = case.cfg, np.asarray(case.sizes, np.int64), len(case.sizes)
  state = {'t': -1 if case.n_prior else 0}
  log_c, log_z, log_r = [], [], []
  planted = {'nan': 0, 'posinf': 0, 'neginf': 0}
  pc, pz = priors(case)

  def score(xc, xz=None):
    t = state['t']
    state['t'] = t + 1
    xc = np.asarray(xc, np.float64).reshape(xc.shape[0], case.width)
    xz = np.zeros((xc.shape[0], 0), np.int32) if xz is None else np.asarray(xz, np.int32)
    r = rewards(case, t, xc, xz)
    if t < 0:
      if opt is not None:
        opt.seed(xc, xz, r)
      return r
    if opt is not None:
      gc, gz = opt.ask()
      np.testing.assert_allclose(gc, xc, rtol=0, atol=1e-12, err_msg=f'{case.name}: continuous batch of step {t}')
      np.testing.assert_array_equal(gz, xz, err_msg=f'{case.name}: categorical batch of step {t}')
      opt.tell(r)
    log_c.append(xc); log_z.append(xz); log_r.append(r)
    planted['nan'] += int(np.sum(np.isnan(r)))
    planted['posinf'] += int(np.sum(np.isposinf(r)))
    planted['neginf'] += int(np.sum(np.isneginf(r)))
    return r

  watch = Watch(case.pool, case.batch, case.steps, cfg)
  common = dict(pool_size=case.pool, batch_size=case.batch, max_evaluations=case.steps * case.batch, count=case.count,
                seed=case.seed, cfg=cfg, on_step=watch)
  if case.q > 1:
    assert dk == 0 and case.norm == 0
    w, wr, _ = eo.run_eagle_optimizer_sets(score, dim=case.dc, n_parallel=case.q, prior_features=pc.reshape(-1, case.dc) if case.n_prior else None,
                                           **common)
    wc, wz = w.reshape(case.count, case.width), np.zeros((case.count, 0), np.int32)
  elif dk or case.norm == 1:
    wc, wz, wr = eo.run_eagle_optimizer_mixed(score, dim=case.dc, sizes=sizes, prior_c=pc if case.n_prior else None,
                                              prior_z=pz if case.n_prior else None, **common)
  else:
    wc, wr, _ = eo.run_eagle_optimizer(score, dim=case.dc, prior_features=pc if case.n_prior else None, **common)
    wz = np.zeros((case.count, 0), np.int32)
  assert state['t'] == case.steps

  # the oracle's incremental top-count merge against one global sort of everything that was evaluated
  ec, ez, er = _expected_winners(log_c, log_z, log_r, case.count)
  np.testing.assert_array_equal(wr, er)
  np.testing.assert_array_equal(wc, ec)
  np.testing.assert_array_equal(wz, ez)
  if opt is not None:
    bc, bz, br = opt.end()
    np.testing.assert_array_equal(br, wr, err_msg=f'{case.name}: winners\' rewards')
    np.testing.assert_array_equal(bz, wz, err_msg=f'{case.name}: winners\' categories')
    np.testing.assert_allclose(bc, wc, rtol=0, atol=1e-12, err_msg=f'{case.name}: winners\' features')

  # ---- coverage: the branch this schedule exists for was reached ----
  last, tied = watch.last, int(np.sum(wr[1:] == wr[:-1]))
  rep = dict(trims=watch.trims, protected=watch.protected, neginf_steps=watch.neginf_steps, tied_pairs=tied, **planted)
  if case.schedule == 'decaying':
    assert watch.trims >= case.pool - int(np.sum(last.rewards == last.best_reward)), rep    # all but the best (and its ties)
    assert watch.protected >= 1 and np.any(last.rewards == last.best_reward), rep       # the best fly survived
    assert max(watch.trim_steps) + case.nb < case.steps and watch.neginf_steps >= case.nb, rep   # every trimmed fly was visited again
  elif case.schedule == 'improving':
    assert watch.trims == 0 and np.all(last.perturbations == cfg.perturbation), rep
  elif case.schedule == 'quantised':
    if case.count >= 16:
      assert tied >= 10, rep
  else:
    assert planted['nan'] >= case.batch + 2 and planted['posinf'] >= 1 and planted['neginf'] >= 1, rep
    # the fly that took BIG in a batch with a NaN holds best_reward: penalised below the bound, never trimmed
    assert watch.trims >= 1 and watch.big_kept and watch.nan_fly_visits >= 1, rep
    if case.steps * case.batch - planted['nan'] >= case.count:
      assert not np.any(np.isnan(wr)), rep
  return rep


def _c(name, schedule, dc, pool, batch, count, steps=None, **kw):
  if steps is None:
    steps = {'decaying': decaying_steps, 'nonfinite': nonfinite_steps}[schedule](pool, batch)
  return Case(name, schedule, dc, pool, batch, steps, count, **kw)


# Shapes at the edges of k_eagle_suggest (one warp per fly, lanes over D and over categories, 8 flies per CTA, the pool's
# forces in shared memory), k_eagle_update (256 threads over B and over B + count) and k_eagle_seed_priors.
CASES = [
    _c('B1', 'decaying', 3, 4, 1, 1),
    _c('B5-P20-count40', 'quantised', 4, 20, 5, 40, steps=30),                       # count > B
    _c('B5-count-above-evaluations', 'quantised', 4, 20, 5, 40, steps=6, n_prior=3),  # the winners end in -inf padding
    _c('nb1', 'decaying', 4, 25, 25, 3),
    _c('nb1-nonfinite', 'nonfinite', 4, 25, 25, 8, n_prior=30),
    _c('B27-D33', 'decaying', 33, 54, 27, 5),                                        # B % 8 != 0, D > 32
    _c('B300-trims', 'decaying', 4, 600, 300, 256),                                  # B and B + count above 256 threads
    _c('B300-ties', 'quantised', 2, 600, 300, 256, steps=8),
    _c('P3000', 'improving', 4, 3000, 25, 3, steps=130, n_prior=3),                   # the shared-memory ceiling of suggest
    _c('D1', 'quantised', 1, 10, 5, 16, steps=24),
    _c('D64-nonfinite', 'nonfinite', 64, 50, 25, 8),
    _c('D64-improving', 'improving', 64, 50, 25, 1, steps=9),
    _c('priors-4P', 'quantised', 3, 50, 25, 16, steps=10, n_prior=200),               # the closest-fly replacement pass
    _c('cat-1-2-33-64', 'decaying', 3, 50, 25, 3, sizes=(1, 2, 33, 64), n_prior=10),
    _c('cat-nonfinite-random', 'nonfinite', 3, 20, 5, 8, sizes=(1, 2, 33, 64), norm=1, n_prior=80),
    _c('cat-only', 'decaying', 0, 25, 25, 3, sizes=(3, 40, 2, 64)),                  # the x30 perturbation factor
    _c('cat-only-ties', 'quantised', 0, 20, 5, 40, steps=20, sizes=(1, 5, 2), n_prior=80),
    _c('random-norm', 'nonfinite', 5, 50, 25, 8, norm=1),
    _c('random-norm-trims', 'decaying', 2, 20, 5, 3, norm=1),
    _c('sets-q3', 'decaying', 4, 25, 25, 3, q=3, n_prior=3),
    _c('sets-q3-D63', 'nonfinite', 21, 20, 5, 8, q=3, n_prior=80),
]
