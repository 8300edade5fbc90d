"""The lock-step harness of tests/eagle_lockstep.py, rehearsed without a GPU.

1. Every case's coverage assertion holds on the oracle's side (it depends on the seed alone), so the GPU run of
   tests/test_gpu_eagle_steps.py exercises the branch each case is named after.
2. The harness accepts a NumPy stand-in built from eagle_oracle.suggest / update and rejects the same stand-in with one
   planted fault: `>=` for `>` in the improvement test, no protection of the best fly, trim draws numbered by the pool
   index instead of the batch slot, winners' ties to the later evaluation, and best_reward that skips a batch holding
   a NaN (the reference's rule, DESIGN.md 6b).
"""
import numpy as np
import pytest

import eagle_lockstep as el
from oracle import eagle_oracle as eo


class NumpyLoop:
  """ask / tell / end over the oracle's strategy steps: continuous flies (q >= 1), MEAN normalisation."""

  def __init__(self, case: el.Case, fault: str = ''):
    assert not case.sizes and case.norm == 0
    self.c, self.cfg, self.fault, self.t = case, case.cfg, fault, 0
    pool = eo.philox_uniform(case.seed, eo.STREAM_INIT_POOL, 0, case.pool * case.width).reshape(case.pool, case.width)
    self.state = eo.init_state(pool, self.cfg)
    self.best = (np.zeros((case.count, case.width)), np.full(case.count, -np.inf),
                 np.full(case.count, np.iinfo(np.int64).max, dtype=np.int64))

  def seed(self, pc, pz, r):
    pool = eo.philox_uniform(self.c.seed, eo.STREAM_INIT_POOL, 0, self.c.pool * self.c.width).reshape(self.c.pool, self.c.width)
    self.state = eo.init_state(pool, self.cfg, pc, r)

  def ask(self):
    c = self.c
    if c.q > 1:
      dirs = eo.set_perturbation_directions(c.seed, self.t, c.batch, c.q, c.dc)
    else:
      dirs = eo.philox_signs(c.seed, self.t, c.batch * c.dc).reshape(c.batch, c.dc)
    self.x = eo.suggest(self.state, c.batch, dirs, self.cfg, norm_dim=c.dc)
    return self.x, np.zeros((c.batch, 0), np.int32)

  def tell(self, r):
    c, st, f = self.c, self.state, self.fault
    start = (st.iterations % c.nb) * c.batch
    if f == 'trim_by_pool_index':
      rnd = eo.philox_uniform(c.seed, eo.STREAM_TRIM, self.t, c.pool * c.width).reshape(c.pool, c.width)[start:start + c.batch]
    else:
      rnd = eo.philox_uniform(c.seed, eo.STREAM_TRIM, self.t, c.batch * c.width).reshape(c.batch, c.width)
    if f in ('improve_on_ties', 'no_protection', 'nan_batch_skipped'):
      self.state = self._faulty_update(r, rnd)
    else:
      self.state = eo.update(st, c.batch, self.x, r, rnd, self.cfg)
    ids = np.arange(c.batch, dtype=np.int64) + self.t * c.batch
    if f == 'ties_to_later':
      ids = -ids
    self.best = eo.update_best(*self.best, self.x, r, ids, c.count)
    self.t += 1

  def _faulty_update(self, r, rnd):
    """eagle_oracle.update with the one line the fault names changed."""
    c, cfg, st, f = self.c, self.cfg, self.state, self.fault
    new_best = max(st.best_reward, float(np.max(r))) if f == 'nan_batch_skipped' else eo.batch_best(st.best_reward, r)
    start = (st.iterations % c.nb) * c.batch
    sl = slice(start, start + c.batch)
    out = st.copy()
    out.iterations, out.best_reward = st.iterations + 1, new_best
    if st.iterations < c.nb:
      out.features[sl], out.rewards[sl] = self.x, r
      return out
    improve = (r >= st.rewards[sl]) if f == 'improve_on_ties' else (r > st.rewards[sl])
    nf = np.where(improve[:, None], self.x, st.features[sl])
    nr = np.where(improve, r, st.rewards[sl])
    npert = np.where(improve, st.perturbations[sl], st.perturbations[sl] * cfg.penalize_factor)
    trim = npert < cfg.perturbation_lower_bound
    if f != 'no_protection':
      trim &= nr != new_best
    out.features[sl] = np.where(trim[:, None], rnd, nf)
    out.perturbations[sl] = np.where(trim, cfg.perturbation, npert)
    out.rewards[sl] = np.where(trim, -np.inf, nr)
    return out

  def end(self):
    return self.best[0], np.zeros((self.c.count, 0), np.int32), self.best[1]


BY_NAME = {c.name: c for c in el.CASES}


@pytest.mark.parametrize('case', el.CASES, ids=lambda c: c.name)
def test_schedule_reaches_its_branch(case):
  rep = el.run(case, None)
  print(case.name, rep)


@pytest.mark.parametrize('case', [c for c in el.CASES if not c.sizes and c.norm == 0 and c.pool <= 600], ids=lambda c: c.name)
def test_harness_accepts_the_oracle_standin(case):
  el.run(case, NumpyLoop(case))


@pytest.mark.parametrize('fault,name', [('improve_on_ties', 'B300-ties'), ('improve_on_ties', 'D1'),
                                        ('no_protection', 'nb1'), ('no_protection', 'B27-D33'),
                                        ('trim_by_pool_index', 'B27-D33'), ('trim_by_pool_index', 'sets-q3-D63'),
                                        ('ties_to_later', 'B5-P20-count40'), ('ties_to_later', 'B300-ties'),
                                        ('nan_batch_skipped', 'nb1-nonfinite'), ('nan_batch_skipped', 'D64-nonfinite')])
def test_harness_catches_a_planted_fault(fault, name):
  with pytest.raises(AssertionError):
    el.run(BY_NAME[name], NumpyLoop(BY_NAME[name], fault))
