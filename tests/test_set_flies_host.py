"""Set flies of up to 1024 coordinates (n_parallel = q points of Dc continuous features), without a GPU: the set
optimiser of tests/set_flies_oracle.py in both normalisations, the oracle's perturbations on wide flies, the Python limits of the set optimisers, and
the ptxas report of the suggest kernels."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import eagle_oracle as eo

import set_flies_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'vizier_b200', 'csrc')


def _f(x):
  w = 1.0 + np.arange(x.shape[-1]) % 3
  return -np.sum(w * (x - 0.3) ** 2, axis=-1) / np.sum(w)


@pytest.mark.parametrize('n_prior', [0, 30])
def test_random_set_runner_at_q1_is_the_single_point_runner(n_prior):
  """With q = 1 a set fly is a point: the set runner's RANDOM mode must retrace run_eagle_optimizer_mixed."""
  dim, pool, batch, steps = 5, 50, 25, 12
  cfg = eo.EagleConfig(mutate_normalization_type=1)
  prior = np.random.default_rng(3).uniform(size=(n_prior, dim)) if n_prior else None
  ws, wr = so.run_sets(lambda s: _f(s[:, 0, :]), dim=dim, n_parallel=1, pool_size=pool, batch_size=batch,
                        max_evaluations=steps * batch, count=4, seed=9, cfg=cfg, prior_features=prior)
  mc, _, mr = eo.run_eagle_optimizer_mixed(lambda xc, xz: _f(xc), dim=dim, sizes=(), pool_size=pool, batch_size=batch,
                                           max_evaluations=steps * batch, count=4, seed=9, cfg=cfg, prior_c=prior,
                                           prior_z=np.zeros((n_prior, 0), np.int32) if n_prior else None)
  np.testing.assert_array_equal(wr, mr)
  np.testing.assert_array_equal(ws[:, 0, :], mc)


@pytest.mark.parametrize('dim,q,n_prior', [(3, 4, 0), (20, 4, 40), (64, 16, 0)])
def test_mean_set_runner_is_the_oracle_set_optimiser(dim, q, n_prior):
  pool, batch, steps = 50, 25, 6
  prior = np.random.default_rng(5).uniform(size=(n_prior, dim)) if n_prior else None
  score = lambda s: _f(s.reshape(s.shape[0], -1))
  kw = dict(dim=dim, n_parallel=q, pool_size=pool, batch_size=batch, max_evaluations=steps * batch, count=3, seed=2,
            prior_features=prior)
  ws, wr = so.run_sets(score, **kw)
  es, er, _ = eo.run_eagle_optimizer_sets(score, **kw)
  np.testing.assert_array_equal(wr, er)
  np.testing.assert_array_equal(ws, es)


def test_random_force_scale_is_the_oracle_force_scale():
  rng = np.random.default_rng(8)
  pool, batch = rng.uniform(size=(40, 12)), rng.uniform(size=(5, 12))
  rewards, rb = rng.normal(size=40), rng.normal(size=5)
  rewards[3] = -np.inf
  pu, qu = rng.uniform(size=(5, 40)), rng.uniform(size=(5, 40))
  cfg = eo.EagleConfig(mutate_normalization_type=1)
  np.testing.assert_array_equal(so.random_force_scale(pool, rewards, batch, rb, cfg, pu, qu, 12),
                                eo.force_scale(pool, rewards, batch, rb, cfg, pull_u=pu, push_u=qu))
  assert not np.array_equal(so.random_force_scale(pool, rewards, batch, rb, cfg, pu, qu, 3),
                            eo.force_scale(pool, rewards, batch, rb, cfg, pull_u=pu, push_u=qu))


def test_random_and_mean_set_runners_differ():
  dim, q, pool, batch, steps = 20, 4, 50, 25, 8
  runs = [so.run_sets(lambda s: _f(s.reshape(s.shape[0], -1)), dim=dim, n_parallel=q, pool_size=pool, batch_size=batch,
                      max_evaluations=steps * batch, count=2, seed=4,
                      cfg=eo.EagleConfig(mutate_normalization_type=m))[0] for m in (0, 1)]
  assert not np.allclose(runs[0], runs[1])


@pytest.mark.parametrize('dim,q', [(20, 4), (64, 16), (33, 2)])
def test_wide_set_perturbations_peak_at_pert_per_feature(dim, q):
  """A suggest step without forces (every reward -inf) moves each fly by its perturbation alone: over the q members of
  a feature the largest move is the fly's perturbation, at every width up to 1024."""
  pool, batch = 50, 25
  width = q * dim
  rng = np.random.default_rng(dim + q)
  pert = rng.uniform(0.05, 0.3, size=pool)
  state = eo.EagleState(pool // batch, np.full((pool, width), 0.5), np.full(pool, -np.inf), -np.inf, pert)
  dirs = eo.set_perturbation_directions(11, pool // batch, batch, q, dim)
  x = eo.suggest(state, batch, dirs * 1.0, eo.EagleConfig(), norm_dim=dim)
  moves = np.abs(x - 0.5).reshape(batch, q, dim)
  want = np.broadcast_to(pert[:batch, None], (batch, dim))
  np.testing.assert_allclose(moves.max(axis=1), want, rtol=1e-12)
  assert np.all(moves <= want[:, None, :] * (1 + 1e-12))


class _Reached(AttributeError):
  """Raised by the stand-in model once a set optimiser got past its limits."""


class _NoModel:
  def __getattr__(self, name):
    raise _Reached(name)


def _optimizer(dc, dk=0, random=False):
  from vizier_b200 import optimizers as vb
  factory = vb.random_strategy_factory if random else vb.VectorizedEagleStrategyFactory()
  return vb.VectorizedOptimizer(factory, dc, dk, 25, 500, tuple([3] * dk))


@pytest.mark.parametrize('dc,q', [(64, 16), (20, 4), (50, 3), (1, 16), (33, 2)])
def test_set_optimisers_accept_flies_up_to_1024_coordinates(dc, q):
  from vizier_b200 import gp
  opt = _optimizer(dc)
  with pytest.raises(_Reached):
    opt.optimize_sets(_NoModel(), _NoModel(), gp.UcbPeAcquisition(mode=1), n_parallel=q)
  with pytest.raises(_Reached):
    opt.optimize_qsets(_NoModel(), gp.QAcquisition(1), n_parallel=q)


@pytest.mark.parametrize('dc,q,dk,random', [(64, 17, 0, False), (4, 17, 0, False), (20, 4, 1, False),
                                            (4, 3, 0, True)])
def test_set_pe_rejects_what_it_cannot_run(dc, q, dk, random):
  from vizier_b200 import gp
  with pytest.raises(NotImplementedError):
    _optimizer(dc, dk, random).optimize_sets(_NoModel(), _NoModel(), gp.UcbPeAcquisition(mode=1), n_parallel=q)


@pytest.mark.parametrize('dc,q,dk', [(64, 17, 0), (20, 4, 2)])
def test_eagle_qsets_reject_what_they_cannot_run(dc, q, dk):
  from vizier_b200 import gp
  with pytest.raises(NotImplementedError):
    _optimizer(dc, dk).optimize_qsets(_NoModel(), gp.QAcquisition(1), n_parallel=q)


def test_set_limits_match_the_library():
  from vizier_b200 import optimizers as vb
  text = open(os.path.join(CSRC, 'acq_fn.cuh')).read()
  assert f'kMaxSetPoints = {vb.MAX_SET_POINTS};' in text
  assert f'kMaxFlyDim = {vb.MAX_FLY_DIM};' in text


# ---------------------------------------------------------------------------------------------------------------------
# k_eagle_suggest and k_eagle_suggest_wide: the chunk loop fits its registers
# ---------------------------------------------------------------------------------------------------------------------
def _nvcc():
  for c in (os.environ.get('NVCC'), shutil.which('nvcc'),
            os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc')):
    if c and os.path.isfile(c) and os.access(c, os.X_OK):
      return c
  return None


@pytest.mark.parametrize('name', ['_ZN4vzgp15k_eagle_suggestENS_8EagleDevE', '_ZN4vzgp20k_eagle_suggest_wideENS_8EagleDevE'])
def test_k_eagle_suggest_has_no_spills_and_no_stack_frame(tmp_path, name):
  """k_eagle_suggest_wide walks flies wider than 64 coordinates in chunks; k_eagle_suggest takes the narrower ones."""
  nvcc = _nvcc()
  if nvcc is None:
    pytest.skip('nvcc not found')
  text = open(os.path.join(CSRC, 'Makefile')).read()
  var = {m.group(1): m.group(2).strip() for m in re.finditer(r'^(\w+)\s*:=\s*(.*)$', text, re.M)}
  flags = var['NVFLAGS'].replace('$(ARCH)', var['ARCH']).replace('$(EXTRA)', '').split()
  cmd = [nvcc] + flags + ['-Xptxas', '-v', '-c', os.path.join(CSRC, 'eagle.cu'), '-o', str(tmp_path / 'eagle.o')]
  res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
  assert res.returncode == 0, res.stderr[-4000:]
  m = re.search(rf"Function properties for {name}\s*\n\s*(\d+) bytes stack "
                r"frame, (\d+) bytes spill stores, (\d+) bytes spill loads\s*\n[^\n]*Used (\d+) registers", res.stderr)
  assert m, res.stderr[-4000:]
  stack, stores, loads, regs = (int(g) for g in m.groups())
  print(f'{name}: {regs} registers')
  assert (stack, stores, loads) == (0, 0, 0)
