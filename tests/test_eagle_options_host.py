"""The Eagle strategy's UNNORMALIZED force normalisation, its MULTIPLICATIVE perturbation and categorical features of
more than 64 values, on the CPU: tests/eagle_options_oracle.py against hand-worked cases from eagle_strategy.py:847-935
and against oracle/eagle_oracle.py where the two overlap, the Python enums and config checks, and the ptxas report of
the suggest kernels."""
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import eagle_oracle as eo

import eagle_options_oracle as xo
import set_flies_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'vizier_b200', 'csrc')


# ---------------------------------------------------------------------------------------------------------------------
# hand-worked moves: one fly at 0.4 (reward 0) between a better fly at 0.2 (reward 1) and a worse one at 0.6 (reward -1)
# ---------------------------------------------------------------------------------------------------------------------
POOL = np.array([[0.2], [0.6]])
REWARDS = np.array([1.0, -1.0])
BATCH = np.array([[0.4]])
F = math.exp(-0.45 * 0.04 / 1 * 10.0)        # exp(-visibility * d^2 / D * 10), d^2 = 0.04 for both flies


def _scale(norm):
  return xo.force_scale(POOL, REWARDS, BATCH, np.array([0.0]), eo.EagleConfig(mutate_normalization_type=norm))


def test_unnormalized_forces_are_the_raw_pull_and_push():
  np.testing.assert_allclose(_scale(xo.UNNORMALIZED), [[1.5 * F, -0.008 * F]], rtol=1e-15)
  # MEAN divides each side by its number of flies (one here) and scales by normalization_scale = 0.5
  np.testing.assert_allclose(_scale(xo.MEAN), [[0.75 * F, -0.004 * F]], rtol=1e-15)
  moved = xo.move(POOL, BATCH, _scale(xo.UNNORMALIZED), np.zeros((1, 1)), xo.ADDITIVE)
  np.testing.assert_allclose(moved, [[0.4 + 1.5 * F * (0.2 - 0.4) - 0.008 * F * (0.6 - 0.4)]], rtol=1e-15)


@pytest.mark.parametrize('sign', [1.0, -1.0])
def test_multiplicative_perturbation_scales_the_moved_feature(sign):
  s = _scale(xo.MEAN)
  moved = 0.4 + 0.75 * F * (0.2 - 0.4) - 0.004 * F * (0.6 - 0.4)
  p = np.array([[sign * 0.16]])
  np.testing.assert_allclose(xo.move(POOL, BATCH, s, p, xo.ADDITIVE), [[moved + sign * 0.16]], rtol=1e-15)
  np.testing.assert_allclose(xo.move(POOL, BATCH, s, p, xo.MULTIPLICATIVE), [[moved * math.exp(sign * 0.16)]],
                             rtol=1e-15)


def test_unnormalized_logits_take_the_raw_forces():
  """_create_logits_vector (:954-985) with the raw scale: category c sums the forces of the pool flies in c."""
  cfg = eo.EagleConfig(mutate_normalization_type=xo.UNNORMALIZED)
  pool_z, batch_z, sizes = np.array([[2], [0]], np.int32), np.array([[0]], np.int32), [3]
  s = xo.force_scale(POOL, REWARDS, BATCH, np.array([0.0]), cfg, pool_z, batch_z)
  f = math.exp(-0.45 * (0.04 + 1.0) / 2 * 10.0)     # d^2 = 0.04 + one Hamming mismatch, over Dc + Dk = 2 dimensions
  g = math.exp(-0.45 * 0.04 / 2 * 10.0)             # the fly in the batch fly's own category
  np.testing.assert_allclose(s, [[1.5 * f, -0.008 * g]], rtol=1e-15)
  lg = xo.categorical_logits(pool_z, batch_z, s, sizes, cfg)[0, 0]
  ld, ls = math.log(0.02 / 2), math.log(0.98)
  np.testing.assert_allclose(lg, [-0.008 * g + ld - (1.5 * f - 0.008 * g) + ls - ld, ld, 1.5 * f + ld], rtol=1e-14)


# ---------------------------------------------------------------------------------------------------------------------
# overlap with the existing oracle: MEAN / RANDOM with ADDITIVE retrace it
# ---------------------------------------------------------------------------------------------------------------------
def _f(xc, xz):
  out = np.zeros(xc.shape[0])
  if xc.shape[1]:
    out -= np.sum((xc - 0.3) ** 2, axis=1)
  if xz.shape[1]:
    out -= 0.3 * np.mean(xz != 1, axis=1)
  return out


@pytest.mark.parametrize('norm', [xo.MEAN, xo.RANDOM])
@pytest.mark.parametrize('dim,sizes', [(3, ()), (3, (1, 2, 33, 64)), (0, (3, 40))])
def test_mixed_runner_retraces_the_oracle(norm, dim, sizes):
  cfg = eo.EagleConfig(mutate_normalization_type=norm, perturbation_lower_bound=0.05)
  kw = dict(dim=dim, sizes=np.asarray(sizes, np.int64), pool_size=20, batch_size=5, max_evaluations=5 * 30, count=6,
            seed=11, cfg=cfg)
  want = eo.run_eagle_optimizer_mixed(_f, **kw)
  got = xo.run_mixed(_f, **kw)
  for w, g in zip(want, got):
    np.testing.assert_allclose(g, w, rtol=0, atol=1e-14)


@pytest.mark.parametrize('norm', [xo.MEAN, xo.RANDOM])
@pytest.mark.parametrize('q', [1, 3])
def test_set_runner_retraces_the_set_flies_oracle(norm, q):
  cfg = eo.EagleConfig(mutate_normalization_type=norm, perturbation_lower_bound=0.05)
  score = lambda x: _f(x.reshape(x.shape[0], -1), np.zeros((x.shape[0], 0), np.int32))
  kw = dict(dim=4, n_parallel=q, pool_size=20, batch_size=5, max_evaluations=5 * 30, count=3, seed=5, cfg=cfg)
  want = so.run_sets(score, **kw)
  got = xo.run_sets(score, **kw)
  for w, g in zip(want, got):
    np.testing.assert_allclose(g, w, rtol=0, atol=1e-14)


def test_options_change_the_trajectory():
  """Each new option changes the winners of a mixed run and of a set run (so the GPU cases exercise them)."""
  kw = dict(dim=3, sizes=np.asarray((4, 100), np.int64), pool_size=20, batch_size=5, max_evaluations=150, count=4,
            seed=3)
  base = xo.run_mixed(_f, cfg=eo.EagleConfig(), **kw)[0]
  unn = xo.run_mixed(_f, cfg=eo.EagleConfig(mutate_normalization_type=xo.UNNORMALIZED), **kw)[0]
  mul = xo.run_mixed(_f, cfg=eo.EagleConfig(), perturbation_type=xo.MULTIPLICATIVE, **kw)[0]
  assert not np.allclose(base, unn) and not np.allclose(base, mul)


# ---------------------------------------------------------------------------------------------------------------------
# categories past 64
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('big', [65, 257, 1000])
def test_logits_and_uniform_categories_past_64(big):
  rng = np.random.default_rng(big)
  sizes = np.array([1, 5, big])
  pool_z = np.stack([rng.integers(0, s, size=40) for s in sizes], axis=1).astype(np.int32)
  batch_z = pool_z[:6].copy()
  scale = rng.normal(size=(6, 40))
  cfg = eo.EagleConfig()
  want = eo.categorical_logits(pool_z, batch_z, scale, sizes, cfg)
  got = xo.categorical_logits(pool_z, batch_z, scale, sizes, cfg)
  assert got.shape == (6, 3, big)
  fin = np.isfinite(want)
  np.testing.assert_array_equal(np.isfinite(got), fin)
  np.testing.assert_allclose(got[fin], want[fin], rtol=0, atol=1e-13)
  assert np.all(np.isneginf(got[:, 1, 5:])) and np.all(np.isfinite(got[:, 2, :]))

  u = eo.philox_uniform(9, eo.STREAM_INIT_CAT, 0, 3 * 20000).reshape(20000, 3)
  z = eo.uniform_categories(u, sizes)
  assert z.dtype == np.int32 and np.all(z >= 0) and np.all(z < sizes)
  np.testing.assert_array_equal(z[:, 2], np.floor(u[:, 2] * big).astype(np.int32))
  counts = np.bincount(z[:, 2], minlength=big)
  assert counts[0] > 0 and counts[-1] > 0 and np.all(counts > 20000 / big / 4)
  # the boundary draw lands on the last category, not past it
  np.testing.assert_array_equal(eo.uniform_categories(np.array([[1.0 - 2.0 ** -53]]), np.array([big])), [[big - 1]])


# ---------------------------------------------------------------------------------------------------------------------
# Python interface
# ---------------------------------------------------------------------------------------------------------------------
def test_enums_carry_the_reference_values():
  from vizier_b200 import optimizers as vb
  assert {m.name: int(m) for m in vb.MutateNormalizationType} == {'MEAN': 0, 'RANDOM': 1, 'UNNORMALIZED': 2}
  assert {m.name: int(m) for m in vb.ContinuousFeaturePerturbationType} == {'ADDITIVE': 0, 'MULTIPLICATIVE': 1}
  c = vb.EagleStrategyConfig()
  assert c.mutate_normalization_type == vb.MutateNormalizationType.MEAN
  assert c.continuous_feature_perturbation_type == vb.ContinuousFeaturePerturbationType.ADDITIVE
  c = vb.EagleStrategyConfig(mutate_normalization_type=1,
                             continuous_feature_perturbation_type=vb.ContinuousFeaturePerturbationType.MULTIPLICATIVE)
  assert c.mutate_normalization_type == vb.MutateNormalizationType.RANDOM


@pytest.mark.parametrize('field,value', [('mutate_normalization_type', 3), ('mutate_normalization_type', -1),
                                         ('continuous_feature_perturbation_type', 2)])
def test_invalid_option_values_are_rejected(field, value):
  from vizier_b200 import optimizers as vb
  with pytest.raises(ValueError):
    vb.EagleStrategyConfig(**{field: value})


def test_header_documents_the_options():
  text = open(os.path.join(ROOT, 'include', 'vzgp.h')).read()
  assert '"eagle_perturbation"' in text and 'UNNORMALIZED' in text
  assert '(<= 64)' not in text


# ---------------------------------------------------------------------------------------------------------------------
# ptxas: the suggest kernels that take the new paths keep no stack frame and no spills
# ---------------------------------------------------------------------------------------------------------------------
def _nvcc():
  for c in (os.environ.get('NVCC'), shutil.which('nvcc'),
            os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc')):
    if c and os.path.isfile(c) and os.access(c, os.X_OK):
      return c
  return None


_PTXAS = {}


def _ptxas(src, tmp):
  if src not in _PTXAS:
    nvcc = _nvcc()
    if nvcc is None:
      pytest.skip('nvcc not found')
    text = open(os.path.join(CSRC, 'Makefile')).read()
    var = {m.group(1): m.group(2).strip() for m in re.finditer(r'^(\w+)\s*:=\s*(.*)$', text, re.M)}
    flags = var['NVFLAGS'].replace('$(ARCH)', var['ARCH']).replace('$(EXTRA)', '').split()
    cmd = [nvcc] + flags + ['-Xptxas', '-v', '-c', os.path.join(CSRC, src), '-o', str(tmp / (src + '.o'))]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    _PTXAS[src] = res.stderr
  return _PTXAS[src]


@pytest.mark.parametrize('src,name', [
    ('eagle.cu', '_ZN4vzgp15k_eagle_suggestENS_8EagleDevE'),
    ('eagle.cu', '_ZN4vzgp20k_eagle_suggest_wideENS_8EagleDevE'),
    ('eagle_grid.cu', '_ZN4vzgp12k_eagle_gridILb0EEEvNS_8GridArgsE'),
    ('eagle_grid.cu', '_ZN4vzgp12k_eagle_gridILb1EEEvNS_8GridArgsE'),
    ('eagle_grid.cu', '_ZN4vzgp24k_eagle_grid_pe_ensembleENS_11GridEnsArgsE'),
])
def test_suggest_kernels_have_no_spills_and_no_stack_frame(tmp_path, src, name):
  log = _ptxas(src, tmp_path)
  m = re.search(rf"Function properties for {re.escape(name)}\s*\n\s*(\d+) bytes stack "
                r"frame, (\d+) bytes spill stores, (\d+) bytes spill loads\s*\n[^\n]*Used (\d+) registers", log)
  assert m, log[-4000:]
  stack, stores, loads, regs = (int(g) for g in m.groups())
  print(f'{name}: {regs} registers')
  assert (stack, stores, loads) == (0, 0, 0)
