"""CPU tests of models with more than 32 categorical features: the ptxas reports of the wide kernel forms, the
oracle's duplication identity (the reference the GPU tests hold the wide forms to), and the host shapes of a
100-categorical search space."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import gp_oracle as go

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'vizier_b200', 'csrc')


# ---------------------------------------------------------------------------------------------------------------------
# ptxas: the wide forms keep no stack frame and no spills; the narrow forms of the same templates spill nothing
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


def _report(log, kernel, wide):
  m = re.search(rf"Function properties for _ZN4vzgp\d+{kernel}ILb{int(wide)}E\w*\s*\n\s*(\d+) bytes stack "
                r"frame, (\d+) bytes spill stores, (\d+) bytes spill loads\s*\n[^\n]*Used (\d+) registers", log)
  assert m, log[-4000:]
  return tuple(int(g) for g in m.groups())


KERNELS = [('linalg.cu', 'k_kernel_matrix'), ('linalg.cu', 'k_cross_kernel'), ('nll.cu', 'k_nll_grad_tiles'),
           ('nll_small.cu', 'k_nll_grad_small'), ('multi.cu', 'k_mean_multi'), ('eagle.cu', 'k_random_pool_cat')]


@pytest.mark.parametrize('src,kernel', KERNELS)
def test_wide_kernels_have_no_spills_and_no_stack_frame(tmp_path, src, kernel):
  log = _ptxas(src, tmp_path)
  stack, stores, loads, regs = _report(log, kernel, True)
  print(f'{kernel}<true>: {regs} registers')
  assert (stack, stores, loads) == (0, 0, 0)
  # the narrow form: no spills (k_random_pool_cat indexes its by-value size table, a stack frame it always had)
  stack, stores, loads, regs = _report(log, kernel, False)
  print(f'{kernel}<false>: {regs} registers, {stack} bytes stack frame')
  assert (stores, loads) == (0, 0)


# The Eagle kernels read the category counts through cat_size (eagle_dev.cuh), wide or not.  Stack frame and spill bytes
# (stack, stores, loads) of the build before that change: none of them may grow.  k_eagle_persistent64 is capped at 64
# registers and spilled already; k_eagle_update spilled too.
EAGLE_BEFORE = {
    ('eagle.cu', '_ZN4vzgp15k_eagle_suggestENS_8EagleDevE'): (0, 0, 0),
    ('eagle.cu', '_ZN4vzgp20k_eagle_suggest_wideENS_8EagleDevE'): (0, 0, 0),
    ('eagle.cu', '_ZN4vzgp12k_eagle_initENS_8EagleDevE'): (0, 0, 0),
    ('eagle.cu', '_ZN4vzgp14k_eagle_updateENS_8EagleDevE'): (24, 20, 56),
    ('eagle.cu', '_ZN4vzgp19k_eagle_seed_priorsENS_8EagleDevEPKdPKiS2_iPiPd'): (0, 0, 0),
    ('eagle.cu', '_ZN4vzgp20k_eagle_persistent64ILb0EEEvNS_8EagleDevENS_10SmallModelES2_NS_8SmallAcqEimPi'): (120, 172, 1080),
    ('eagle.cu', '_ZN4vzgp20k_eagle_persistent64ILb1EEEvNS_8EagleDevENS_10SmallModelES2_NS_8SmallAcqEimPi'): (144, 200, 1148),
    ('eagle_grid.cu', '_ZN4vzgp12k_eagle_gridILb0EEEvNS_8GridArgsE'): (0, 0, 0),
    ('eagle_grid.cu', '_ZN4vzgp12k_eagle_gridILb1EEEvNS_8GridArgsE'): (0, 0, 0),
    ('eagle_grid.cu', '_ZN4vzgp24k_eagle_grid_pe_ensembleENS_11GridEnsArgsE'): (0, 0, 0),
}


@pytest.mark.parametrize('src,name', sorted(EAGLE_BEFORE), ids=lambda v: v if v.endswith('.cu') else v[7:40])
def test_eagle_kernels_gain_no_spills(tmp_path, src, name):
  log = _ptxas(src, tmp_path)
  m = re.search(rf"Function properties for {re.escape(name)}\s*\n\s*(\d+) bytes stack "
                r"frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
  assert m, log[-4000:]
  got = tuple(int(g) for g in m.groups())
  before = EAGLE_BEFORE[(src, name)]
  print(f'{name}: {got} (before {before})')
  assert all(g <= b for g, b in zip(got, before)), (got, before)


def test_header_documents_the_categorical_limit():
  text = open(os.path.join(ROOT, 'include', 'vzgp.h')).read()
  assert 'Dk <= 1024' in text


# ---------------------------------------------------------------------------------------------------------------------
# the oracle's duplication identity
# ---------------------------------------------------------------------------------------------------------------------
def _dup_case(n, dc, dk, seed):
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, dc))
  z = rng.integers(0, 3, size=(n, dk)).astype(np.int32)
  y = np.sin(3.0 * x.sum(1)) + 0.3 * np.cos(z.sum(1)) + 0.05 * rng.normal(size=n)
  po = go.GPParams(0.8, 0.3 * (1.0 + np.arange(dc) / dc), 2e-3, np.linspace(0.5, 1.5, dk) * dk / 4)
  po2 = go.GPParams(po.signal_variance, po.continuous_length_scale_squared, po.observation_noise_variance,
                    np.repeat(2.0 * po.categorical_length_scale_squared, 2))
  return x, y, z, np.repeat(z, 2, axis=1), po, po2


@pytest.mark.parametrize('n', [20, 90])
def test_oracle_duplication_identity(n):
  x, y, z, z2, po, po2 = _dup_case(n, 3, 32, n)
  np.testing.assert_allclose(go.kernel_matrix(po2, x, z2), go.kernel_matrix(po, x, z), rtol=1e-13, atol=0)
  l1, g1 = go.loss_and_grad(po.to_vector(), x, y, z)
  l2, g2 = go.loss_and_grad(po2.to_vector(), x, y, z2)
  d1, d2 = l1 - go.regularizer(po), l2 - go.regularizer(po2)
  assert abs(d2 - d1) <= 1e-12 * abs(d1)
  dreg = lambda l: 0.02 * np.log(l / 0.5) / l   # noqa: E731
  a = g1[:32] - dreg(po.categorical_length_scale_squared)
  b = (g2[:64] - dreg(po2.categorical_length_scale_squared)).reshape(32, 2)
  np.testing.assert_allclose(4.0 * b[:, 0], a, rtol=1e-11, atol=1e-14)
  np.testing.assert_allclose(4.0 * b[:, 1], a, rtol=1e-11, atol=1e-14)
  np.testing.assert_allclose(g2[64:], g1[32:], rtol=1e-11, atol=1e-14)
  xs = np.random.default_rng(1).uniform(size=(50, 3))
  zs = np.random.default_rng(2).integers(0, 3, size=(50, 32)).astype(np.int32)
  mu1, sd1 = go.predict(go.precompute_predictive(po, x, y, z), xs, zs)
  mu2, sd2 = go.predict(go.precompute_predictive(po2, x, y, z2), xs, np.repeat(zs, 2, axis=1))
  np.testing.assert_allclose(mu2, mu1, rtol=1e-11, atol=1e-13)
  np.testing.assert_allclose(sd2, sd1, rtol=1e-11, atol=1e-13)


# ---------------------------------------------------------------------------------------------------------------------
# host shapes of a 100-categorical space
# ---------------------------------------------------------------------------------------------------------------------
def test_converter_and_bounds_of_a_100_categorical_space():
  from vizier_b200 import converters, gp, vz
  p = vz.ProblemStatement()
  for i in range(3):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  for i in range(100):
    p.search_space.root.add_categorical_param(f'c{i}', [f'v{j}' for j in range(2 + i % 5)])
  p.metric_information.append(vz.MetricInformation(name='m', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  c = converters.TrialToModelInputConverter.from_problem(p)
  assert (c.n_continuous, c.n_categorical) == (3, 100)
  rng = np.random.default_rng(0)
  trials = []
  for t in range(7):
    params = {f'x{i}': float(rng.uniform()) for i in range(3)}
    params.update({f'c{i}': f'v{rng.integers(0, 2 + i % 5)}' for i in range(100)})
    tr = vz.Trial(parameters=params, id=t + 1)
    tr.complete(vz.Measurement({'m': float(t)}))
    trials.append(tr)
  (cont, cat), y = c.to_xy(trials)
  assert cont.shape == (7, 3) and cat.shape == (7, 100) and cat.dtype == np.int32 and y.shape == (7, 1)
  back = c.to_parameters(cont, cat)
  assert [b.as_dict() for b in back] == [pytest.approx(t.parameters.as_dict()) for t in trials]
  lo, hi = gp.param_bounds(3, 100)
  assert lo.shape == hi.shape == (105,)
  theta = 0.5 * (lo + hi)
  hp = gp.GPHyperParams.from_vector(theta, 3, 100)
  assert hp.categorical_length_scale_squared.shape == (100,)
  np.testing.assert_array_equal(hp.to_vector(), theta)
