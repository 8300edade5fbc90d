"""MaxValueEntropySearch without a GPU: the oracle's MES value and slopes against mpmath, its max-value fit, the
reference's acquisitions_test.py:183-234 on the oracle, the designer's construction rules, the ctypes prototypes,
and the ptxas report of the kernels that evaluate MES."""
import ctypes as C
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import mes_oracle as mo
from oracle import eagle_oracle as eo
from oracle import gp_oracle as go

mp = pytest.importorskip('mpmath')
mp.mp.dps = 50

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'vizier_b200', 'csrc')

GAMMAS = np.concatenate([-np.logspace(-3, 3, 120), np.logspace(-3, 3, 120), [0.0, -12.0, -12.000001, -11.999999],
                         -np.arange(37.0, 40.01, 0.5), np.arange(37.0, 40.01, 0.5)])


def _t(g):
  """t(g) = g phi / (2 Phi) - log Phi at 50 digits, with log Phi(g) = log1p(-Phi(-g)) for g > 0."""
  g = mp.mpf(g)
  lp = mp.log(mp.ncdf(g)) if g < 0 else mp.log1p(-mp.ncdf(-g))
  return g * mp.npdf(g) / (2 * mp.exp(lp)) - lp


def _rel(a, b):
  return float(abs(mp.mpf(a) - b) / max(abs(b), mp.mpf('1e-300')))


def test_value_against_mpmath():
  t, _ = mo.terms(GAMMAS)
  worst = max(_rel(a, _t(g)) for g, a in zip(GAMMAS, t))
  assert worst < 1e-13, worst


def test_log_ndtr_is_finite_where_log_normcdf_is_not():
  from scipy.special import ndtr
  z = np.array([-38.5, -40.0, -1e3])
  with np.errstate(divide='ignore'):
    assert np.all(np.isneginf(np.log(ndtr(z))))
  got = mo.log_ndtr(z)
  for a, g in zip(got, z):
    assert _rel(a, mp.log(mp.ncdf(mp.mpf(g)))) < 1e-14


@pytest.mark.parametrize('g', [-1e3, -500.0, -40.0, -13.0, -12.5, -11.5, -5.0, -1.0, -1e-3, 0.0, 0.5, 3.0, 10.0, 30.0])
def test_slope_against_mpmath_and_central_differences(g):
  _, d = mo.terms(np.array([g]))
  want = mp.diff(_t, mp.mpf(g))
  # the direct branch forms 1 + g c from c = g + r with r from erfcx: ~ g^2 ulps of relative error just above -12
  assert _rel(d[0], want) < (5e-12 if -12 <= g < -5 else 1e-13), (g, _rel(d[0], want))
  h = 1e-6 * max(1.0, abs(g))
  tp, _ = mo.terms(np.array([g + h]))
  tm, _ = mo.terms(np.array([g - h]))
  assert abs((tp[0] - tm[0]) / (2 * h) - d[0]) < 1e-6 * max(1.0, abs(d[0]))


def test_mes_slopes_chain_rule():
  rng = np.random.default_rng(0)
  ys = rng.normal(size=7) + 1.0
  mu, sd = rng.normal(size=20), rng.uniform(0.05, 2.0, size=20)
  v, s_mu, s_sd = mo.value_and_slopes(ys, mu, sd)
  h = 1e-6
  np.testing.assert_allclose(s_mu, (mo.value(ys, mu + h, sd) - mo.value(ys, mu - h, sd)) / (2 * h), rtol=1e-6, atol=1e-8)
  np.testing.assert_allclose(s_sd, (mo.value(ys, mu, sd + h) - mo.value(ys, mu, sd - h)) / (2 * h), rtol=1e-6, atol=1e-8)


def test_clamped_variance_limits():
  ys = np.array([1.0, 2.0, 3.0])
  v, s_mu, s_sd = mo.value_and_slopes(ys, np.array([0.5, 1.0, 3.5]), np.zeros(3))
  assert v[0] == 0.0 and v[1] == pytest.approx(math.log(2.0) / 3, rel=1e-15) and v[2] == np.inf
  assert np.all(s_mu == 0) and np.all(s_sd == 0)


def _moments(n, seed, sd_scale=0.1):
  rng = np.random.default_rng(seed)
  return rng.normal(size=n), rng.uniform(0.5, 1.5, size=n) * sd_scale


def test_fit_hits_the_quartiles():
  mu, sd = _moments(30, 1)
  best = float(np.max(mu)) - 0.3
  out = mo.fit(mu, sd, best, 1e-4)
  assert not out['degenerate']
  for q, r in out['r'].items():
    assert abs(math.exp(mo.log_p(r, mu, sd)) - q) < 1e-12
  want = np.fmax(out['a'] - out['b'] * np.log(-np.log(eo.philox_uniform(123, mo.STREAM_MES, 0, 100))), out['floor'])
  np.testing.assert_array_equal(out['samples'], want)
  np.testing.assert_array_equal(mo.fit(mu, sd, best, 1e-4)['samples'], out['samples'])
  assert not np.array_equal(mo.fit(mu, sd, best, 1e-4, seed=124)['samples'], out['samples'])


def test_fit_degenerate_branch_and_floor():
  mu, sd = _moments(10, 2)
  best = float(np.max(mu + 3 * sd))          # P(best) > 0.25
  out = mo.fit(mu, sd, best, 0.01)
  assert out['degenerate']
  np.testing.assert_array_equal(out['samples'], np.full(100, best + 0.5))
  # the floor binds the left tail of the Gumbel draws
  left = float(np.max(mu)) - 1.0
  r50 = mo.fit(mu, sd, left, 1e-12)['r'][0.5]
  out = mo.fit(mu, sd, left, ((r50 - left) / 5.0) ** 2)      # floor at the median
  assert not out['degenerate'] and abs(out['floor'] - r50) < 1e-12
  assert 20 < np.sum(out['samples'] == out['floor']) < 80 and np.min(out['samples']) == out['floor']


def test_fit_step_at_zero_stddev():
  mu = np.array([0.0, 1.0, 2.0])
  sd = np.array([0.0, 0.0, 0.0])
  assert mo.log_p(2.5, mu, sd) == 0.0 and mo.log_p(1.5, mu, sd) == -np.inf
  out = mo.fit(mu, sd, -1.0, 1e-6)
  # P is the step at max(mu) = 2: every quartile converges onto it
  for r in out['r'].values():
    assert abs(r - 2.0) < 1e-12


def test_reference_max_value_entropy_search_on_the_oracle():
  """acquisitions_test.py:183-234: 10 observations, 6 points, 3 dimensions, trust region: shape (6,), all finite."""
  rng = np.random.default_rng(0)
  x = rng.uniform(size=(10, 3))
  y = rng.normal(size=10)
  pred = go.precompute_predictive(go.GPParams(1.0, np.ones(3), 1e-3), x, y)
  ys = mo.fit_predictive(pred, float(np.max(y)))['samples']
  score, aux = mo.score_with_aux(pred, rng.uniform(size=(6, 3)), ys, use_trust_region=True)
  assert score.shape == (6,) and np.all(np.isfinite(score))
  assert set(aux) >= {'raw_acquisition', 'linf_distance', 'radius'}


def _problem(categorical=False):
  from vizier_b200 import vz
  p = vz.ProblemStatement()
  for i in range(3):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  if categorical:
    p.search_space.root.add_categorical_param('c', ['a', 'b'])
  p.metric_information.append(vz.MetricInformation(name='obj', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  return p


def test_designer_construction_rules():
  from vizier_b200 import acquisitions as acq
  from vizier_b200 import optimizers as vb
  from vizier_b200.designers import gp_bandit
  mes = acq.MaxValueEntropySearch.scoring_fn_factory
  with pytest.raises(ValueError, match='Categorical'):
    gp_bandit.VizierGPBandit(_problem(True), scoring_function_factory=mes)
  with pytest.raises(ValueError, match='ensemble'):
    gp_bandit.VizierGPBandit(_problem(), scoring_function_factory=mes, ensemble_size=2)
  with pytest.raises(NotImplementedError):
    gp_bandit.VizierGPBandit(_problem(), scoring_function_factory=mes, scoring_function_is_parallel=True)
  d = gp_bandit.VizierGPBandit(_problem(), scoring_function_factory=mes)
  with pytest.raises(NotImplementedError):
    d.set_priors([])
  gp_bandit.VizierGPBandit(_problem(), scoring_function_factory=mes, acquisition_optimizer_factory=vb.LBFGSBOptimizerFactory())
  gp_bandit.VizierGPBandit(_problem(), scoring_function_factory=mes, linear_coef=0.1)
  data = acq.ModelData(features=None, labels=acq.PaddedArray.as_padded(np.zeros((0, 1))))
  sf = mes(data, None, None, True)
  assert sf.best_label == -np.inf and sf.use_trust_region and sf.num_max_value_samples == 100 and sf.seed == 123


def test_ctypes_prototypes():
  from vizier_b200 import _lib
  assert _lib.ACQ_MES == 4 and _lib.MES_MAX_SAMPLES == 256
  lib = _lib.load()
  assert lib.vzgp_mes_fit.argtypes == [C.c_void_p, C.c_double, C.c_int, C.c_uint64, C.c_void_p]
  assert lib.vzgp_set_mes.argtypes == [C.c_void_p, C.c_void_p, C.c_int]
  header = open(os.path.join(ROOT, 'include', 'vzgp.h')).read()
  assert 'VZGP_ACQ_MES = 4' in header
  assert 'int vzgp_mes_fit(vzgp_handle* h, double best_label, int num_samples, uint64_t seed, double* max_values_out);' in header
  assert 'int vzgp_set_mes(vzgp_handle* h, const double* host_values, int num_samples);' in header


def _nvcc():
  for c in (os.environ.get('NVCC'), shutil.which('nvcc'), os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc')):
    if c and os.path.isfile(c) and os.access(c, os.X_OK):
      return c
  return None


# every kernel that evaluates MES (or, k_mes_fit, log Phi for the fit), by the source file that holds it.
# k_eagle_persistent64 is left out: both of its instances already had a stack frame and spills before MES.
MES_KERNELS = {
    'score.cu': ['k_score_finalize', 'k_small_finalize', 'k_general_finalize', 'k_var_small', 'k_ensemble_combine'],
    'score_i8.cu': ['k_score_i8'],
    'eagle_grid.cu': ['k_eagle_gridILb1'],
    'score_grad.cu': ['k_grad_combine'],
    'mes.cu': ['k_mes_fit'],
}


@pytest.mark.parametrize('src', sorted(MES_KERNELS))
def test_mes_kernels_have_no_stack_frame_or_spills(src, tmp_path):
  nvcc = _nvcc()
  if nvcc is None:
    pytest.skip('nvcc not found')
  text = open(os.path.join(CSRC, 'Makefile')).read()
  var = {m.group(1): m.group(2).strip() for m in re.finditer(r'^(\w+)\s*:=\s*(.*)$', text, re.M)}
  flags = var['NVFLAGS'].replace('$(ARCH)', var['ARCH']).replace('$(EXTRA)', '').split()
  res = subprocess.run([nvcc] + flags + ['-Xptxas', '-v', '-c', os.path.join(CSRC, src), '-o', str(tmp_path / 'o.o')],
                       cwd=CSRC, capture_output=True, text=True)
  assert res.returncode == 0, res.stderr[-4000:]
  found = 0
  for m in re.finditer(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", res.stderr):
    if any(k in m.group(1) for k in MES_KERNELS[src]):
      found += 1
      assert (int(m.group(2)), int(m.group(3)), int(m.group(4))) == (0, 0, 0), m.group(0)
  assert found >= len(MES_KERNELS[src]), res.stderr[-2000:]
