"""GP-UCB-PE over uniform ensembles on the host: the tests-side oracle (pe_ensemble_oracle.py) against the single-model
oracle, the two-pass mixture against the one-pass form, the designer's all-members noise rule and constructor checks,
and the register budget of the new kernels."""
import fractions
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import gp_oracle as go
import pe_ensemble_oracle as peo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'vizier_b200', 'csrc')


def _members(n, n_pending, d, e, seed, same=False):
  """E members of A (n trials) and of B (n + n_pending trials, real labels then 0), member e with its own
  hyper-parameters (or all the same)."""
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, d))
  y = np.sin(3 * x[:, 0]) - np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  xb = np.concatenate([x, rng.uniform(size=(n_pending, d))])
  yb = np.concatenate([y, np.zeros(n_pending)])
  params = []
  for k in range(e):
    s = 0 if same else k
    params.append(go.GPParams(1.0 + 0.3 * s, 0.4 * (1 + np.arange(d) / d) * (1 + 0.25 * s), 1e-3 * (1 + s)))
  pa = [go.precompute_predictive(p, x, y) for p in params]
  pb = [go.precompute_predictive(p, xb, yb) for p in params]
  return rng, x, xb, pa, pb


@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('radius', [None, 0.2, 0.7])
def test_single_member_is_the_single_model(mode, radius):
  rng, x, xb, pa, pb = _members(30, 4, 3, 1, 1)
  xs = rng.uniform(size=(200, 3))
  thr = go.ucb_threshold(pa[0], pb[0])
  assert peo.ucb_threshold(pa, pb) == thr
  kw = dict(mode=mode, threshold=thr, trust_radius_value=radius, use_trust_region=radius is not None)
  got, aux = peo.ucb_pe_ensemble_score(pa, pb, xs, **kw)
  want, waux = go.ucb_pe_score(pa[0], pb[0], xs, **kw)
  np.testing.assert_allclose(got, want, rtol=1e-15, atol=0)
  for k in ('mean', 'stddev', 'stddev_from_all'):
    np.testing.assert_allclose(aux[k], waux[k], rtol=1e-15, atol=0)


def test_identical_members_give_the_single_model():
  rng, x, xb, pa, pb = _members(30, 4, 3, 4, 2, same=True)
  xs = rng.uniform(size=(100, 3))
  for mode in (0, 1):
    got, aux = peo.ucb_pe_ensemble_score(pa, pb, xs, mode=mode, threshold=0.1, trust_radius_value=0.3)
    want, waux = go.ucb_pe_score(pa[0], pb[0], xs, mode=mode, threshold=0.1, trust_radius_value=0.3)
    np.testing.assert_allclose(got, want, rtol=1e-14, atol=1e-14)
    np.testing.assert_allclose(aux['stddev_from_all'], waux['stddev_from_all'], rtol=1e-14)


def test_mixture_variance_is_at_least_the_mean_member_variance():
  rng, x, xb, pa, pb = _members(40, 6, 4, 5, 3)
  xs = rng.uniform(size=(300, 4))
  mus, sds = zip(*[go.predict(p, xs) for p in pb])
  _, sd = peo.mixture(np.stack(mus), np.stack(sds))
  mean_var = np.mean(np.stack(sds) ** 2, axis=0)
  assert np.all(sd ** 2 >= mean_var * (1 - 1e-15))
  assert np.any(sd ** 2 > mean_var * 1.01)      # the members' means differ: the spread adds to the variance


def _exact_sd(mus, sds):
  """sqrt of the mixture variance from exact rational arithmetic on the float inputs."""
  out = []
  for j in range(mus.shape[1]):
    m = [fractions.Fraction(float(v)) for v in mus[:, j]]
    s = [fractions.Fraction(float(v)) for v in sds[:, j]]
    e = len(m)
    mean = sum(m) / e
    var = sum(v * v for v in s) / e + sum((v - mean) ** 2 for v in m) / e
    out.append(np.sqrt(float(var)))
  return np.asarray(out)


def test_two_pass_survives_the_cancellation_that_breaks_the_one_pass_form():
  """Model B in high-noise mode: stddev ~1e-5 at the trials while |mean| ~1.  The one-pass form loses about six
  digits of the variance; the two-pass form keeps it."""
  rng = np.random.default_rng(4)
  e, b = 3, 64
  mus = 1.0 + 1e-7 * rng.normal(size=(e, b)) + rng.uniform(-0.5, 0.5, size=(1, b))
  sds = 1e-5 * (1.0 + 0.1 * rng.uniform(size=(e, b)))
  exact = _exact_sd(mus, sds)
  _, two = peo.mixture(mus, sds)
  _, one = peo.one_pass_mixture(mus, sds)
  assert np.max(np.abs(two - exact) / exact) < 1e-13
  assert np.max(np.abs(one - exact) / exact) > 1e-8


class _P:
  def __init__(self, sf2, sn2):
    self.signal_variance, self.observation_noise_variance = sf2, sn2


def test_noise_rule_needs_every_member():
  low, high = _P(0.1, 1.0), _P(1.0, 0.01)          # snr 0.1 and 100 against the threshold 0.7
  assert peo.noise_is_high([low, low, low], 0.7)
  assert not peo.noise_is_high([low, high], 0.7)   # member 0 alone would say high
  assert not peo.noise_is_high([high, low], 0.7)   # any member would say high
  from vizier_b200 import gp
  from vizier_b200.designers import gp_ucb_pe as ucbpe
  d = ucbpe.VizierGPUCBPEBandit(_problem(1), ensemble_size=3, rng=1)
  mk = lambda p: gp.GPHyperParams(p.signal_variance, np.ones(2), p.observation_noise_variance)   # noqa: E731
  for members in ([low, low, low], [low, high, low], [high, low, low], [low, low, high]):
    assert d._noise_is_high([mk(p) for p in members]) == peo.noise_is_high(members, 0.7)
  assert d._noise_is_high(mk(low)) and not d._noise_is_high(mk(high))


def _problem(n_metrics):
  from vizier_b200 import vz
  p = vz.ProblemStatement()
  p.search_space.root.add_float_param('x0', -2.0, 2.0)
  p.search_space.root.add_float_param('x1', 0.0, 1.0)
  for k in range(n_metrics):
    p.metric_information.append(vz.MetricInformation(name=f'm{k}', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  return p


def test_constructor_checks():
  from vizier_b200.designers import gp_ucb_pe as ucbpe
  for e in (1, 2, 3, 5):
    ucbpe.VizierGPUCBPEBandit(_problem(1), ensemble_size=e)                   # 1 fixed + 4 random initialisations
  ucbpe.VizierGPUCBPEBandit(_problem(1), ensemble_size=3, mixes_linear_kernel=True)
  ucbpe.VizierGPUCBPEBandit(_problem(1), ensemble_size=3,
                            config=ucbpe.UCBPEConfig(optimize_set_acquisition_for_exploration=True))
  with pytest.raises(ValueError):
    ucbpe.VizierGPUCBPEBandit(_problem(1), ensemble_size=6)
  with pytest.raises(ValueError):
    ucbpe.VizierGPUCBPEBandit(_problem(1), ensemble_size=3, ard_random_restarts=1)
  with pytest.raises(ValueError):
    ucbpe.VizierGPUCBPEBandit(_problem(1), ensemble_size=-1)
  with pytest.raises(NotImplementedError):
    ucbpe.VizierGPUCBPEBandit(_problem(2), ensemble_size=2)


def _nvcc():
  for c in (os.environ.get('NVCC'), shutil.which('nvcc'),
            os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc')):
    if c and os.path.isfile(c) and os.access(c, os.X_OK):
      return c
  return None


def _makefile_flags():
  text = open(os.path.join(CSRC, 'Makefile')).read()
  var = {m.group(1): m.group(2).strip() for m in re.finditer(r'^(\w+)\s*:=\s*(.*)$', text, re.M)}
  flags = var['NVFLAGS'].replace('$(ARCH)', var['ARCH']).replace('$(EXTRA)', '')
  assert '$(' not in flags, flags
  return flags.split()


def _ptxas(tmp_path_factory, src):
  nvcc = _nvcc()
  if nvcc is None:
    pytest.skip('nvcc not found')
  out = tmp_path_factory.mktemp('pe_ens_ptxas')
  cmd = [nvcc] + _makefile_flags() + ['-Xptxas', '-v', '-c', os.path.join(CSRC, src), '-o', str(out / 'k.o')]
  res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
  assert res.returncode == 0, res.stderr[-4000:]
  report = {}
  for m in re.finditer(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", res.stderr):
    report[m.group(1)] = {'stack': int(m.group(2)), 'spill_stores': int(m.group(3)), 'spill_loads': int(m.group(4))}
  return report


def test_combine_kernel_has_no_spills_and_no_stack_frame(tmp_path_factory):
  report = _ptxas(tmp_path_factory, 'score.cu')
  names = [n for n in report if re.match(r'_ZN4vzgp21k_pe_ensemble_combineE', n)]
  assert len(names) == 1, sorted(report)
  assert report[names[0]] == {'stack': 0, 'spill_stores': 0, 'spill_loads': 0}, report[names[0]]

