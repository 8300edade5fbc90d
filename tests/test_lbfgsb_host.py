"""The L-BFGS-B acquisition optimiser without a GPU: the oracle's analytic gradient against finite differences and the
complex step, the reference's lbfgsb_optimizer_test.py through `LBFGSBOptimizer.optimize_host`, the lock-step driver
against SciPy run one restart at a time, the constructor and call checks, and the ptxas report of score_grad.cu."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import scipy.optimize as sopt

from oracle import gp_oracle as go
import lbfgsb_oracle as lo
from vizier_b200 import ard, vz
from vizier_b200 import optimizers as vb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'vizier_b200', 'csrc')


def _members(rng, n, dc, E, linear):
  x, y, _ = lo.make_model(rng, n, dc, linear=linear)
  return x, [lo.predictive(x, y, lo.make_model(rng, 1, dc, linear=linear, seed_params=e)[2]) for e in range(E)]


def _acq(name, best, tr_radius=None):
  from vizier_b200 import gp
  spec = lo.acquisitions(best)[name]
  if tr_radius is None:
    return gp.Acquisition(1.8, False, 1.0, acq_fn=spec)
  return gp.Acquisition(1.8, True, tr_radius, acq_fn=spec)


@pytest.mark.parametrize('linear', [False, True])
@pytest.mark.parametrize('E', [1, 2, 3])
@pytest.mark.parametrize('name', ['ucb', 'lcb', 'ei', 'pi', 'atr_ucb_pi', 'atr_ucb_lcb'])
def test_oracle_gradient_is_the_derivative_of_the_value(name, E, linear):
  """Central differences (h = 1e-6, relative 1e-6 of the gradient's max-norm) and the complex step (relative 1e-12)."""
  rng = np.random.default_rng(E * 10 + linear)
  x, preds = _members(rng, 12, 3, E, linear)
  xs = rng.uniform(0.05, 0.95, size=(6, 3))
  acq = _acq(name, best=0.3)
  got = lo.score_and_grad(preds, xs, acq)
  f = lo.value_fn(preds, acq)
  np.testing.assert_allclose(np.real(f(xs.astype(complex))), got['score'], rtol=1e-12, atol=1e-12)
  h = 1e-6
  fd = np.stack([(lo.score_and_grad(preds, xs + h * np.eye(3)[d], acq)['score']
                  - lo.score_and_grad(preds, xs - h * np.eye(3)[d], acq)['score']) / (2 * h) for d in range(3)], axis=1)
  scale = np.max(np.abs(got['grad']))      # relative to the gradient's max-norm over the points
  assert np.all(np.abs(fd - got['grad']) <= 1e-6 * scale + 1e-9), (fd, got['grad'])
  cs = np.stack([np.imag(f(xs + 1e-30j * np.eye(3)[d])) / 1e-30 for d in range(3)], axis=1)
  assert np.all(np.abs(cs - got['grad']) <= 1e-12 * scale), (cs, got['grad'])


@pytest.mark.parametrize('linear', [False, True])
def test_oracle_value_is_gp_oracle_predict(linear):
  rng = np.random.default_rng(5)
  x, preds = _members(rng, 15, 4, 3, linear)
  xs = rng.uniform(size=(9, 4))
  got = lo.score_and_grad(preds[:1], xs, _acq('ucb', 0.0))
  mu, sd = go.predict(preds[0], xs)
  np.testing.assert_allclose(got['mean'], mu, rtol=1e-12, atol=1e-12)
  np.testing.assert_allclose(got['stddev'], sd, rtol=1e-12, atol=1e-12)
  mean, sd = go.predict_ensemble(preds, xs)
  got = lo.score_and_grad(preds, xs, _acq('ucb', 0.0))
  np.testing.assert_allclose(got['mean'], mean, rtol=1e-12, atol=1e-12)
  np.testing.assert_allclose(got['stddev'], sd, rtol=1e-9)


@pytest.mark.parametrize('E', [1, 2])
def test_oracle_gradient_outside_the_trust_region(E):
  """Outside the region the score is -1e4 - dist; its gradient, -d dist / dx, against central differences."""
  rng = np.random.default_rng(7 + E)
  x, preds = _members(rng, 6, 3, E, False)
  xs = rng.uniform(size=(40, 3))
  acq = _acq('ucb', 0.0, tr_radius=0.25)
  got = lo.score_and_grad(preds, xs, acq)
  dist = go.min_linf_distance(xs, x, np.ones(3, bool))
  np.testing.assert_array_equal(got['linf_distance'], dist)
  outside = dist > 0.25
  assert outside.any() and (~outside).any()
  np.testing.assert_array_equal(got['score'][outside], -1e4 - dist[outside])
  h = 1e-5
  fd = np.stack([(lo.score_and_grad(preds, xs + h * np.eye(3)[d], acq)['score']
                  - lo.score_and_grad(preds, xs - h * np.eye(3)[d], acq)['score']) / (2 * h) for d in range(3)], axis=1)
  np.testing.assert_allclose(fd[outside], got['grad'][outside], atol=1e-6)
  assert np.all(np.sum(np.abs(got['grad'][outside]), axis=1) == 1.0)


def _converter(bounds):
  from vizier_b200 import converters
  p = vz.ProblemStatement()
  for i, (lo_, hi) in enumerate(bounds):
    p.search_space.root.add_float_param(f'f{i + 1}', lo_, hi)
  p.metric_information.append(vz.MetricInformation(name='acquisition', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  return converters.TrialToModelInputConverter.from_problem(p)


def _sum(points):
  return np.sum(points, axis=-1), np.ones_like(points)


def test_optimize_candidates_len():
  """lbfgsb_optimizer_test.py::test_optimize_candidates_len."""
  opt = vb.LBFGSBOptimizerFactory(random_restarts=10, maxiter=20)(_converter([(0, 10)] * 3))
  assert len(opt.optimize_host(_sum).rewards) == 1


def test_singleton_constraints_are_respected():
  """lbfgsb_optimizer_test.py::test_singleton_constraints_are_respected: the fixed parameter stays at 0.5 and the
  reward is the score of the returned candidate, re-read from its parameters."""
  conv = _converter([(0, 10), (0, 10), (5, 5)])
  opt = vb.LBFGSBOptimizerFactory(random_restarts=10, maxiter=20)(conv)
  assert opt.bounds == ((0.0, 1.0), (0.0, 1.0), (0.5, 0.5))
  res = opt.optimize_host(_sum)
  params = conv.to_parameters(res.features)
  feats, _ = conv.to_features([vz.Trial(parameters=p) for p in params])
  np.testing.assert_allclose(_sum(feats)[0], res.rewards)
  assert params[0]['f3'].value == 5.0


def _quadratic(points):
  return -np.sum(np.square(points - 0.52), axis=(-1, -2) if points.ndim == 3 else -1), -2.0 * (points - 0.52)


def test_best_candidates_count_is_1():
  """lbfgsb_optimizer_test.py::test_best_candidates_count_is_1."""
  conv = _converter([(0, 1), (0, 1)])
  res = vb.LBFGSBOptimizerFactory(random_restarts=10, maxiter=20)(conv).optimize_host(_quadratic)
  p = conv.to_parameters(res.features)[0]
  assert abs(p['f1'].value - 0.52) <= 1e-6 and abs(p['f2'].value - 0.52) <= 1e-6
  assert abs(res.rewards[0]) <= 1e-6


def test_batch_candidates():
  """lbfgsb_optimizer_test.py::test_batch_candidates: one set of n_parallel = 3 points."""
  conv = _converter([(0, 1)] * 3)
  res = vb.LBFGSBOptimizerFactory(random_restarts=10, maxiter=20)(conv).optimize_host(_quadratic, count=1, n_parallel=3)
  params = conv.to_parameters(res.features)
  assert len(params) == 3
  for p in params:
    assert abs(p['f1'].value - 0.52) <= 1e-6 and abs(p['f2'].value - 0.52) <= 1e-6
  assert np.all(np.abs(res.rewards) <= 1e-6)


def test_lockstep_restarts_take_scipy_minimize_iterates():
  """Each restart of the optimiser's lock-step run evaluates exactly the points `scipy.optimize.minimize` evaluates
  when that restart runs alone, and ends at the same point and value."""
  if ard._setulb is None:
    pytest.skip('scipy.optimize._lbfgsb not importable')
  rng = np.random.default_rng(11)
  c = rng.uniform(size=4)

  def f(x):
    return float(np.sum((x - c) ** 2 * (1 + x)) + np.sin(3 * x).sum()), 2 * (x - c) * (1 + x) + (x - c) ** 2 + 3 * np.cos(3 * x)

  bounds = [(0.0, 1.0)] * 4
  inits = rng.uniform(-0.2, 1.2, size=(6, 4))
  seen = {i: [] for i in range(6)}

  def batch(idx, pts):
    out = [f(p) for p in pts]
    for i, p in zip(idx, pts):
      seen[i].append(np.array(p))
    return [o[0] for o in out], [o[1] for o in out]

  results = ard._lockstep(batch, inits, bounds, stop_nonfinite=True, maxiter=30, gtol=1e-8, maxls=20)
  for i, x0 in enumerate(inits):
    alone = []

    def g(x):
      alone.append(np.array(x))
      return f(x)
    want = sopt.minimize(g, np.clip(x0, 0, 1), jac=True, method='L-BFGS-B', bounds=bounds,
                         options={'maxiter': 30, 'gtol': 1e-8, 'maxls': 20})
    np.testing.assert_array_equal(np.stack(seen[i]), np.stack(alone))
    np.testing.assert_array_equal(results[i][0], want.x)
    assert results[i][1] == want.fun


def test_non_finite_restart_stops_and_keeps_its_value():
  """A restart whose value or gradient is not finite stops there; the others continue; nothing raises or hangs."""
  opt = vb.LBFGSBOptimizer(((0.0, 1.0), (0.0, 1.0)), random_restarts=8, maxiter=50)

  def fn(points):
    v, g = _quadratic(points)
    bad = points[:, 0] > 0.6
    return np.where(bad, np.nan, v), np.where(bad[:, None], np.nan, g)

  res = opt.optimize_host(fn, count=8)
  assert np.isnan(res.rewards).any() and np.isfinite(res.rewards[0])
  np.testing.assert_allclose(res.features[0], 0.52, atol=1e-6)
  res = opt.optimize_host(lambda p: (np.full(len(p), np.nan), np.full(p.shape, np.nan)))
  assert np.isnan(res.rewards).all()


def test_constructor_and_call_checks():
  from vizier_b200 import acquisitions as acq_lib
  from vizier_b200.designers import gp_bandit, gp_ucb_pe
  p = vz.ProblemStatement()
  p.search_space.root.add_float_param('x', 0.0, 1.0)
  p.search_space.root.add_categorical_param('c', ['a', 'b'])
  p.metric_information.append(vz.MetricInformation(name='m', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  from vizier_b200 import converters
  with pytest.raises(ValueError, match='categorical'):
    vb.LBFGSBOptimizerFactory()(converters.TrialToModelInputConverter.from_problem(p))
  with pytest.raises(ValueError, match='categorical'):
    gp_bandit.VizierGPBandit(p, acquisition_optimizer_factory=vb.LBFGSBOptimizerFactory())
  opt = vb.LBFGSBOptimizerFactory(random_restarts=4)(_converter([(0, 1)]))
  with pytest.raises(ValueError, match='n_parallel'):
    opt.optimize_host(_quadratic, count=2, n_parallel=3)
  with pytest.raises(ValueError, match='random_restarts'):
    opt.optimize_host(_quadratic, count=5)
  saved = ard._setulb
  ard._setulb = None          # a SciPy without the reverse-communication routine
  try:
    with pytest.raises(NotImplementedError, match='setulb'):
      opt.optimize_host(_quadratic)
  finally:
    ard._setulb = saved

  def problem(n_metrics):
    q = vz.ProblemStatement()
    q.search_space.root.add_float_param('x', 0.0, 1.0)
    for i in range(n_metrics):
      q.metric_information.append(vz.MetricInformation(name=f'm{i}', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
    return q

  f = vb.LBFGSBOptimizerFactory()
  with pytest.raises(NotImplementedError, match='multi-metric'):
    gp_bandit.VizierGPBandit(problem(2), acquisition_optimizer_factory=f)
  with pytest.raises(NotImplementedError, match='parallel'):
    gp_bandit.VizierGPBandit(problem(1), acquisition_optimizer_factory=f, scoring_function_is_parallel=True,
                             scoring_function_factory=acq_lib.bayesian_scoring_function_factory(lambda d: acq_lib.QEI()))
  d = gp_bandit.VizierGPBandit(problem(1), acquisition_optimizer_factory=f)
  with pytest.raises(NotImplementedError, match='priors'):
    d.set_priors([])
  with pytest.raises(NotImplementedError, match='GP-UCB-PE'):
    gp_ucb_pe.VizierGPUCBPEBandit(problem(1), acquisition_optimizer_factory=f)


def _nvcc():
  for c in (os.environ.get('NVCC'), shutil.which('nvcc'),
            os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc')):
    if c and os.path.isfile(c) and os.access(c, os.X_OK):
      return c
  return None


def test_score_grad_kernels_have_no_spills_and_no_stack_frame(tmp_path):
  nvcc = _nvcc()
  if nvcc is None:
    pytest.skip('nvcc not found')
  text = open(os.path.join(CSRC, 'Makefile')).read()
  var = {m.group(1): m.group(2).strip() for m in re.finditer(r'^(\w+)\s*:=\s*(.*)$', text, re.M)}
  assert 'score_grad.cu' in var['SRCS'].split()
  flags = var['NVFLAGS'].replace('$(ARCH)', var['ARCH']).replace('$(EXTRA)', '').split()
  res = subprocess.run([nvcc] + flags + ['-Xptxas', '-v', '-c', os.path.join(CSRC, 'score_grad.cu'), '-o',
                        str(tmp_path / 'k.o')], cwd=CSRC, capture_output=True, text=True)
  assert res.returncode == 0, res.stderr[-4000:]
  report = {m.group(1): tuple(int(m.group(i)) for i in (2, 3, 4)) for m in re.finditer(
      r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
      res.stderr)}
  for k in ('k_grad_solve', 'k_grad_rows', 'k_grad_combine'):
    names = [n for n in report if k in n]
    assert len(names) == 1, sorted(report)
    assert report[names[0]] == (0, 0, 0), (k, report[names[0]])
