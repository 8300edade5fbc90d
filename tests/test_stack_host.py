"""Transfer-learning stacks of ensemble, linear-kernel and multi-metric levels on the host: the tests-side oracle
(stack_oracle.py) against oracle/gp_oracle.py, the designer's constructor and `set_priors` checks, the level-kind
check of `gp.StackedGP`, and the register budget of the two combine kernels."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import gp_oracle as go
import stack_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'vizier_b200', 'csrc')


def _levels(sizes, d, e, seed, n_metrics=1, same=False, dk=0):
  """Oracle levels fitted on residuals: level l has sizes[l] trials and E members (distinct hyper-parameters unless
  `same`), or one multi-metric member with labels [N, n_metrics]."""
  rng = np.random.default_rng(seed)
  levels = []
  for l, n in enumerate(sizes):
    x = rng.uniform(size=(n, d))
    z = rng.integers(0, 3, size=(n, dk)).astype(np.int32) if dk else None
    y = -np.sum((x - 0.3 - 0.05 * l) ** 2, axis=1) + 0.03 * rng.normal(size=n)
    if n_metrics > 1:
      y = np.stack([y * (1 + 0.5 * m) + 0.1 * m * x[:, 0] for m in range(n_metrics)], axis=1)
    resid = so.residual_labels(levels, x, y, z)
    members = []
    for k in range(e):
      s = 0 if same else k
      lk = np.linspace(0.7, 1.2, dk) if dk else None
      p = go.GPParams(0.8 + 0.3 * l + 0.2 * s, (0.3 + 0.2 * l) * (1 + np.arange(d) / d) * (1 + 0.25 * s),
                      1e-3 * (l + 1) * (1 + s), lk)
      members.append(go.precompute_predictive(p, x, resid, z))
    levels.append(members)
  return rng, levels


@pytest.mark.parametrize('sizes,dk', [((60, 30), 0), ((80, 40, 20), 2)])
def test_single_member_levels_are_predict_stack(sizes, dk):
  rng, levels = _levels(sizes, 3, 1, 1, dk=dk)
  xs = rng.uniform(size=(300, 3))
  zs = rng.integers(0, 3, size=(300, dk)).astype(np.int32) if dk else None
  mean, sd = so.predict(levels, xs, zs)
  want_mean, want_sd = go.predict_stack([lv[0] for lv in levels], xs, zs)
  np.testing.assert_allclose(mean, want_mean, rtol=1e-15, atol=0)
  np.testing.assert_allclose(sd, want_sd, rtol=1e-15, atol=0)
  x, y = levels[-1][0].x, rng.normal(size=sizes[-1])
  np.testing.assert_allclose(so.residual_labels(levels, x, y), go.stack_residual_labels([lv[0] for lv in levels], x, y),
                             rtol=1e-15, atol=0)


def test_one_level_is_the_plain_model():
  rng, levels = _levels((50,), 4, 1, 2)
  xs = rng.uniform(size=(200, 4))
  mean, sd = so.predict(levels, xs)
  want_mean, want_sd = go.predict(levels[0][0], xs)
  np.testing.assert_array_equal(mean, want_mean)
  np.testing.assert_allclose(sd, want_sd, rtol=1e-15, atol=0)
  # and one ensemble level is the two-pass mixture of its members
  rng, levels = _levels((50,), 4, 3, 2)
  mean, sd = so.predict(levels, xs)
  mus, sds = zip(*[go.predict(p, xs) for p in levels[0]])
  np.testing.assert_allclose(mean, np.mean(mus, axis=0), rtol=1e-15)
  np.testing.assert_allclose(sd, np.sqrt(np.mean(np.square(sds), axis=0) + np.var(mus, axis=0)), rtol=1e-13)


def test_identical_members_are_that_member():
  rng, levels = _levels((60, 30, 15), 3, 4, 3, same=True)
  xs = rng.uniform(size=(250, 3))
  mean, sd = so.predict(levels, xs)
  want_mean, want_sd = go.predict_stack([lv[0] for lv in levels], xs)
  np.testing.assert_allclose(mean, want_mean, rtol=1e-13, atol=1e-15)
  np.testing.assert_allclose(sd, want_sd, rtol=1e-13)


def test_each_metric_of_a_multi_metric_stack_is_a_single_metric_stack():
  """Independent multi-task levels share the hyper-parameters and the factor: metric m of the stack is the
  single-metric stack trained on column m (residuals per metric against that metric's stack mean)."""
  rng, multi = _levels((70, 35, 12), 3, 1, 4, n_metrics=3)
  xs = rng.uniform(size=(200, 3))
  mean, sd = so.predict(multi, xs)
  assert mean.shape == (200, 3) and sd.shape == (200,)
  for m in range(3):
    single = []
    for lv in multi:
      p = lv[0]
      resid_m = (p.chol @ (p.chol.T @ p.alpha))[:, m]   # K_y alpha = the level's labels
      single.append([go.precompute_predictive(p.params, p.x, resid_m)])
    mean_m, sd_m = so.predict(single, xs)
    np.testing.assert_allclose(mean[:, m], mean_m, rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(sd, sd_m, rtol=1e-13)


def test_multi_metric_score_is_the_scalarised_ucb_of_the_stack():
  rng, multi = _levels((50, 25), 3, 1, 5, n_metrics=2)
  xs = rng.uniform(size=(150, 3))
  w = np.abs(rng.normal(size=(16, 2)))
  w /= np.linalg.norm(w, axis=1, keepdims=True)
  ref = np.array([-0.8, -1.2])
  best = rng.uniform(0.0, 0.01, size=16)
  got, mean, sd = so.scalarized_score(multi, xs, w, ref, best, 1.8)
  u = np.maximum(mean + 1.8 * sd[:, None] - ref, 0.0)
  want = np.mean(np.maximum(np.min(u[None, :, :] / w[:, None, :], axis=-1) ** 2, best[:, None]), axis=0)
  np.testing.assert_allclose(got, want, rtol=1e-14)


def test_trust_region_is_measured_against_the_top_level():
  rng, levels = _levels((60, 30), 3, 2, 6)
  xs = rng.uniform(size=(400, 3))
  acq, mean, sd, dist = so.score(levels, xs, trust_radius_value=0.2)
  np.testing.assert_array_equal(dist, go.min_linf_distance(xs, levels[-1][0].x, np.ones(3, bool)))
  assert np.all(acq[dist > 0.2] < -1e3) and np.all(acq[dist <= 0.2] == go.ucb(mean, sd)[dist <= 0.2])


def _problem(n_metrics=1):
  from vizier_b200 import vz
  p = vz.ProblemStatement()
  p.search_space.root.add_float_param('x0', -2.0, 2.0)
  p.search_space.root.add_float_param('x1', 0.0, 1.0)
  for k in range(n_metrics):
    p.metric_information.append(vz.MetricInformation(name=f'm{k}', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  return p


def test_constructor_and_set_priors_checks():
  """Every model spec the designer accepts also accepts priors, except parallel scoring functions and the separable
  multi-task types; multi-metric ensembles and multi-metric linear kernels stay refused at construction."""
  from vizier_b200 import acquisitions as acq
  from vizier_b200.designers import gp_bandit
  for kw, n_metrics in (({}, 1), ({'ensemble_size': 3}, 1), ({'linear_coef': 0.4}, 1),
                        ({'ensemble_size': 4, 'linear_coef': 0.4}, 1), ({}, 2), ({}, 3)):
    d = gp_bandit.VizierGPBandit(_problem(n_metrics), **kw)
    d.set_priors([])                        # no prior study: no stack
    assert d._stack is None
  qei = acq.bayesian_scoring_function_factory(lambda data: acq.QEI(acq.get_best_labels(data.labels)))
  d = gp_bandit.VizierGPBandit(_problem(), scoring_function_factory=qei, scoring_function_is_parallel=True)
  with pytest.raises(NotImplementedError, match='parallel'):
    d.set_priors([])
  for t in ('SEPARABLE_NORMAL_TASK_KERNEL_PRIOR', 'SEPARABLE_LKJ_TASK_KERNEL_PRIOR', 'SEPARABLE_DIAG_TASK_KERNEL_PRIOR'):
    d = gp_bandit.VizierGPBandit(_problem(2), multitask_type=t)
    with pytest.raises(NotImplementedError, match='separable'):
      d.set_priors([])
  with pytest.raises(NotImplementedError):
    gp_bandit.VizierGPBandit(_problem(2), ensemble_size=2)
  with pytest.raises(NotImplementedError):
    gp_bandit.VizierGPBandit(_problem(2), linear_coef=0.4)


class _Level:
  """A fitted-level stand-in: the attributes StackedGP.push reads."""

  def __init__(self, n_metrics=1, n=10):
    self.n_metrics, self.dc, self.dk, self.n, self.device = n_metrics, 2, 0, n, None


def test_stack_levels_have_one_kind():
  from vizier_b200 import gp
  s = gp.StackedGP(0)
  s.push(_Level(), 40)
  s.push(_Level(), 10)
  assert (s.ensemble_size, s.n_metrics) == (1, 1)
  assert s.alphas == [0.0, gp.transfer_alpha(10, 40, 4)]
  with pytest.raises(ValueError, match='same kind'):
    s.push(_Level(n_metrics=2), 10)
  m = gp.StackedGP(0)
  m.push(_Level(n_metrics=3), 40)
  assert m.n_metrics == 3
  with pytest.raises(ValueError, match='same kind'):
    m.push(_Level(), 10)


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
  out = tmp_path_factory.mktemp('stack_ptxas')
  cmd = [nvcc] + _makefile_flags() + ['-Xptxas', '-v', '-c', os.path.join(CSRC, src), '-o', str(out / 'k.o')]
  res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
  assert res.returncode == 0, res.stderr[-4000:]
  report = {}
  for m in re.finditer(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", res.stderr):
    report[m.group(1)] = {'stack': int(m.group(2)), 'spill_stores': int(m.group(3)), 'spill_loads': int(m.group(4))}
  return report


@pytest.mark.parametrize('src,kernel', [('score.cu', r'_ZN4vzgp24k_stack_ensemble_combineE'),
                                        ('multi.cu', r'_ZN4vzgp21k_stack_multi_combineE')])
def test_combine_kernels_have_no_spills_and_no_stack_frame(tmp_path_factory, src, kernel):
  report = _ptxas(tmp_path_factory, src)
  names = [n for n in report if re.match(kernel, n)]
  assert len(names) == 1, sorted(report)
  assert report[names[0]] == {'stack': 0, 'spill_stores': 0, 'spill_loads': 0}, report[names[0]]
