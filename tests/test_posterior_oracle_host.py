"""CPU checks of the joint-posterior oracle (posterior_oracle.py) against gp_oracle's marginal and joint forms, and of
VizierGPBandit's per-metric label warping (no GPU)."""
import dataclasses

import numpy as np
import pytest

from oracle import gp_oracle as go
import posterior_oracle as po_


def _case(n, dc, dk, nv, metrics=1, linear=False, seed=0):
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, dc))
  z = rng.integers(0, 3, size=(n, dk)).astype(np.int32) if dk else None
  f = np.sin(3 * x[:, 0]) + np.sum(x, axis=1)
  y = f if metrics == 1 else np.stack([f * (1 + k) + 0.1 * k for k in range(metrics)], 1)
  params = go.GPParams(0.8, 0.3 * (1 + np.arange(dc) / dc), 2e-3, np.linspace(0.6, 1.2, dk) if dk else None,
                       go.LinearParams(0.7, 0.9, 0.2, -0.3) if linear else None)
  pred = go.precompute_predictive(params, x, y, z, row_valid=np.arange(n) < nv)
  xs = np.concatenate([x[:3], rng.uniform(size=(9, dc))])
  xs[5] = xs[4]                                             # training points and a duplicated query
  zs = rng.integers(0, 3, size=(xs.shape[0], dk)).astype(np.int32) if dk else None
  return pred, xs, zs


@pytest.mark.parametrize('n,dc,nv,linear', [(1, 1, 1, False), (20, 3, 20, False), (40, 5, 31, True)])
@pytest.mark.parametrize('add_noise', [True, False])
def test_matches_predictive_covariance_without_categoricals(n, dc, nv, linear, add_noise):
  pred, xs, _ = _case(n, dc, 0, nv, linear=linear)
  mean, cov = po_.joint_posterior(pred, xs, add_noise=add_noise)
  want = go.predictive_covariance(pred, xs)
  if not add_noise:
    want = want - pred.params.observation_noise_variance * np.eye(xs.shape[0])
  np.testing.assert_allclose(cov, want, atol=1e-13, rtol=0)
  mu, sd = go.predict(pred, xs)
  np.testing.assert_allclose(mean, mu, atol=1e-13, rtol=0)
  noise = 0.0 if add_noise else pred.params.observation_noise_variance
  np.testing.assert_allclose(np.diag(cov) + noise, sd ** 2, atol=1e-13, rtol=0)


@pytest.mark.parametrize('dk', [1, 3])
def test_categorical_queries_match_the_marginals(dk):
  pred, xs, zs = _case(30, 2, dk, 27, linear=True)
  mean, cov = po_.joint_posterior(pred, xs, zs)
  mu, sd = go.predict(pred, xs, zs)
  np.testing.assert_allclose(mean, mu, atol=1e-13, rtol=0)
  np.testing.assert_allclose(np.diag(cov), sd ** 2, atol=1e-13, rtol=0)
  # the categorical part matters: without it the covariance of two queries that differ only in z is the diagonal's
  flip = xs[:2].copy(), np.array([[0] * dk, [1] * dk], np.int32)
  _, c2 = po_.joint_posterior(pred, np.stack([flip[0][0], flip[0][0]]), flip[1])
  assert c2[0, 1] < c2[0, 0] - 1e-3
  # and it is symmetric, as the device returns it
  np.testing.assert_array_equal(cov, cov.T)


def test_metric_rows_equal_the_single_metric_posteriors():
  pred, xs, zs = _case(25, 3, 2, 25, metrics=3)
  mean, cov = po_.joint_posterior(pred, xs, zs)
  assert mean.shape == (3, xs.shape[0])
  for m in range(3):
    one = dataclasses.replace(pred, alpha=pred.alpha[:, m])
    mu, c1 = po_.joint_posterior(one, xs, zs)
    np.testing.assert_allclose(mean[m], mu, atol=1e-14, rtol=0)
    np.testing.assert_array_equal(cov, c1)


def test_factor_and_mixture_draws():
  pred, xs, zs = _case(25, 3, 2, 25)
  mean, cov = po_.joint_posterior(pred, xs[:4], zs[:4])
  np.testing.assert_array_equal(po_.factor(cov), np.linalg.cholesky(cov))
  g = np.random.default_rng(3)
  s = po_.mixture_draws([(mean, cov)], g, 7)
  normals = np.random.default_rng(3).standard_normal((7, 4))
  np.testing.assert_allclose(s, mean[None, :] + normals @ np.linalg.cholesky(cov).T, atol=1e-14, rtol=0)
  # two members: normals first, then the member indices
  s2 = po_.mixture_draws([(mean, cov), (mean + 10.0, cov)], np.random.default_rng(3), 7)
  g = np.random.default_rng(3)
  g.standard_normal((7, 4))
  member = g.integers(0, 2, size=7)
  np.testing.assert_allclose(s2 - s, 10.0 * member[:, None] * np.ones((1, 4)), atol=1e-12, rtol=0)


def _two_metric_designer(multitask_type=None):
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit
  p = vz.ProblemStatement()
  p.search_space.root.add_float_param('x0', 0.0, 1.0)
  p.search_space.root.add_float_param('x1', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='big', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  p.metric_information.append(vz.MetricInformation(name='small', goal=vz.ObjectiveMetricGoal.MINIMIZE))
  return gp_bandit.VizierGPBandit(p, rng=2, multitask_type=multitask_type), vz


def _trials(vz, rng, n, start):
  out = []
  for i in range(n):
    t = vz.Trial(parameters={'x0': float(rng.uniform()), 'x1': float(rng.uniform())}, id=start + i)
    t.complete(vz.Measurement({'big': float(rng.normal(1000.0, 50.0)), 'small': float(rng.normal(-3.0, 0.1))}))
    out.append(t)
  return out


@pytest.mark.parametrize('multitask_type', [None, 'SEPARABLE_LKJ_TASK_KERNEL_PRIOR'])
def test_multi_metric_labels_are_warped_one_metric_at_a_time(multitask_type):
  """Every metric's warped labels equal, bit for bit, those of a fresh default warper fitted on that metric alone,
  before and after a second update(); and each metric's warper unwarps back onto its own metric's scale."""
  from vizier_b200 import output_warpers
  d, vz = _two_metric_designer(multitask_type)
  rng = np.random.default_rng(0)
  for start, n in ((1, 12), (100, 7)):
    d.update(vz.CompletedTrials(_trials(vz, rng, n, start)), vz.ActiveTrials())
    _, _, warped = d._trials_to_data(d._trials)
    _, raw = d._converter.to_xy(d._trials)
    assert warped.shape == raw.shape == (len(d._trials), 2)
    for m in range(2):
      want = output_warpers.create_default_warper().warp(raw[:, m:m + 1])[:, 0]
      np.testing.assert_array_equal(warped[:, m], want)
      back = d._output_warpers[m].unwarp(warped[:, m:m + 1])[:, 0]
      np.testing.assert_allclose(back, raw[:, m], rtol=1e-9)
  assert d._output_warpers[0] is d._output_warper and d._output_warpers[1] is not d._output_warper


def test_a_user_warper_is_copied_for_the_other_metrics():
  from vizier_b200 import output_warpers, vz
  from vizier_b200.designers import gp_bandit
  p = vz.ProblemStatement()
  p.search_space.root.add_float_param('x0', 0.0, 1.0)
  for k in range(3):
    p.metric_information.append(vz.MetricInformation(name=f'm{k}', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  w = output_warpers.create_default_warper(half_rank_warp=False)
  d = gp_bandit.VizierGPBandit(p, rng=1, output_warper=w)
  assert d._output_warper is w and len(d._output_warpers) == 3
  assert len({id(x) for x in d._output_warpers}) == 3
  assert all([type(c) for c in x.warpers] == [type(c) for c in w.warpers] for x in d._output_warpers)
