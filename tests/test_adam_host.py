"""OptaxTrain (Adam ARD) on the host: SoftClip, the Adam steps, the epoch loop and its ranking, construction errors.
No GPU: the loss callables here are NumPy functions."""
import math

import numpy as np
import pytest

import adam_oracle as ao
from vizier_b200 import ard
from vizier_b200 import gp


def _bounds(dc=2, dk=1):
  return gp.param_bounds(dc, dk)


def test_soft_clip_round_trip_range_and_monotonicity():
  lo, hi = _bounds()
  rng = np.random.default_rng(0)
  th = ard.log_uniform_init(rng, 2, 1, 200)
  u = ard.soft_clip_inverse(th, lo, hi)
  back, _ = ard.soft_clip(u, lo, hi)
  np.testing.assert_allclose(back, th, rtol=1e-9, atol=1e-15)
  np.testing.assert_allclose(ao.soft_clip_inverse(th, lo, hi), u, rtol=1e-12, atol=1e-12)
  grid = np.linspace(-5.0, 150.0, 20001)
  for p in range(lo.shape[0]):
    y, d = ard.soft_clip(grid, lo[p], hi[p])
    slack = 4 * np.spacing(hi[p])      # hi - (hi - lo) rounds at the scale of hi
    assert np.all(y >= lo[p] - slack) and np.all(y <= hi[p])
    assert np.all(np.diff(y) >= 0.0)
    assert np.all(d >= 0.0) and np.all(d <= 1.0)
    np.testing.assert_allclose(y, ao.soft_clip(grid, lo[p], hi[p]), rtol=1e-13, atol=slack)


def test_soft_clip_derivative_matches_finite_differences():
  lo, hi = _bounds()
  for p in range(lo.shape[0]):
    u = lo[p] + np.array([-0.03, -0.005, 0.0, 0.004, 0.02, 0.5 * (hi[p] - lo[p]), hi[p] - lo[p] - 0.01])
    h = 1e-6
    fd = (ard.soft_clip(u + h, lo[p], hi[p])[0] - ard.soft_clip(u - h, lo[p], hi[p])[0]) / (2 * h)
    _, d = ard.soft_clip(u, lo[p], hi[p])
    np.testing.assert_allclose(d, fd, rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(d, ao.soft_clip_grad(u, lo[p], hi[p]), rtol=1e-12, atol=1e-300)


def test_unbounded_parameters_use_the_identity():
  lo, hi = gp.param_bounds(2, 0, linear=True)
  assert np.isinf(lo).sum() == 2
  u = np.linspace(-3.0, 3.0, lo.shape[0])
  th, d = ard.soft_clip(u, lo, hi)
  free = ~np.isfinite(lo)
  np.testing.assert_array_equal(th[free], u[free])
  np.testing.assert_array_equal(d[free], 1.0)
  np.testing.assert_array_equal(ard.soft_clip_inverse(th, lo, hi)[free], u[free])


def test_points_on_a_bound_map_to_finite_coordinates():
  lo, hi = _bounds()
  for th in (lo, hi, lo - 1.0, hi + 1.0):
    u = ard.soft_clip_inverse(th, lo, hi)
    assert np.all(np.isfinite(u))


def test_first_adam_steps_by_hand():
  """Two parameters, loss = sum (theta - c)^2 in the unconstrained identity form: the first two updates."""
  lo = np.array([-np.inf, -np.inf])
  hi = np.array([np.inf, np.inf])
  c = np.array([1.0, -2.0])
  opt = ard.adam(0.1, b1=0.9, b2=0.99, eps=1e-8)
  th0 = np.array([[0.0, 0.0]])

  def f(idx, ths):
    return [float(np.sum((t - c) ** 2)) for t in ths], [2.0 * (t - c) for t in ths]

  th, final, trace = ard.adam_host_epochs(opt, 2, th0, lo, hi, f)
  g1 = 2.0 * (th0[0] - c)
  mu, nu = 0.1 * g1, 0.01 * g1 * g1
  u1 = th0[0] - 0.1 * (mu / 0.1) / (np.sqrt(nu / 0.01) + 1e-8)   # first step: -lr sign(g)
  np.testing.assert_allclose(u1, [0.1, -0.1], rtol=1e-7)
  g2 = 2.0 * (u1 - c)
  mu = 0.9 * mu + 0.1 * g2
  nu = 0.99 * nu + 0.01 * g2 * g2
  u2 = u1 - 0.1 * (mu / (1 - 0.9 ** 2)) / (np.sqrt(nu / (1 - 0.99 ** 2)) + 1e-8)
  np.testing.assert_allclose(th[0], u2, rtol=1e-14)
  np.testing.assert_allclose(trace[:, 0], [np.sum((th0[0] - c) ** 2), np.sum((u1 - c) ** 2)], rtol=1e-14)
  assert final[0] == trace[-1, 0]


def _quadratic_problem():
  lo, hi = gp.param_bounds(2, 0)
  centre = np.array([0.7, 3.0, 0.01, 1.5])

  def loss_and_grad(theta):
    d = np.log(theta) - np.log(centre)
    return float(np.sum(d * d)), 2.0 * d / theta

  return lo, hi, loss_and_grad


def test_loop_on_a_quadratic_matches_the_oracle_and_ranks_pre_update_losses():
  lo, hi, fn = _quadratic_problem()
  rng = np.random.default_rng(3)
  th0 = ard.log_uniform_init(rng, 2, 0, 5)
  opt = ard.OptaxTrain(ard.adam(0.05), epochs=40)
  best, final = opt(th0, fn, list(zip(lo, hi)), best_n=3)
  want_th, want_final, want_trace = ao.adam_train(th0, lo, hi, fn, learning_rate=0.05, epochs=40)
  m = opt.last_metrics
  assert m['route'] == 'host' and m['loss'].shape == (40, 5)
  np.testing.assert_allclose(m['loss'], want_trace, rtol=1e-9)
  np.testing.assert_allclose(final, want_final, rtol=1e-9)
  # final losses are those of the last evaluation, i.e. before the last update
  np.testing.assert_array_equal(final, m['loss'][-1])
  order = ao.best_n(want_final, 3)
  for k, i in enumerate(order):
    np.testing.assert_allclose(best[k], want_th[i], rtol=1e-9)
    # the returned parameters are those after the last update: their loss differs from the ranking loss
    assert fn(best[k])[0] != final[i]
  assert np.all(want_trace[-1] < want_trace[0])


def test_nan_restarts_stop_and_sort_last_and_ties_keep_their_order():
  lo, hi, fn = _quadratic_problem()
  th0 = np.tile(ard.log_uniform_init(np.random.default_rng(4), 2, 0, 1), (4, 1))
  calls = {'n': 0}

  def batch(idx, ths):
    calls['n'] += 1
    out_l, out_g = [], []
    for i, t in zip(idx, ths):
      l, g = fn(t)
      if i == 0 and calls['n'] >= 3:     # restart 0 fails at its third evaluation
        l = math.nan
      if i == 2:                         # restart 2 hits the loss callables' non-finite sentinel at once
        l, g = 1e300, np.zeros_like(t)
      out_l.append(l)
      out_g.append(g)
    return out_l, out_g

  batch.n_restarts = 4
  opt = ard.OptaxTrain(ard.adam(0.02), epochs=6)
  best, final = opt(th0, batch, list(zip(lo, hi)), best_n=4)
  trace = opt.last_metrics['loss']
  assert np.all(np.isnan(trace[2:, 0])) and np.all(np.isfinite(trace[:2, 0]))
  assert np.all(np.isnan(trace[:, 2]))
  assert np.isnan(final[0]) and np.isnan(final[2])
  # restarts 1 and 3 are identical: a stable sort keeps 1 first; the NaN restarts come last in index order
  assert final[1] == final[3]
  np.testing.assert_array_equal(best[0], best[1])
  th_stop = ard.soft_clip(ard.soft_clip_inverse(th0[2], lo, hi), lo, hi)[0]
  np.testing.assert_array_equal(best[3], th_stop)        # restart 2 kept the parameters of its failed evaluation
  assert [int(i) for i in np.argsort(final, kind='stable')] == [1, 3, 0, 2]


def test_restarts_split_between_handles_give_the_single_handle_results():
  """Host-stepped epochs over three equivalent loss callables (one per handle) evaluate the restarts concurrently and
  return exactly what one callable returns."""
  import threading
  lo, hi, fn = _quadratic_problem()
  th0 = ard.log_uniform_init(np.random.default_rng(5), 2, 0, 7)
  seen = [set() for _ in range(3)]

  def on_handle(j):
    def f(theta):
      seen[j].add(threading.get_ident())
      return fn(theta)
    return f

  one = ard.OptaxTrain(ard.adam(0.05), epochs=12)
  many = ard.OptaxTrain(ard.adam(0.05), epochs=12)
  best_1, final_1 = one(th0, fn, list(zip(lo, hi)), best_n=7)
  best_3, final_3 = many(th0, [on_handle(j) for j in range(3)], list(zip(lo, hi)), best_n=7)
  np.testing.assert_array_equal(final_1, final_3)
  np.testing.assert_array_equal(one.last_metrics['loss'], many.last_metrics['loss'])
  np.testing.assert_array_equal(np.array(best_1), np.array(best_3))
  assert all(seen)


def test_construction_errors():
  with pytest.raises(NotImplementedError):
    ard.OptaxTrain(ard.ScipyLbfgsB(), epochs=10)
  with pytest.raises(NotImplementedError):
    ard.OptaxTrain(object(), epochs=10)
  with pytest.raises(NotImplementedError):
    ard.OptaxTrain(ard.adam(1e-2), epochs=0)
  with pytest.raises(TypeError):
    ard.OptaxTrain(ard.adam(1e-2))          # epochs is a required keyword, as in the reference
  t = ard.OptaxTrain(ard.adam(1e-2), epochs=5, verbose=True)
  assert t.verbose == 1 and t.epochs == 5


def _problem(n_metrics=1):
  from vizier_b200 import vz
  problem = vz.ProblemStatement()
  problem.search_space.root.add_float_param('x', 0.0, 1.0)
  problem.search_space.root.add_categorical_param('c', ['a', 'b'])
  for m in range(n_metrics):
    problem.metric_information.append(vz.MetricInformation(name=f'm{m}', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  return problem


def test_separable_types_raise_and_designers_stay_off_the_device(monkeypatch):
  from vizier_b200.designers import gp_bandit
  from vizier_b200.designers import gp_ucb_pe

  def no_device(*a, **k):
    raise AssertionError('constructing a designer touched the device')

  monkeypatch.setattr(gp.DeviceGP, '__init__', no_device)
  adam_ard = ard.OptaxTrain(ard.adam(5e-2), epochs=100)
  gp_bandit.VizierGPBandit(_problem(), ard_optimizer=adam_ard, ensemble_size=2)
  gp_bandit.VizierGPBandit(_problem(2), ard_optimizer=adam_ard)
  gp_bandit.VizierGPBandit(_problem(), ard_optimizer=adam_ard, linear_coef=0.1)
  gp_ucb_pe.VizierGPUCBPEBandit(_problem(), ard_optimizer=adam_ard)
  gp_ucb_pe.VizierGPUCBPEBandit(_problem(2), ard_optimizer=adam_ard)
  for mt in ('SEPARABLE_NORMAL_TASK_KERNEL_PRIOR', 'SEPARABLE_LKJ_TASK_KERNEL_PRIOR', 'SEPARABLE_DIAG_TASK_KERNEL_PRIOR'):
    with pytest.raises(NotImplementedError):
      gp_bandit.VizierGPBandit(_problem(2), ard_optimizer=adam_ard, multitask_type=mt)
    with pytest.raises(NotImplementedError):
      ard.train_gp(None, np.zeros((3, 1)), np.zeros((3, 2)), rng=np.random.default_rng(0), optimizer=adam_ard,
                   multitask_type=mt)
