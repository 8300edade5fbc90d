"""Separable multi-task GP on the GPU against the dense oracle (separable_oracle.py): NLL, base and task-covariance
gradients of every type, the shared jitter shift, scalarised-UCB scores on every scoring route, the Eagle loop, the
joint posterior, and the designer end to end."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from oracle import eagle_oracle as eo  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402
import separable_oracle as so  # noqa: E402


def _setup(n, d, m, dk=0, seed=0, corr=0.6):
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, d))
  f = -np.sum((x - 0.3) ** 2, axis=1)
  y = np.stack([f * (1 + 0.2 * k) + corr * np.sin(3 * x[:, 0] + k) + 0.05 * rng.normal(size=n) for k in range(m)], 1)
  z = rng.integers(0, 3, size=(n, dk)).astype(np.int32) if dk else None
  ls2 = 0.5 * (1 + np.arange(d) / d)
  lk = np.linspace(0.7, 1.3, dk) if dk else None
  return rng, x, y, z, ls2, lk


def _theta(kind, m, rng):
  from vizier_b200 import task_kernels as tk
  th = tk.init(kind, rng, m, 1)[0]
  return np.clip(th, 0.3, 1.0) if kind == tk.DIAG else th


def _raw_batch(devs, m, ps, tcs, x, y, z, nv):
  """vzgp_nll_grad_separable_batch on R = len(ps) restarts: (losses, base grads, dL/dT, status)."""
  from vizier_b200 import _lib, gp
  f = devs[0]
  xt, zt = f._xz(x, z)
  n, dc = xt.shape
  yt, _ = f._labels(y, n)
  for d in devs[1:]:
    d._stream.wait_stream(torch.cuda.current_stream(d.device))
  dk = 0 if zt is None else zt.shape[1]
  r = len(ps)
  cps = (_lib.Params * r)(*[p._c() for p in ps])
  t = np.ascontiguousarray(np.stack(tcs), np.float64)
  loss, grad = np.zeros(r), np.zeros((r, dc + dk + 2))
  gt, st = np.zeros((r, m, m)), (C.c_int * r)()
  hs = (C.c_void_p * len(devs))(*[d._h for d in devs])
  pd = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
  _lib.check('vzgp_nll_grad_separable_batch', f._lib.vzgp_nll_grad_separable_batch(
      hs, r, m, gp._ptr(xt), gp._ptr(zt), gp._ptr(yt), n, dc, dk, nv, cps, pd(t), None, pd(loss), pd(grad), pd(gt), st))
  return loss, grad, gt, list(st)


@pytest.mark.parametrize('n,d,m,dk,nv', [(40, 3, 2, 0, 40), (130, 5, 3, 1, 120), (300, 6, 2, 0, 300)])
def test_separable_nll_grad_matches_oracle(n, d, m, dk, nv):
  from vizier_b200 import gp
  from vizier_b200 import task_kernels as tk
  rng, x, y, z, ls2, lk = _setup(n, d, m, dk, 1)
  valid = np.arange(n) < nv
  devs = [gp.DeviceGP(0) for _ in range(4 * m)]
  for kind in tk.TYPES:
    ps, tcs, want = [], [], []
    for r in range(4):
      po = go.GPParams(0.7 + 0.1 * r, ls2 * (1 + 0.05 * r), 2e-3, lk)
      t = so.task_cov(kind, _theta(kind, m, rng), m)
      ps.append(gp.GPHyperParams(po.signal_variance, po.continuous_length_scale_squared, 2e-3, lk))
      tcs.append(t)
      want.append(so.loss_and_grad(po, t, x, y, z, valid))
    for _ in range(2):   # capture, then graph replay
      loss, grad, gt, st = _raw_batch(devs, m, ps, tcs, x, y, z, nv)
      for r in range(4):
        wl, wg, wt, wi = want[r]
        assert st[r] == wi == 0
        assert abs(loss[r] - wl) < 1e-9 * max(1.0, abs(wl))
        np.testing.assert_allclose(grad[r], wg, atol=1e-8 * max(1.0, np.max(np.abs(wg))), rtol=0)
        np.testing.assert_allclose(gt[r], wt, atol=1e-8 * max(1.0, np.max(np.abs(wt))), rtol=0)
    one = _raw_batch(devs[:m], m, ps[2:3], tcs[2:3], x, y, z, nv)   # R = 1 equals restart 2 of the batch
    assert abs(one[0][0] - loss[2]) <= 1e-12 * abs(loss[2])
    np.testing.assert_allclose(one[1][0], grad[2], rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(one[2][0], gt[2], rtol=1e-12, atol=1e-14)
    routes = {dv.get_int('nll_route') for dv in devs}
    assert routes == ({2} if n <= 64 else {3})    # eager below 65 trials, graph branches above


def test_separable_jitter_uses_one_shift():
  """Every trial three times and sn2 = 1e-30 (the fixtures of test_gpu_fit_routes.py) with a rank-one T: alone, the
  eigen-task with lambda = 2 needs one retry and the one with lambda = 0 none, the dense matrix one.  Both tasks must
  be factored at the 1e-4 shift: the loss and the posterior match the dense oracle only then."""
  from vizier_b200 import _lib, gp
  rng = np.random.default_rng(5)
  x0 = rng.uniform(size=(30, 3))
  x = np.concatenate([x0] * 3)
  y = np.concatenate([rng.normal(size=(30, 2))] * 3)
  ls2 = 0.5 * (1 + np.arange(3) / 3)
  po = go.GPParams(1.0, ls2, 1e-30)
  pg = gp.GPHyperParams(1.0, ls2, 1e-30)
  t = np.ones((2, 2))
  wl, _, _, wi = so.loss_and_grad(po, t, x, y)
  assert wi == 1
  devs = [gp.DeviceGP(0) for _ in range(2)]
  loss, _, _, st = _raw_batch(devs, 2, [pg], [t], x, y, None, 90)
  assert st[0] == wi
  assert abs(loss[0] - wl) < 1e-7 * abs(wl)
  assert {d.get_int('nll_route') for d in devs} == {2}     # the ladder runs eagerly on both members
  sep = gp.SeparableGP(0, 2)
  f = sep.members[0]
  xt, _ = f._xz(x, None)
  yt, _ = f._labels(y, 90)
  p = pg._c()
  tc = np.ascontiguousarray(t)
  retries = _lib.check('vzgp_fit_separable', f._lib.vzgp_fit_separable(
      sep._handles(), 2, gp._ptr(xt), None, gp._ptr(yt), 90, 3, 0, 90, C.byref(p), tc.ctypes.data_as(C.POINTER(C.c_double))))
  assert retries == wi
  for d in [sep] + sep.members:
    d.n, d.dc, d.dk = 90, 3, 0
  xs = rng.uniform(size=(50, 3))
  mu, sd = so.marginals(po, t, x, y, xs)
  out = sep.score_multi(xs, gp.ScalarizedUcbAcquisition(np.array([[0.6, 0.8]]), np.zeros(2)), with_aux=True)
  sep.synchronize()
  np.testing.assert_allclose(out['mean'].cpu().numpy().T, mu, atol=1e-6, rtol=0)
  np.testing.assert_allclose(out['stddev'].cpu().numpy().T, sd, atol=1e-6, rtol=0)


@pytest.fixture(scope='module')
def big_model():
  from vizier_b200 import gp
  from vizier_b200 import task_kernels as tk
  rng, x, y, _, ls2, _ = _setup(1000, 20, 2, 0, 2)
  pg = gp.GPHyperParams(1.0, ls2, 1e-3, multitask_type=tk.LKJ, task_params=np.array([0.8, 0.9, 0.6]))
  po = go.GPParams(1.0, ls2, 1e-3)
  sep = gp.SeparableGP(0, 2)
  assert sep.fit(x, y, pg) == 0
  w = np.abs(rng.normal(size=(200, 2)))
  w /= np.linalg.norm(w, axis=1, keepdims=True)
  ref = go.hv_reference_point(y)
  best = go.hv_max_scalarized(y, w, ref)
  return rng, x, y, po, pg, sep, w, ref, best


@pytest.mark.parametrize('mc', [300, 5000, 20000])
def test_separable_scores_match_oracle(big_model, mc):
  from vizier_b200 import gp
  rng, x, y, po, pg, sep, w, ref, best = big_model
  xs = np.random.default_rng(mc).uniform(size=(mc, 20))
  pick = np.unique(np.concatenate([np.arange(min(mc, 300)), np.arange(0, mc, max(1, mc // 700))]))
  mu, sd = so.marginals(po, pg.task_covariance(), x, y, xs[pick])
  for floor in (best, None):
    out = sep.score_multi(xs, gp.ScalarizedUcbAcquisition(w, ref, floor, 1.8), with_aux=True)
    sep.synchronize()
    want = so.scalarized_ucb(mu, sd, w, ref, floor)
    np.testing.assert_allclose(out['mean'].cpu().numpy().T[pick], mu, atol=1e-10, rtol=0)
    np.testing.assert_allclose(out['stddev'].cpu().numpy().T[pick], sd, atol=1e-10, rtol=0)
    np.testing.assert_allclose(out['score'].cpu().numpy()[pick], want, atol=1e-10 * max(1.0, np.max(np.abs(want))), rtol=0)
  routes = {m.get_int('score_route') for m in sep.members}
  assert routes == {0} if mc == 300 else routes <= {1, 2}     # small-pool kernels, then k_score (split / cluster)


def test_identity_task_covariance_scores_as_independent():
  from vizier_b200 import gp
  from vizier_b200 import task_kernels as tk
  rng, x, y, z, ls2, lk = _setup(200, 6, 3, 2, 4)
  sep = gp.SeparableGP(0, 3)
  sep.fit(x, y, gp.GPHyperParams(1.0, ls2, 1e-3, lk, multitask_type=tk.DIAG, task_params=np.ones(3)), z=z)
  ind = gp.DeviceGP(0)
  ind.fit(x, y, gp.GPHyperParams(1.0, ls2, 1e-3, lk), z=z)
  xs = rng.uniform(size=(3000, 6))
  zs = rng.integers(0, 3, size=(3000, 2)).astype(np.int32)
  w = np.abs(rng.normal(size=(50, 3)))
  w /= np.linalg.norm(w, axis=1, keepdims=True)
  acq = gp.ScalarizedUcbAcquisition(w, go.hv_reference_point(y), None, 1.8)
  a = sep.score_multi(xs, acq, zs=zs, with_aux=True)
  b = ind.score_multi(xs, acq, zs=zs, with_aux=True)
  torch.cuda.synchronize()
  np.testing.assert_allclose(a['score'].cpu().numpy(), b['score'].cpu().numpy(), atol=1e-12, rtol=0)
  np.testing.assert_allclose(a['mean'].cpu().numpy(), b['mean'].cpu().numpy(), atol=1e-12, rtol=0)


def test_eagle_with_separable_scorer_matches_oracle():
  from vizier_b200 import _lib, gp
  from vizier_b200 import task_kernels as tk
  n, d, m = 80, 4, 2
  rng, x, y, _, ls2, _ = _setup(n, d, m, 0, 3)
  pg = gp.GPHyperParams(1.0, ls2, 1e-3, multitask_type=tk.NORMAL, task_params=np.array([0.3, 0.7, 0.1]))
  po = go.GPParams(1.0, ls2, 1e-3)
  t = pg.task_covariance()
  sep = gp.SeparableGP(0, m)
  sep.fit(x, y, pg)
  w = np.abs(rng.normal(size=(64, m)))
  w /= np.linalg.norm(w, axis=1, keepdims=True)
  ref = go.hv_reference_point(y)
  best = go.hv_max_scalarized(y, w, ref)

  def score_fn(q):
    mu, sd = so.marginals(po, t, x, y, q)
    return so.scalarized_ucb(mu, sd, w, ref, best)

  cfg_o = eo.EagleConfig()
  pool, batch, steps = 25, 25, 7
  wx, wr, _ = eo.run_eagle_optimizer(score_fn, dim=d, pool_size=pool, batch_size=batch, max_evaluations=steps * batch,
                                     count=3, seed=11, cfg=cfg_o, prior_features=x)
  cfg = _lib.EagleConfig(cfg_o.visibility, cfg_o.gravity, cfg_o.negative_gravity, cfg_o.perturbation,
                         cfg_o.perturbation_lower_bound, cfg_o.penalize_factor, cfg_o.normalization_scale,
                         cfg_o.prior_trials_pool_pct, pool, batch, steps * batch)
  bx, _, br = sep.eagle_run(cfg, gp.ScalarizedUcbAcquisition(w, ref, best, 1.8), count=3, seed=11, prior=x)
  np.testing.assert_allclose(br, wr, atol=1e-9 * max(1.0, np.max(np.abs(wr))))
  np.testing.assert_allclose(bx, wx, atol=1e-9)


@pytest.mark.parametrize('add_noise', [True, False])
def test_separable_joint_posterior_matches_oracle(add_noise):
  from vizier_b200 import gp
  from vizier_b200 import task_kernels as tk
  rng, x, y, z, ls2, lk = _setup(150, 4, 3, 1, 6)
  pg = gp.GPHyperParams(0.9, ls2, 5e-3, lk, multitask_type=tk.LKJ, task_params=np.array([0.5, -0.3, 1.2, 0.9, 0.6, 0.8]))
  po = go.GPParams(0.9, ls2, 5e-3, lk)
  sep = gp.SeparableGP(0, 3)
  sep.fit(x, y, pg, z=z)
  xs = rng.uniform(size=(9, 4))
  zs = rng.integers(0, 3, size=(9, 1)).astype(np.int32)
  mean, cov = sep.posterior(xs, zs, add_noise=add_noise)
  wm, wc = so.posterior(po, pg.task_covariance(), x, y, xs, z, zs, add_noise=add_noise)
  np.testing.assert_allclose(mean.cpu().numpy(), wm.T, atol=1e-10, rtol=0)
  np.testing.assert_allclose(cov.cpu().numpy(), so.to_metric_major(wc, 9, 3), atol=1e-10, rtol=0)


@pytest.mark.parametrize('nq', [63, 65, 129])
def test_separable_joint_posterior_across_query_tiles(nq):
  """The per-eigen-task posteriors cross the 64-row query tiles of k_cov_update and k_gemm_nt_tri before they are
  recombined into the [M n, M n] covariance."""
  from vizier_b200 import gp
  from vizier_b200 import task_kernels as tk
  rng, x, y, z, ls2, lk = _setup(150, 4, 2, 2, nq)
  pg = gp.GPHyperParams(0.9, ls2, 5e-3, lk, multitask_type=tk.NORMAL, task_params=np.array([0.8, 0.3, 1.1]))
  po = go.GPParams(0.9, ls2, 5e-3, lk)
  sep = gp.SeparableGP(0, 2)
  sep.fit(x, y, pg, z=z)
  xs = rng.uniform(size=(nq, 4))
  zs = rng.integers(0, 3, size=(nq, 2)).astype(np.int32)
  xs[:3], zs[:3] = x[:3], z[:3]
  xs[-1], zs[-1] = xs[nq // 2], zs[nq // 2]
  mean, cov = sep.posterior(xs, zs)
  wm, wc = so.posterior(po, pg.task_covariance(), x, y, xs, z, zs)
  np.testing.assert_allclose(mean.cpu().numpy(), wm.T, atol=1e-10, rtol=0)
  np.testing.assert_allclose(cov.cpu().numpy(), so.to_metric_major(wc, nq, 2), atol=1e-10, rtol=0)


@pytest.mark.parametrize('multitask_type', ['SEPARABLE_NORMAL_TASK_KERNEL_PRIOR', 'SEPARABLE_LKJ_TASK_KERNEL_PRIOR',
                                            'SEPARABLE_DIAG_TASK_KERNEL_PRIOR'])
def test_multi_metrics_separable_designer(multitask_type):
  """gp_bandit_test.py:476-510 (test_multi_metrics) for the separable types: suggest with both optimiser strategies,
  predictions of shape (n, M); two strongly correlated metrics give a fitted task correlation above 0.9."""
  from vizier_b200 import gp
  from vizier_b200 import optimizers as vb
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit
  p = vz.ProblemStatement()
  for i in range(3):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='a', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  p.metric_information.append(vz.MetricInformation(name='b', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  rng = np.random.default_rng(0)

  def evaluate(params):
    x = np.array([params[f'x{i}'].value for i in range(3)])
    f = float(-np.sum((x - 0.6) ** 2))
    return {'a': f, 'b': 2.0 * f + 0.1}

  for factory in (vb.VectorizedOptimizerFactory(strategy_factory=vb.VectorizedEagleStrategyFactory(), max_evaluations=1000,
                                                suggestion_batch_size=25),
                  vb.VectorizedOptimizerFactory(strategy_factory=vb.random_strategy_factory, max_evaluations=2000,
                                                suggestion_batch_size=2000)):
    d = gp_bandit.VizierGPBandit(p, rng=3, acquisition_optimizer_factory=factory, num_scalarizations=50,
                                 multitask_type=multitask_type)
    trials = []
    for i in range(20):
      xv = rng.uniform(size=3)
      t = vz.Trial(parameters={f'x{j}': float(xv[j]) for j in range(3)}, id=i + 1)
      t.complete(vz.Measurement(evaluate(t.parameters)))
      trials.append(t)
    d.update(vz.CompletedTrials(trials), vz.ActiveTrials())
    for step in range(2):
      sugg = d.suggest(2)
      assert len(sugg) == 2
      new = []
      for k, s in enumerate(sugg):
        assert p.search_space.contains(s.parameters)
        t = s.to_trial(100 + 10 * step + k)
        t.complete(vz.Measurement(evaluate(t.parameters)))
        new.append(t)
      d.update(vz.CompletedTrials(new), vz.ActiveTrials())
    assert isinstance(d._dev, gp.SeparableGP)
    t = d._last_params.task_covariance()
    if multitask_type != 'SEPARABLE_DIAG_TASK_KERNEL_PRIOR':
      assert t[0, 1] / np.sqrt(t[0, 0] * t[1, 1]) > 0.9
    s = d.sample(trials[:4], rng=1, num_samples=100)
    assert s.shape == (100, 4, 2)
    pred = d.predict(trials[:4], rng=1, num_samples=200)
    assert pred.mean.shape == (4, 2) and pred.stddev.shape == (4, 2)
