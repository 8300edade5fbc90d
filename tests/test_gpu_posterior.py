"""The joint posterior (vzgp_posterior_multi, csrc/c_abi.cu) against the fp64 oracle of posterior_oracle.py, the
factor the designers sample with, and every designer's sample() / predict() rebuilt on the host.

vzgp_posterior_multi builds K* and K** with k_cross_kernel on 64-row padded queries, W = K* L^-T with k_gemm_nt_tri,
C = K** - W W^T (+ sn2 I) with k_cov_update on an mp x mp grid of 64-row tiles, and one k_gemv_rows per metric for
the means.  The grid crosses the 64-row tiles of queries (M) and of training points (N), pads training rows
(n_valid < N), takes L^-1 from the panel kernels (N <= 64) or k_chol_dataflow (N > 64), and runs the wide
categorical kernels (Dk > 32).  Mean and covariance are held to 1e-10 absolute (DESIGN.md §2).

The designers' draws are rebuilt from the oracle posterior at the hyper-parameters the designer fitted, with the
designer's random stream and draw order, and unwarped by a warper fitted on each metric's labels alone."""
import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

import fit_fixtures as ff  # noqa: E402
import posterior_oracle as po_  # noqa: E402
import separable_oracle as so  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402
from oracle import hp_oracle as hp  # noqa: E402

TOL = 1e-10
PANEL, DATAFLOW = 0, 1        # vzgp_get_int "factor_route"
GRAPH = 1                     # vzgp_get_int "nll_route"


def _gp():
  from vizier_b200 import gp
  return gp


@pytest.fixture(scope='module')
def dev():
  d = _gp().DeviceGP(0)
  yield d
  d.close()


def _hyper(po):
  lin = po.linear
  kw = {} if lin is None else dict(linear_coef=lin.coef, linear_slope_amplitude=lin.slope_amplitude,
                                   linear_shift=lin.shift, mean_constant=lin.mean_constant)
  return _gp().GPHyperParams(po.signal_variance, po.continuous_length_scale_squared, po.observation_noise_variance,
                             po.categorical_length_scale_squared if po.categorical_length_scale_squared.size else None,
                             **kw)


def _params(dc, dk, linear=False, sn2=5e-3, scale=1.0):
  """Length scales that grow with the dimension, so K is neither diagonal nor of low numerical rank at Dc = 64 or
  Dk = 40."""
  ls_c = scale * 0.15 * dc * (1.0 + np.arange(dc) / dc)
  ls_k = scale * 0.5 * dk * np.linspace(0.6, 1.2, dk) if dk else None
  return go.GPParams(0.8 * scale, ls_c, sn2, ls_k, go.LinearParams(0.7, 0.9, 0.2, -0.3) if linear else None)


def _problem(n, m, dc, dk, metrics, seed):
  """Training set (x, z, y [N] or [N, metrics]) and queries (xs, zs) [M]: the first queries are training points,
  and some are duplicated."""
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, dc))
  z = rng.integers(0, 4, size=(n, dk)).astype(np.int32) if dk else None
  f = np.sin(3.0 * x[:, 0]) + np.mean(x, axis=1) + (0.3 * np.mean(z, axis=1) if dk else 0.0)
  y = f + 0.05 * rng.normal(size=n)
  if metrics > 1:
    y = np.stack([y * (1 + 0.5 * k) + 0.2 * k * np.cos(5.0 * x[:, -1]) for k in range(metrics)], 1)
  xs = rng.uniform(size=(m, dc))
  zs = rng.integers(0, 4, size=(m, dk)).astype(np.int32) if dk else None
  t = min(m, n, 3)
  xs[:t] = x[:t]
  if dk:
    zs[:t] = z[:t]
  for a, b in ((4, 3), (m - 1, m // 2)):
    if m > a and a != b:
      xs[a] = xs[b]
      if dk:
        zs[a] = zs[b]
  return x, z, y, xs, zs


def _assert_posterior(mean, cov, want_mean, want_cov):
  np.testing.assert_allclose(mean.cpu().numpy(), want_mean, atol=TOL, rtol=0)
  np.testing.assert_allclose(cov.cpu().numpy(), want_cov, atol=TOL, rtol=0)


def _assert_matches_score(d, xs, zs, mean, cov, sn2, add_noise, metrics):
  """vzgp_score / vzgp_score_multi at the same points: the mean and stddev^2 equal the posterior's mean and
  diagonal (the scores always carry the predictive noise)."""
  gp = _gp()
  if metrics > 1:
    acq = gp.ScalarizedUcbAcquisition(np.full((1, metrics), 1.0 / np.sqrt(metrics)), np.zeros(metrics), None, 0.0)
    out = d.score_multi(xs, acq, zs=zs, with_aux=True)
  else:
    out = d.score(xs, gp.Acquisition(1.8, False, 1.0), zs=zs, with_aux=True)
  d.synchronize()
  var = np.diag(cov.cpu().numpy()) + (0.0 if add_noise else sn2)
  np.testing.assert_allclose(out['mean'].cpu().numpy(), mean.cpu().numpy(), atol=TOL, rtol=0)
  np.testing.assert_allclose(out['stddev'].cpu().numpy() ** 2, var, atol=TOL, rtol=0)


# (M queries, N training points, n_valid, Dc, Dk, model, add_noise); every value of each axis appears at least once.
CASES = [
    (1, 1, 1, 1, 0, 'gp', True),
    (2, 5, 3, 20, 3, 'linear', False),
    (63, 64, 64, 1, 3, 'metrics2', True),
    (64, 65, 65, 20, 0, 'gp', False),
    (65, 200, 170, 64, 0, 'linear', True),
    (128, 64, 50, 20, 40, 'gp', True),
    (129, 200, 200, 1, 40, 'metrics8', False),
    (300, 1000, 1000, 20, 3, 'gp', True),
    (1000, 65, 60, 20, 0, 'metrics2', False),
    (65, 1000, 950, 20, 40, 'ensemble', True),
    (129, 5, 5, 20, 3, 'ensemble', False),
    (65, 4097, 4000, 8, 2, 'gp', True),       # k_cov_update and the mean gemv against np = 4160
]


@pytest.mark.parametrize('m,n,nv,dc,dk,model,add_noise', CASES)
def test_posterior_matches_oracle(dev, m, n, nv, dc, dk, model, add_noise):
  gp = _gp()
  metrics = {'metrics2': 2, 'metrics8': 8}.get(model, 1)
  x, z, y, xs, zs = _problem(n, m, dc, dk, metrics, seed=m + 7 * n + dc + dk)
  route = DATAFLOW if n > 64 else PANEL
  valid = np.arange(n) < nv
  if model == 'ensemble':
    pos = [_params(dc, dk, sn2=s, scale=c) for s, c in ((5e-3, 1.0), (2e-2, 0.6), (1e-3, 1.5))]
    ens = gp.EnsembleGP(0, len(pos))
    try:
      ens.fit(x, y, [_hyper(p) for p in pos], z=z, n_valid=nv)
      comps = ens.posterior(xs, zs, add_noise=add_noise)
      for mem, p, (mean, cov) in zip(ens.members, pos, comps):
        assert mem.get_int('factor_route') == route
        pred = go.precompute_predictive(p, x, y, z, row_valid=valid)
        _assert_posterior(mean, cov, *po_.joint_posterior(pred, xs, zs, add_noise))
        _assert_matches_score(mem, xs, zs, mean, cov, p.observation_noise_variance, add_noise, 1)
    finally:
      for mem in ens.members:
        mem.close()
    return
  p = _params(dc, dk, linear=model == 'linear')
  assert dev.fit(x, y, _hyper(p), z=z, n_valid=nv) == 0
  assert dev.get_int('factor_route') == route
  mean, cov = dev.posterior(xs, zs, add_noise=add_noise)
  assert tuple(mean.shape) == ((metrics, m) if metrics > 1 else (m,))
  pred = go.precompute_predictive(p, x, y, z, row_valid=valid)
  _assert_posterior(mean, cov, *po_.joint_posterior(pred, xs, zs, add_noise))
  _assert_matches_score(dev, xs, zs, mean, cov, p.observation_noise_variance, add_noise, metrics)


@pytest.mark.skipif(not hp.has_extended_precision(), reason='np.longdouble is fp64 on this platform')
def test_ill_conditioned_posterior_vs_long_double(dev):
  """sn2 = 1e-8, ls2 = 0.05 and duplicated trials (cond(K_y) ~ 1e10): the posterior stddev within 1e-7 of the
  long-double one, the mean as accurate as the fp64 oracle's (test_gpu_score_routes.py measures the same inputs)."""
  n, d, m = 300, 6, 200
  rng = np.random.default_rng(77)
  x = rng.uniform(size=(n, d))
  x[1::10] = x[0::10]
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  p = go.GPParams(1.0, np.full(d, 0.05), 1e-8)
  xs = rng.uniform(size=(m, d))
  near = rng.permutation(m)[:m // 4]
  xs[near] = x[rng.integers(0, n, near.size)] + rng.uniform(-0.02, 0.02, size=(near.size, d))
  assert dev.fit(x, y, _hyper(p)) == 0
  assert dev.get_int('factor_route') == DATAFLOW
  mean, cov = dev.posterior(xs, add_noise=True)
  mu_h, sd_h = hp.predict(hp.precompute_predictive(p, x, y), xs)
  mu_f, _ = go.predict(go.precompute_predictive(p, x, y), xs)
  sd = np.sqrt(np.maximum(np.diag(cov.cpu().numpy()), 0.0))
  assert np.max(np.abs((sd - sd_h).astype(np.float64))) < 1e-7
  err_f = float(np.max(np.abs((mu_f - mu_h).astype(np.float64))))
  assert float(np.max(np.abs((mean.cpu().numpy() - mu_h).astype(np.float64)))) <= 4.0 * err_f + 1e-12


@pytest.mark.parametrize('m,dk', [(65, 0), (130, 3)])
def test_leading_dimension_leaves_the_padding_alone(dev, m, dk):
  """ldc > M through the C ABI: the M x M block equals the dense call bit for bit, the padding columns keep their
  sentinel bits."""
  from vizier_b200 import _lib
  gp = _gp()
  x, z, y, xs, zs = _problem(100, m, 4, dk, 1, seed=m)
  dev.fit(x, y, _hyper(_params(4, dk)), z=z)
  want_mean, want_cov = dev.posterior(xs, zs)
  ldc = m + 7
  xst, zst = dev._xz(xs, zs)
  mean = torch.empty((m,), dtype=torch.float64, device=dev.device)
  cov = torch.full((m, ldc), -7.25e300, dtype=torch.float64, device=dev.device)
  sentinel = cov[0, 0].view(torch.int64).item()
  dev._stream.wait_stream(torch.cuda.current_stream(dev.device))
  _lib.check('vzgp_posterior_multi', dev._lib.vzgp_posterior_multi(
      dev._h, gp._ptr(xst), gp._ptr(zst), m, 1, gp._ptr(mean), gp._ptr(cov), ldc))
  dev.synchronize()
  assert torch.equal(cov[:, :m], want_cov) and torch.equal(mean, want_mean)
  assert bool((cov[:, m:].contiguous().view(torch.int64) == sentinel).all())


def test_posterior_growing_kinv_leaves_nll_graph_and_scores_intact():
  """The posterior writes its workspace into the handle's Kinv buffer, which the captured NLL graph also points
  into.  M = 1000 on np = 128 grows that buffer: the next NLL evaluation must notice, give the same loss and
  gradient bit for bit and replay a graph again; scores before and after are bit-identical."""
  gp = _gp()
  x, z, y, xs, _ = _problem(128, 1000, 5, 0, 1, seed=5)
  p = _params(5, 0)
  a, b = gp.DeviceGP(0), gp.DeviceGP(0)
  try:
    xt, yt = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    l1, g1, _ = a.loss_and_grad(xt, yt, _hyper(p))
    l1b, g1b, _ = a.loss_and_grad(xt, yt, _hyper(p))
    assert a.get_int('nll_route') == GRAPH
    a.fit(x, y, _hyper(p))              # an NLL evaluation replaces the fitted model: the posterior needs a fit
    a.posterior(xs)
    l2, g2, _ = a.loss_and_grad(xt, yt, _hyper(p))
    assert a.get_int('nll_route') == GRAPH
    assert l1 == l1b == l2
    np.testing.assert_array_equal(g1, g2)
    np.testing.assert_array_equal(g1, g1b)

    b.fit(x, y, _hyper(p))
    acq = gp.Acquisition(1.8, False, 1.0)
    q = np.random.default_rng(9).uniform(size=(3000, 5))
    before = {k: v.clone() for k, v in b.score(q, acq, with_aux=True).items() if k != '_inputs'}
    b.synchronize()
    b.posterior(xs)
    after = b.score(q, acq, with_aux=True)
    b.synchronize()
    for k, v in before.items():
      assert torch.equal(v, after[k]), k
  finally:
    a.close()
    b.close()


# ---------------------------------------------------------------------------------------------------------------
# The factor the designers sample with: cholesky_retry(cov, jitter=1e-10, max_iters=8)
# ---------------------------------------------------------------------------------------------------------------
def _check_retry(dev, cov):
  l, shift, retries = dev.cholesky_retry(cov, jitter=1e-10, max_iters=8)
  assert dev.get_int('factor_route') == PANEL
  l = l.cpu().numpy()
  want_l, want_shift, want_it = go.retrying_cholesky(cov, 1e-10, 8)
  if np.isnan(want_l).any():
    assert retries == 9 and np.isnan(l).any()
    return retries
  assert (retries, shift) == (want_it, want_shift)
  a = cov + shift * np.eye(cov.shape[0])
  ev = np.linalg.eigvalsh(a)
  scale = max(1.0, np.max(np.abs(want_l)))
  assert np.max(np.abs(l @ l.T - a)) <= 1e-13 * max(1.0, np.max(np.abs(a)))
  np.testing.assert_allclose(l, want_l, atol=max(1e-12, 1e-15 * ev[-1] / ev[0]) * scale, rtol=0)
  assert np.all(np.triu(l, 1) == 0)
  return retries


@pytest.mark.parametrize('m', [1, 2, 17, 64, 65])
def test_sampling_factor_of_device_covariances(dev, m):
  """Well-conditioned posteriors, and duplicated queries with noise 1e-10 (cov singular up to the noise)."""
  x, z, y, xs, zs = _problem(30, m, 3, 2, 1, seed=3 * m)
  dev.fit(x, y, _hyper(_params(3, 2)), z=z)
  _, cov = dev.posterior(xs, zs)
  assert _check_retry(dev, cov.cpu().numpy()) == 0
  dup = np.repeat(xs[:(m + 1) // 2], 2, axis=0)[:m]
  zdup = np.repeat(zs[:(m + 1) // 2], 2, axis=0)[:m]
  dev.fit(x, y, _hyper(_params(3, 2, sn2=1e-10)), z=z)
  _, cov = dev.posterior(dup, zdup)
  _check_retry(dev, cov.cpu().numpy())


# lambda_min -> retries on the 1e-10 ladder (shift k = 1e-10 * 10^(k-1)), 3x inside each interval; 9 = exhausted
LADDER_1E10 = {0: 1e-2, 1: -3e-11, 2: -3e-10, 3: -3e-9, 6: -3e-6, 8: -3e-4, 9: -3.0}


@pytest.mark.parametrize('m', [2, 64, 65])
def test_sampling_factor_ladder(dev, m):
  for want, lam in LADDER_1E10.items():
    a = ff.spd_with_lambda_min(m, lam, seed=m + want)
    assert _check_retry(dev, a) == want, (m, want)


# ---------------------------------------------------------------------------------------------------------------
# Designers: sample() and predict() rebuilt on the host
# ---------------------------------------------------------------------------------------------------------------
NUM_SAMPLES = 64
SEED = 5


def _designer_problem(n_metrics, categorical=False):
  from vizier_b200 import vz
  p = vz.ProblemStatement()
  p.search_space.root.add_float_param('x0', -2.0, 2.0)
  p.search_space.root.add_float_param('x1', 0.0, 1.0)
  if categorical:
    p.search_space.root.add_categorical_param('c', ['a', 'b', 'c'])
  for k in range(n_metrics):
    p.metric_information.append(vz.MetricInformation(name=f'm{k}', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  return p


def _metric_values(x0, x1, c, n_metrics, scales):
  f = np.sin(1.5 * x0) - (x1 - 0.4) ** 2 + 0.2 * c
  return {f'm{k}': float(scales[k][0] + scales[k][1] * (f + 0.3 * k * x1)) for k in range(n_metrics)}


def _trials(n, n_metrics, seed, categorical=False, start=1, scales=None):
  from vizier_b200 import vz
  scales = scales or [(0.0, 1.0 + k) for k in range(n_metrics)]
  rng = np.random.default_rng(seed)
  out = []
  for i in range(n):
    params = {'x0': float(rng.uniform(-2, 2)), 'x1': float(rng.uniform())}
    c = int(rng.integers(0, 3))
    if categorical:
      params['c'] = 'abc'[c]
    t = vz.Trial(parameters=params, id=start + i)
    t.complete(vz.Measurement(_metric_values(params['x0'], params['x1'], c if categorical else 0, n_metrics, scales)))
    out.append(t)
  return out


def _queries(categorical=False):
  from vizier_b200 import vz
  pts = [(-1.7, 0.9, 'b'), (0.3, 0.15, 'a'), (1.1, 0.55, 'c'), (1.9, 0.05, 'a')]
  return [vz.Trial(parameters={'x0': a, 'x1': b, **({'c': c} if categorical else {})}) for a, b, c in pts]


def _unwarp(raw, m, warped):
  """Unwarps warped samples of metric m with a default warper fitted on metric m's labels alone."""
  from vizier_b200 import output_warpers
  w = output_warpers.create_default_warper()
  w.warp(raw[:, m:m + 1])
  return w.unwarp(warped.reshape(-1, 1)).reshape(warped.shape)


def _assert_samples(got, want, d=None, trials=None, rng=None):
  """sample() within 1e-8 of each metric's sample spread; with a designer, predict() its sample mean and stddev."""
  got, want = np.asarray(got), np.asarray(want)
  assert got.shape == want.shape
  g3, w3 = got.reshape(got.shape[0], got.shape[1], -1), want.reshape(want.shape[0], want.shape[1], -1)
  for m in range(w3.shape[2]):
    spread = float(np.std(w3[:, :, m]))
    assert spread > 0
    np.testing.assert_allclose(g3[:, :, m], w3[:, :, m], atol=1e-8 * spread, rtol=0, err_msg=f'metric {m}')
  if d is None:
    return
  pred = d.predict(trials, rng=rng, num_samples=want.shape[0])
  for m in range(w3.shape[2]):
    spread = float(np.std(w3[:, :, m]))
    mean, sd = np.asarray(pred.mean).reshape(len(trials), -1), np.asarray(pred.stddev).reshape(len(trials), -1)
    np.testing.assert_allclose(mean[:, m], w3[:, :, m].mean(0), atol=1e-8 * spread, rtol=0)
    np.testing.assert_allclose(sd[:, m], w3[:, :, m].std(0), atol=1e-8 * spread, rtol=0)


def _host_inputs(d, trials):
  cont, cat = d._converter.to_features(trials)
  zq = cat if cat.shape[1] else None
  return np.nan_to_num(cont, nan=0.0), zq


def _expected_bandit(d, trials):
  """VizierGPBandit.sample rebuilt on the host from the oracle posterior (non-stacked models)."""
  from vizier_b200.designers import gp_bandit
  cont, cat, labels = d._trials_to_data(d._trials)
  _, raw = d._converter.to_xy(d._trials)
  z = cat if cat.shape[1] else None
  xs, zs = _host_inputs(d, trials)
  g = np.random.default_rng(gp_bandit._seed_from(SEED))
  nm = labels.shape[1]
  if d._multitask_type:
    hpar = d._last_params
    mean, cov = so.posterior(po_.to_oracle_params(hpar), hpar.task_covariance(), cont, labels, xs, z, zs)
    n = xs.shape[0]
    chol = po_.factor(so.to_metric_major(cov, n, nm))
    normals = g.standard_normal((NUM_SAMPLES, nm * n))
    warped = (mean.T.reshape(-1)[None, :] + normals @ chol.T).reshape(NUM_SAMPLES, nm, n)
    return np.stack([_unwarp(raw, m, warped[:, m, :]) for m in range(nm)], axis=-1)
  y = labels[:, 0] if nm == 1 else labels
  params = d._last_params if isinstance(d._last_params, list) else [d._last_params]
  comps = [po_.joint_posterior(go.precompute_predictive(po_.to_oracle_params(p), cont, y, z), xs, zs) for p in params]
  if nm == 1:
    return _unwarp(raw, 0, po_.mixture_draws(comps, g, NUM_SAMPLES))
  mean, cov = comps[0]
  chol = po_.factor(cov)
  out = []
  for m in range(nm):
    out.append(_unwarp(raw, m, mean[m][None, :] + g.standard_normal((NUM_SAMPLES, xs.shape[0])) @ chol.T))
  return np.stack(out, axis=-1)


BANDIT_FORMS = {
    'gp': (1, {}, False),
    'ensemble': (1, {'ensemble_size': 3}, False),
    'linear': (1, {'linear_coef': 0.4}, False),
    'categorical': (1, {}, True),
    'metrics': (2, {}, False),
    'metrics-categorical': (3, {}, True),
    'separable-normal': (2, {'multitask_type': 'SEPARABLE_NORMAL_TASK_KERNEL_PRIOR'}, False),
    'separable-lkj': (2, {'multitask_type': 'SEPARABLE_LKJ_TASK_KERNEL_PRIOR'}, False),
    'separable-diag': (2, {'multitask_type': 'SEPARABLE_DIAG_TASK_KERNEL_PRIOR'}, False),
}


@pytest.mark.parametrize('form', list(BANDIT_FORMS))
def test_bandit_sample_reproduced(form):
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit
  nm, kw, categorical = BANDIT_FORMS[form]
  d = gp_bandit.VizierGPBandit(_designer_problem(nm, categorical), rng=1, **kw)
  d.update(vz.CompletedTrials(_trials(18, nm, 2, categorical)), vz.ActiveTrials())
  q = _queries(categorical)
  got = d.sample(q, rng=SEED, num_samples=NUM_SAMPLES)
  _assert_samples(got, _expected_bandit(d, q), d, q, SEED)


@pytest.mark.parametrize('n_metrics', [1, 2])
def test_bandit_stack_sample_reproduced(monkeypatch, n_metrics):
  """Transfer-learning stacks: each level's hyper-parameters and residual labels as the designer trained them; the
  combined prediction is a diagonal normal per metric."""
  from vizier_b200 import ard, vz
  from vizier_b200.designers import gp_bandit
  levels = []
  train = ard.train_gp

  def record(dev, x, y, z=None, **kw):
    best, losses = train(dev, x, y, z, **kw)
    levels.append((x, np.array(y), z, best[0]))
    return best, losses

  monkeypatch.setattr(ard, 'train_gp', record)
  d = gp_bandit.VizierGPBandit(_designer_problem(n_metrics), rng=1)
  d.set_priors([vz.CompletedTrials(_trials(30, n_metrics, 3)), vz.CompletedTrials(_trials(20, n_metrics, 4, 100))])
  d.update(vz.CompletedTrials(_trials(12, n_metrics, 5, 200)), vz.ActiveTrials())
  q = _queries()
  got = d.sample(q, rng=SEED, num_samples=NUM_SAMPLES)
  assert len(levels) == 3
  preds = [go.precompute_predictive(po_.to_oracle_params(p), x, y, z) for x, y, z, p in levels]
  xs, zs = _host_inputs(d, q)
  mean, sd = go.predict_stack(preds, xs, zs)
  _, raw = d._converter.to_xy(d._trials)
  g = np.random.default_rng(gp_bandit._seed_from(SEED))
  mean = mean.reshape(xs.shape[0], -1)
  if n_metrics == 1:
    want = _unwarp(raw, 0, mean[:, 0][None, :] + g.standard_normal((NUM_SAMPLES, xs.shape[0])) * sd[None, :])
  else:
    want = np.stack([_unwarp(raw, m, mean[:, m][None, :] + g.standard_normal((NUM_SAMPLES, xs.shape[0])) * sd[None, :])
                     for m in range(n_metrics)], axis=-1)
  _assert_samples(got, want, d, q, SEED)


@pytest.mark.parametrize('form', ['gp', 'ensemble', 'metrics'])
def test_ucb_pe_sample_reproduced(form):
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit, gp_ucb_pe
  nm = 2 if form == 'metrics' else 1
  d = gp_ucb_pe.VizierGPUCBPEBandit(_designer_problem(nm), rng=1, ensemble_size=3 if form == 'ensemble' else 1)
  fitted = []
  build = d._build_gp_model_and_optimize_parameters

  def record(*a):
    fitted.append(build(*a))
    return fitted[-1]

  d._build_gp_model_and_optimize_parameters = record
  d.update(vz.CompletedTrials(_trials(18, nm, 2)), vz.ActiveTrials())
  q = _queries()
  got = d.sample(q, rng=SEED, num_samples=NUM_SAMPLES)
  cont, cat, labels = d._trials_to_data(d._all_completed_trials)
  _, raw = d._converter.to_xy(d._all_completed_trials)
  xs, zs = _host_inputs(d, q)
  params = fitted[-1] if isinstance(fitted[-1], list) else [fitted[-1]]
  y = d._fit_labels(labels)
  comps = [po_.joint_posterior(go.precompute_predictive(po_.to_oracle_params(p), cont, y, None), xs, zs) for p in params]
  g = np.random.default_rng(gp_bandit._seed_from(SEED))
  if nm == 1:
    want = _unwarp(raw, 0, po_.mixture_draws(comps, g, NUM_SAMPLES))
  else:
    mean, cov = comps[0]
    chol = po_.factor(cov)
    want = np.stack([_unwarp(raw, m, mean[m][None, :] + g.standard_normal((NUM_SAMPLES, xs.shape[0])) @ chol.T)
                     for m in range(nm)], axis=-1)
  # predict() retrains with the designer's advancing stream (new ARD restarts), so only sample() is reproduced
  _assert_samples(got, want)


SCALES = [(1.0e6, 5.0e4), (-3.0, 0.1)]


@pytest.mark.parametrize('designer,kw', [
    ('bandit', {}),
    ('bandit', {'multitask_type': 'SEPARABLE_LKJ_TASK_KERNEL_PRIOR'}),
    ('bandit-stack', {}),
    ('ucb_pe', {}),
], ids=['independent', 'separable', 'stack', 'ucb-pe'])
def test_each_metric_predicted_on_its_own_scale(designer, kw):
  """Two metrics about 10^6 apart: each metric's predicted mean lies in that metric's label range."""
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit, gp_ucb_pe
  if designer == 'ucb_pe':
    d = gp_ucb_pe.VizierGPUCBPEBandit(_designer_problem(2), rng=1)
  else:
    d = gp_bandit.VizierGPBandit(_designer_problem(2), rng=1, **kw)
  if designer == 'bandit-stack':
    d.set_priors([vz.CompletedTrials(_trials(20, 2, 3, scales=SCALES))])
  trials = _trials(18, 2, 2, scales=SCALES)
  d.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  pred = d.predict(trials[:6] + _queries(), rng=1, num_samples=300)
  labels = np.array([[t.final_measurement.metrics[f'm{k}'].value for k in range(2)] for t in trials])
  lo, hi = labels.min(0), labels.max(0)
  pad = 0.1 * (hi - lo)
  mean = np.asarray(pred.mean)
  assert mean.shape == (10, 2)
  for k in range(2):
    assert np.all((mean[:, k] >= lo[k] - pad[k]) & (mean[:, k] <= hi[k] + pad[k])), (k, mean[:, k], lo[k], hi[k])
