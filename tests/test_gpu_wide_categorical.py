"""Models with more than 32 categorical features (csrc: the WIDE kernel forms, tiles.cuh for_cat_tiles) against the
oracle: kernel matrices, fits, every NLL + gradient route, scoring on the general route, Eagle on the replayed graph
and the stepped loop, random search, and the designers.

The duplication identity ties the wide forms to the narrow ones: a Dk = 64 model whose categorical columns are each
repeated twice, with doubled length scales, is the Dk = 32 model up to the order of the Hamming sum.
"""
import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

import eagle_lockstep as el  # noqa: E402
import eagle_options_oracle as xo  # noqa: E402
import fit_fixtures as ff  # noqa: E402
from oracle import eagle_oracle as eo  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402

SMALL, GRAPH, EAGER, BATCH = 0, 1, 2, 3          # vzgp_nll_route
ROUTE_GENERAL = 4                                # vzgp_score_route
EAGLE_GRAPH, EAGLE_STEPPED = 2, 3                # vzgp_eagle_route
UCB = 1.8


def _gp():
  from vizier_b200 import gp
  return gp


def _hyper(po):
  return _gp().GPHyperParams(po.signal_variance, po.continuous_length_scale_squared, po.observation_noise_variance,
                             po.categorical_length_scale_squared)


def _cuda(a, dtype=torch.float64):
  return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to('cuda', dtype)


def _data(n, dc, dk, seed, sizes=3):
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, dc))
  z = rng.integers(0, sizes, size=(n, dk)).astype(np.int32)
  y = (np.sin(3.0 * x.sum(1)) if dc else 0.0) + 0.3 * np.cos(z[:, :5].sum(1)) + 0.05 * rng.normal(size=n)
  # length scales of the order of Dk: the Hamming term stays O(1), so K is far from the identity
  po = go.GPParams(0.8, 0.3 * (1.0 + np.arange(dc) / max(dc, 1)), 2e-3, np.linspace(0.5, 1.5, dk) * dk / 4)
  return x, y, z, po


@pytest.fixture(scope='module')
def dev():
  d = _gp().DeviceGP(0)
  yield d
  d.close()


# ---------------------------------------------------------------------------------------------------------------
# A. kernel matrix and cross kernel
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dk', [33, 64, 65, 100, 257])
@pytest.mark.parametrize('dc', [0, 3, 20])
def test_kernel_matrices(dev, dc, dk):
  x, _, z, po = _data(70, dc, dk, dk + dc)
  nv = 61
  k = dev.kernel_matrix(x, _hyper(po), z=z, n_valid=nv, diag_add=po.observation_noise_variance).cpu().numpy()
  want = go.kernel_matrix(po, x, z, row_valid=np.arange(70) < nv)    # K + sn2 I on the valid rows
  np.testing.assert_allclose(k, want, atol=1e-13, rtol=0)
  xs, _, zs, _ = _data(130, dc, dk, dk + dc + 1)
  ks = dev.cross_kernel(xs, x, _hyper(po), zs=zs, z=z).cpu().numpy()
  np.testing.assert_allclose(ks, go.kernel(po, xs, x, zs, z), atol=1e-13, rtol=0)


# ---------------------------------------------------------------------------------------------------------------
# B. NLL + gradient on every route
# ---------------------------------------------------------------------------------------------------------------
def _assert_nll(loss, grad, want_l, want_g, po, skip_noise):
  reg = go.regularizer(po)
  assert abs((loss - reg) - (want_l - reg)) < 1e-9 * max(1.0, abs(want_l - reg)), (loss, want_l)
  keep = np.ones(len(want_g), bool)
  if skip_noise:
    keep[-2] = False
  scale = max(1.0, float(np.max(np.abs(want_g[keep]))))
  np.testing.assert_allclose(grad[keep], want_g[keep], atol=1e-8 * scale, rtol=0)


# (n, dc, dk, n_valid, n_metrics, route with one jitter retry, route without)
NLL_CASES = [
    (5, 3, 33, 5, 1, SMALL, SMALL),
    (64, 0, 100, 50, 1, SMALL, SMALL),
    (60, 20, 257, 40, 1, SMALL, SMALL),
    (64, 3, 65, 44, 2, EAGER, GRAPH),
    (65, 3, 64, 65, 1, EAGER, GRAPH),
    (200, 20, 100, 180, 1, EAGER, GRAPH),
    (1000, 3, 33, 990, 1, EAGER, GRAPH),
]


@pytest.mark.parametrize('n,dc,dk,nv,m,route_bad,route_good', NLL_CASES)
def test_nll_every_route(dev, n, dc, dk, nv, m, route_bad, route_good):
  x, y, z, po = ff.case_inputs('tripled', n, dc, dk, m, 1e-30)
  valid = np.arange(n) < nv
  assert go.retrying_cholesky(go.kernel_matrix(po, x, z, valid))[2] == 1
  want_l, want_g = go.loss_and_grad(po.to_vector(), x, y, z, valid)
  xt, yt, zt = _cuda(x), _cuda(y), _cuda(z, torch.int32)
  loss, grad, retries = dev.loss_and_grad(xt, yt, _hyper(po), z=zt, n_valid=nv)
  assert dev.get_int('nll_route') == route_bad and retries == 1
  _assert_nll(loss, grad, want_l, want_g, po, skip_noise=True)
  good = go.GPParams(po.signal_variance, po.continuous_length_scale_squared, 1e-2, po.categorical_length_scale_squared)
  want_l, want_g = go.loss_and_grad(good.to_vector(), x, y, z, valid)
  f = dev.make_loss_fn(xt, yt, zt, n_valid=nv)
  l2, g2 = f(_hyper(good).to_vector())
  assert dev.get_int('nll_route') == route_good
  _assert_nll(l2, g2, want_l, want_g, good, skip_noise=False)
  l3, g3 = f(_hyper(good).to_vector())     # the graph replayed with the same parameters
  assert l3 == l2 and np.array_equal(g3, g2)


@pytest.mark.parametrize('n,dc,dk', [(129, 3, 40), (300, 0, 257)])
def test_nll_batch_route(n, dc, dk):
  gp = _gp()
  x, y, z, po = ff.case_inputs('well', n, dc, dk, 1, 1e-2)
  devs = [gp.DeviceGP(0) for _ in range(3)]
  try:
    f = gp.DeviceGP.make_batch_loss_fn(devs, _cuda(x), _cuda(y), _cuda(z, torch.int32))
    thetas = []
    for r in range(3):
      pr = go.GPParams(po.signal_variance * (1 + 0.1 * r), po.continuous_length_scale_squared,
                       po.observation_noise_variance, po.categorical_length_scale_squared * (1 + 0.2 * r))
      thetas.append(pr)
    losses, grads = f(list(range(3)), [_hyper(p).to_vector() for p in thetas])
    for r, pr in enumerate(thetas):
      assert devs[r].get_int('nll_route') == BATCH
      want_l, want_g = go.loss_and_grad(pr.to_vector(), x, y, z)
      _assert_nll(losses[r], grads[r], want_l, want_g, pr, skip_noise=False)
  finally:
    for d in devs:
      d.close()


def test_linear_coef():
  """The linear_coef model: NLL + gradient on the eager route, scoring on the general route."""
  gp = _gp()
  x, y, z, po = _data(90, 3, 40, 3)
  d = gp.DeviceGP(0)
  try:
    lin = go.GPParams(po.signal_variance, po.continuous_length_scale_squared, po.observation_noise_variance,
                      po.categorical_length_scale_squared, go.LinearParams(0.7, 0.9, 0.2, -0.3))
    hp = gp.GPHyperParams(lin.signal_variance, lin.continuous_length_scale_squared, lin.observation_noise_variance,
                          lin.categorical_length_scale_squared, linear_coef=0.7, linear_slope_amplitude=0.9,
                          linear_shift=0.2, mean_constant=-0.3)
    loss, grad, _ = d.loss_and_grad(_cuda(x), _cuda(y), hp, z=_cuda(z, torch.int32))
    assert d.get_int('nll_route') == EAGER
    want_l, want_g = go.loss_and_grad(lin.to_vector(), x, y, z, linear_coef=0.7)
    _assert_nll(loss, grad, want_l, want_g, lin, skip_noise=False)
    d.fit(x, y, hp, z=z)
    xs, _, zs, _ = _data(300, 3, 40, 4)
    out = d.score(xs, gp.Acquisition(UCB, False, 1.0), zs=zs, with_aux=True)
    d.synchronize()
    assert d.get_int('score_route') == ROUTE_GENERAL
    mu, sd = go.predict(go.precompute_predictive(lin, x, y, z), xs, zs)
    np.testing.assert_allclose(out['mean'].cpu().numpy(), mu, atol=1e-10, rtol=0)
    np.testing.assert_allclose(out['stddev'].cpu().numpy(), sd, atol=1e-10, rtol=0)
  finally:
    d.close()


# ---------------------------------------------------------------------------------------------------------------
# C. fit and scoring on the general route
# ---------------------------------------------------------------------------------------------------------------
FIT_CASES = [(5, 3, 33, 5), (64, 0, 100, 50), (65, 20, 65, 65), (1000, 3, 257, 990)]


@pytest.mark.parametrize('n,dc,dk,nv', FIT_CASES)
def test_fit_score_posterior(dev, n, dc, dk, nv):
  gp = _gp()
  x, y, z, po = _data(n, dc, dk, n + dk)
  valid = np.arange(n) < nv
  pred = go.precompute_predictive(po, x, y, z, row_valid=valid)
  assert dev.fit(x, y, _hyper(po), z=z, n_valid=nv) == pred.n_retries
  np.testing.assert_allclose(dev.alpha().cpu().numpy(), pred.alpha, atol=1e-8 * np.max(np.abs(pred.alpha)), rtol=0)
  for m in (1, 25, 4097, 100_000):
    xs, _, zs, _ = _data(m, dc, dk, m)
    out = dev.score(xs, gp.Acquisition(UCB, False, 1.0), zs=zs, with_aux=True)
    dev.synchronize()
    assert dev.get_int('score_route') == ROUTE_GENERAL
    mu, sd, sc = (out[k].cpu().numpy() for k in ('mean', 'stddev', 'score'))
    assert np.isfinite(sc).all()
    idx = np.unique(np.r_[0, m - 1, np.arange(4090, 4100), np.arange(8190, 8194)] % m) if m > 200 else np.arange(m)
    mu_w, sd_w = go.predict(pred, xs[idx], zs[idx])
    np.testing.assert_allclose(mu[idx], mu_w, atol=1e-10, rtol=0)
    np.testing.assert_allclose(sd[idx], sd_w, atol=1e-10, rtol=0)
    np.testing.assert_allclose(sc[idx], go.ucb(mu_w, sd_w, UCB), atol=1e-10, rtol=0)
  xs, _, zs, _ = _data(40, dc, dk, 7)
  mean, cov = dev.posterior(xs, zs, add_noise=True)
  mu_w, sd_w = go.predict(pred, xs, zs)
  np.testing.assert_allclose(mean.cpu().numpy(), mu_w, atol=1e-10, rtol=0)
  np.testing.assert_allclose(np.sqrt(np.diag(cov.cpu().numpy())), sd_w, atol=1e-8, rtol=0)


def test_ucb_pe_scoring():
  """GP-UCB-PE (the member loop of the multi-model launchers) with Dk = 40, both modes, against the oracle."""
  gp = _gp()
  x, y, z, po = _data(120, 3, 40, 11)
  xs, _, zs, _ = _data(5000, 3, 40, 12)
  a = gp.DeviceGP(0)
  b = gp.DeviceGP(0, stream=a.stream)
  try:
    po2 = go.GPParams(po.signal_variance, po.continuous_length_scale_squared, po.observation_noise_variance,
                      po.categorical_length_scale_squared)
    a.fit(x[:80], y[:80], _hyper(po), z=z[:80])
    b.fit(x, np.r_[y[:80], np.full(40, y[:80].mean())], _hyper(po2), z=z)
    pa = go.precompute_predictive(po, x[:80], y[:80], z[:80])
    pb = go.precompute_predictive(po2, x, np.r_[y[:80], np.full(40, y[:80].mean())], z)
    for mode in (0, 1):
      out = a.score_pe(b, xs, gp.UcbPeAcquisition(mode=mode, ucb_coefficient=UCB, use_trust_region=False), zs=zs)
      assert a.get_int('score_route') == ROUTE_GENERAL and b.get_int('score_route') == ROUTE_GENERAL
      want, aux = go.ucb_pe_score(pa, pb, xs[:400], zs[:400], mode=mode, ucb_coefficient=UCB, use_trust_region=False)
      np.testing.assert_allclose(out['score'].cpu().numpy()[:400], want, atol=1e-9, rtol=0)
      np.testing.assert_allclose(out['stddev_from_all'].cpu().numpy()[:400], aux['stddev_from_all'], atol=1e-10, rtol=0)
  finally:
    a.close(); b.close()


# ---------------------------------------------------------------------------------------------------------------
# D. duplication identity: Dk = 64 with every column repeated and doubled length scales is the Dk = 32 model
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [40, 300])
def test_duplication_identity(n):
  gp = _gp()
  x, y, z, po = _data(n, 3, 32, n)
  z2 = np.repeat(z, 2, axis=1)
  po2 = go.GPParams(po.signal_variance, po.continuous_length_scale_squared, po.observation_noise_variance,
                    np.repeat(2.0 * po.categorical_length_scale_squared, 2))
  narrow, wide = gp.DeviceGP(0), gp.DeviceGP(0)
  try:
    k1 = narrow.kernel_matrix(x, _hyper(po), z=z).cpu().numpy()
    k2 = wide.kernel_matrix(x, _hyper(po2), z=z2).cpu().numpy()
    np.testing.assert_allclose(k2, k1, rtol=1e-10, atol=0)
    l1, g1, _ = narrow.loss_and_grad(_cuda(x), _cuda(y), _hyper(po), z=_cuda(z, torch.int32))
    l2, g2, _ = wide.loss_and_grad(_cuda(x), _cuda(y), _hyper(po2), z=_cuda(z2, torch.int32))
    assert narrow.get_int('nll_route') == wide.get_int('nll_route')
    data1, data2 = l1 - go.regularizer(po), l2 - go.regularizer(po2)
    assert abs(data2 - data1) <= 1e-10 * abs(data1)
    dreg = lambda l: 0.02 * np.log(l / 0.5) / l   # noqa: E731  (tuned_gp_models.py regulariser derivative)
    l_k, l_k2 = po.categorical_length_scale_squared, po2.categorical_length_scale_squared
    d1 = g1[:32] - dreg(l_k)
    d2 = (g2[:64] - dreg(l_k2)).reshape(32, 2)
    # d data / d l' = (l / l')^2 d data / d l per copy, l' = 2 l
    np.testing.assert_allclose(d2[:, 0] * 4.0, d1, rtol=1e-10, atol=1e-12 * np.max(np.abs(d1)))
    np.testing.assert_allclose(d2[:, 1] * 4.0, d1, rtol=1e-10, atol=1e-12 * np.max(np.abs(d1)))
    np.testing.assert_allclose(g2[64:], g1[32:], rtol=1e-10, atol=1e-12)
    narrow.fit(x, y, _hyper(po), z=z)
    wide.fit(x, y, _hyper(po2), z=z2)
    xs, _, zs, _ = _data(3000, 3, 32, 5)
    acq = gp.Acquisition(UCB, False, 1.0)
    o1 = narrow.score(xs, acq, zs=zs, with_aux=True)
    o2 = wide.score(xs, acq, zs=np.repeat(zs, 2, axis=1), with_aux=True)
    narrow.synchronize(); wide.synchronize()
    assert wide.get_int('score_route') == ROUTE_GENERAL
    for key in ('mean', 'stddev', 'score'):
      v1, v2 = o1[key].cpu().numpy(), o2[key].cpu().numpy()
      np.testing.assert_allclose(v2, v1, rtol=1e-10, atol=1e-10 * np.max(np.abs(v1)))
  finally:
    narrow.close(); wide.close()


# ---------------------------------------------------------------------------------------------------------------
# E. Eagle: the stepped loop in lock step with the oracle, the fused runs on the replayed graph, random search
# ---------------------------------------------------------------------------------------------------------------
def _config(cfg_o, pool, batch, steps):
  from vizier_b200 import _lib
  return _lib.EagleConfig(cfg_o.visibility, cfg_o.gravity, cfg_o.negative_gravity, cfg_o.perturbation,
                          cfg_o.perturbation_lower_bound, cfg_o.penalize_factor, cfg_o.normalization_scale,
                          cfg_o.prior_trials_pool_pct, pool, batch, steps * batch, cfg_o.categorical_perturbation_factor,
                          cfg_o.pure_categorical_perturbation_factor, cfg_o.prob_same_category_without_perturbation,
                          cfg_o.mutate_normalization_type, 1)


def _sizes(dk):
  return tuple(int(s) for s in (2 + np.arange(dk) % 7) * (1 + (np.arange(dk) % 5 == 0) * 20))


@pytest.mark.parametrize('dk,dc,norm', [(40, 3, 0), (100, 0, 1), (100, 4, 0)])
def test_stepped_loop_in_lock_step(dk, dc, norm):
  gp = _gp()
  c = el.Case(f'wide-{dk}', 'quantised', dc, 20, 5, 30, 8, sizes=_sizes(dk), n_prior=12, norm=norm)
  x, _, z, po = _data(8, dc, dk, 3)
  d = gp.DeviceGP(0)
  try:
    d.fit(x, np.random.default_rng(4).normal(size=8), _hyper(po), z=z)
    se = gp.SteppedEagle(d, _config(c.cfg, c.pool, c.batch, c.steps), c.count, c.seed, n_prior=c.n_prior,
                         cat_sizes=c.sizes)
    assert d.get_int('eagle_route') == EAGLE_STEPPED
    state = {'t': -1}
    pc, pz = el.priors(c)

    def score(xc, xz):
      t = state['t']
      state['t'] = t + 1
      xc = np.asarray(xc, np.float64).reshape(xc.shape[0], dc)
      r = el.rewards(c, t, xc, np.asarray(xz, np.int32))
      if t < 0:
        se.seed(xc if dc else None, xz, r)
        return r
      xs, zs, rew = se.ask()
      with torch.cuda.stream(d.stream):
        if dc:
          np.testing.assert_allclose(xs.cpu().numpy(), xc, rtol=0, atol=1e-12)
        np.testing.assert_array_equal(zs.cpu().numpy(), xz)
        rew.copy_(torch.from_numpy(np.ascontiguousarray(r, np.float64)))
      se.tell()
      return r

    wc, wz, wr = xo.run_mixed(score, dim=dc, sizes=np.asarray(c.sizes, np.int64), prior_c=pc, prior_z=pz,
                              pool_size=c.pool, batch_size=c.batch, max_evaluations=c.steps * c.batch, count=c.count,
                              seed=c.seed, cfg=c.cfg, perturbation_type=xo.ADDITIVE)
    assert state['t'] == c.steps
    bc, bz, br = se.end()
    np.testing.assert_array_equal(br, wr)
    np.testing.assert_array_equal(bz, wz)
    if dc:
      np.testing.assert_allclose(bc, wc, rtol=0, atol=1e-12)
  finally:
    d.close()


@pytest.mark.parametrize('dk,dc', [(40, 3), (100, 0)])
def test_eagle_run_on_graph_against_oracle(dk, dc):
  gp = _gp()
  sizes = _sizes(dk)
  x, y, z, po = _data(150, dc, dk, 17, sizes=2)
  pred = go.precompute_predictive(po, x, y, z)
  prior_c, prior_z = x[:10], z[:10]

  def score(xc, xz):
    mu, sd = go.predict(pred, xc, xz)
    return mu + UCB * sd

  cfg_o = eo.EagleConfig(perturbation_lower_bound=0.05)
  wc, wz, wr = xo.run_mixed(score, dim=dc, sizes=np.asarray(sizes, np.int64), pool_size=50, batch_size=25,
                            max_evaluations=8 * 25, count=6, seed=5, cfg=cfg_o, perturbation_type=xo.ADDITIVE,
                            prior_c=prior_c, prior_z=prior_z)
  d = gp.DeviceGP(0)
  try:
    d.fit(x, y, _hyper(po), z=z)
    bc, bz, br = d.eagle_run(_config(cfg_o, 50, 25, 8), gp.Acquisition(UCB, False, 1.0), 6, 5, prior=prior_c,
                             prior_z=prior_z, cat_sizes=sizes)
    assert d.get_int('eagle_route') == EAGLE_GRAPH
    np.testing.assert_allclose(br, wr, rtol=0, atol=1e-9)
    np.testing.assert_array_equal(bz, wz)
    if dc:
      np.testing.assert_allclose(bc, wc, rtol=0, atol=1e-9)
  finally:
    d.close()


def test_random_search():
  gp = _gp()
  dk, dc, m = 100, 2, 6000
  sizes = _sizes(dk)
  x, y, z, po = _data(40, dc, dk, 8)
  pred = go.precompute_predictive(po, x, y, z)
  d = gp.DeviceGP(0)
  try:
    d.fit(x, y, _hyper(po), z=z)
    bx, bz, bs, bi = d.random_search(m, gp.Acquisition(UCB, False, 1.0), 8, 21, cat_sizes=sizes)
    assert d.get_int('score_route') == ROUTE_GENERAL
  finally:
    d.close()
  xs = eo.philox_uniform(21, eo.STREAM_RANDOM_POOL, 0, m * dc).reshape(m, dc)
  zs = eo.uniform_categories(eo.philox_uniform(21, eo.STREAM_RANDOM_POOL_CAT, 0, m * dk).reshape(m, -1),
                             np.asarray(sizes))
  np.testing.assert_array_equal(bz, zs[bi])
  np.testing.assert_array_equal(bx, xs[bi])
  mu, sd = go.predict(pred, xs, zs)
  want = mu + UCB * sd
  np.testing.assert_allclose(bs, want[bi], rtol=0, atol=1e-9)
  np.testing.assert_array_equal(np.sort(bi), np.sort(np.argsort(-want, kind='stable')[:8]))


# ---------------------------------------------------------------------------------------------------------------
# F. designers
# ---------------------------------------------------------------------------------------------------------------
def _problem(n_cat, n_float, n_metrics):
  from vizier_b200 import vz
  p = vz.ProblemStatement()
  for i in range(n_float):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  for i in range(n_cat):
    p.search_space.root.add_categorical_param(f'c{i}', [f'v{j}' for j in range(2 + i % 4)])
  for k in range(n_metrics):
    p.metric_information.append(vz.MetricInformation(name=f'm{k}', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  return p


def _value(params, name):
  v = params[name]
  return getattr(v, 'value', v)


def _label(params, n_cat, n_float, k):
  v = -sum((float(_value(params, f'x{i}')) - 0.3) ** 2 for i in range(n_float))
  v -= 0.05 * sum(_value(params, f'c{i}') != 'v1' for i in range(n_cat))
  return float(v if k == 0 else 0.5 * v - 0.1 * (_value(params, 'c0') == 'v0'))


DESIGNERS = [('default', {}, 1), ('ensemble', dict(ensemble_size=3), 1), ('two-metrics', {}, 2),
             ('separable', dict(multitask_type='SEPARABLE_NORMAL_TASK_KERNEL_PRIOR'), 2), ('priors', {}, 1),
             ('ucb-pe', {}, 1), ('ucb-pe-two-metrics', {}, 2)]


@pytest.mark.parametrize('n_cat,n_float', [(40, 3), (100, 0)])
@pytest.mark.parametrize('name,kw,n_metrics', DESIGNERS, ids=[d[0] for d in DESIGNERS])
def test_designers(name, kw, n_metrics, n_cat, n_float):
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit, gp_ucb_pe
  p = _problem(n_cat, n_float, n_metrics)
  if name.startswith('ucb-pe'):
    d = gp_ucb_pe.VizierGPUCBPEBandit(p, rng=2)
  else:
    d = gp_bandit.VizierGPBandit(p, rng=2, **kw)
  rng = np.random.default_rng(0)

  def complete(params_list, tid0):
    done = []
    for i, params in enumerate(params_list):
      t = vz.Trial(id=tid0 + i, parameters=params)
      t.complete(vz.Measurement({f'm{k}': _label(t.parameters, n_cat, n_float, k) for k in range(n_metrics)}))
      done.append(t)
    return done

  def random_params():
    out = {f'x{i}': float(rng.uniform()) for i in range(n_float)}
    out.update({f'c{i}': f'v{rng.integers(0, 2 + i % 4)}' for i in range(n_cat)})
    return out

  if name == 'priors':
    d.set_priors([vz.CompletedTrials(complete([random_params() for _ in range(20)], 1000))])
  trials = complete([random_params() for _ in range(12)], 1)
  d.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  tid = 13
  for _ in range(2):
    sugg = d.suggest(2)
    assert len(sugg) == 2
    new = []
    for s in sugg:
      assert p.search_space.contains(s.parameters)
      t = s.to_trial(tid); tid += 1
      t.complete(vz.Measurement({f'm{k}': _label(t.parameters, n_cat, n_float, k) for k in range(n_metrics)}))
      new.append(t)
    trials += new
    d.update(vz.CompletedTrials(new), vz.ActiveTrials())
  pred = d.predict(trials, num_samples=200)
  mean = np.asarray(pred.mean).reshape(len(trials), -1)
  assert np.isfinite(mean).all() and np.isfinite(np.asarray(pred.stddev)).all()
  labels = np.array([[_label(t.parameters, n_cat, n_float, k) for k in range(n_metrics)] for t in trials])
  for k in range(n_metrics):
    assert np.corrcoef(mean[:, k], labels[:, k])[0, 1] > 0.9, (name, k)
  samples = d.sample(trials[:3], num_samples=50)
  assert np.isfinite(np.asarray(samples)).all()
