"""Transfer learning with the designer's model spec on every level (gp_bandit.py:402-447): stacks of uniform ensembles,
linear-kernel levels and multi-metric levels through vzgp_score_stack_ensemble / vzgp_score_stack_multi and their
Eagle loops, against the tests-side oracle (stack_oracle.py); the reference's StackedResidualGPTest matrix
(gp/gp_models_test.py:148-350); and VizierGPBandit.set_priors end to end with ensemble_size = 3, linear_coef = 0.4
and two metrics (gp_bandit_test.py:597-621)."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from oracle import eagle_oracle as eo  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402
import stack_oracle as so  # noqa: E402

SMALL, SPLIT, CLUSTER, GENERAL = 0, 1, 2, 4   # vzgp_score_route
GRAPH = 2                                     # vzgp_eagle_route


def _params(l, k, d, dk, linear, high_noise=False):
  """Member k of level l as an (oracle, device) pair of hyper-parameters."""
  from vizier_b200 import gp
  sf2, sn2 = 0.8 + 0.3 * l + 0.2 * k, (1e-10 if high_noise else 1e-3 * (l + 1) * (1 + k))
  ls2 = (0.3 + 0.2 * l) * (1 + np.arange(d) / d) * (1 + 0.25 * k)
  lk = np.linspace(0.7, 1.2, dk) * (1 + 0.1 * k) if dk else None
  if linear:
    lp = (0.4, 0.6 + 0.1 * k, 0.2 - 0.1 * l, 0.1 * k)
    return (go.GPParams(sf2, ls2, sn2, lk, go.LinearParams(*lp)),
            gp.GPHyperParams(sf2, ls2, sn2, lk, linear_coef=lp[0], linear_slope_amplitude=lp[1], linear_shift=lp[2],
                             mean_constant=lp[3]))
  return go.GPParams(sf2, ls2, sn2, lk), gp.GPHyperParams(sf2, ls2, sn2, lk)


def _members(level):
  return level.members if hasattr(level, 'members') else [level]


def _build(sizes, d, e, seed, dk=0, linear=False, n_metrics=1, high_noise_top=False):
  """A stack with fixed hyper-parameters per member on both sides; checks every level's residual labels against the
  oracle.  Returns (StackedGP, oracle levels, rng, top x, top z)."""
  from vizier_b200 import gp
  rng = np.random.default_rng(seed)
  stack = gp.StackedGP(0)
  levels = []
  for l, n in enumerate(sizes):
    x = rng.uniform(size=(n, d))
    z = rng.integers(0, 3, size=(n, dk)).astype(np.int32) if dk else None
    y = -np.sum((x - 0.3 - 0.05 * l) ** 2, axis=1) + 0.03 * rng.normal(size=n) - (0.2 * (z[:, 0] == 1) if dk else 0.0)
    if n_metrics > 1:
      y = np.stack([y * (1 + 0.5 * m) + 0.2 * m * np.sin(3 * x[:, 0]) for m in range(n_metrics)], axis=1)
    resid_o = so.residual_labels(levels, x, y, z)
    resid_d = y - stack.mean(x, z) if stack.levels else y
    np.testing.assert_allclose(resid_d, resid_o, rtol=0, atol=1e-9)
    ps = [_params(l, k, d, dk, linear, high_noise_top and l == len(sizes) - 1) for k in range(e)]
    levels.append([go.precompute_predictive(po, x, resid_o, z) for po, _ in ps])
    level = stack.new_level(e)
    for h in _members(level):
      h.set_int('score_i8', 0)
      h.set_int('small_tiles', -1)
    level.fit(x, resid_d, [pg for _, pg in ps] if e > 1 else ps[0][1], z=z)
    stack.push(level, n)
  return stack, levels, rng, x, z


def _route(sm, m, n):
  tiles = -(-m // 64)
  if tiles <= 8:
    return SMALL
  nblocks = -(-(-(-n // 64) * 64) // 128)
  nsplit = (nblocks + 1) // 2 if (2 * tiles <= sm and nblocks >= 2) else 1
  return SPLIT if nsplit > 1 else CLUSTER


def _close(got, want, rel=1e-9):
  want = np.asarray(want, np.float64)
  err = np.abs(np.asarray(got) - want)
  tol = rel * np.maximum(1.0, np.abs(want))
  assert np.all(err <= tol), (float(np.max(err / tol)), np.unravel_index(np.argmax(err / tol), err.shape))


# route of the top level, level sizes, d, dk, E, candidates (a callable of the SM count), linear kernel
CASES = [
    pytest.param(SMALL, (60, 30), 3, 0, 2, lambda sm: 300, False, id='small-l2-e2'),
    pytest.param(SMALL, (50, 30, 20), 3, 2, 3, lambda sm: 400, False, id='small-l3-e3-cat'),
    pytest.param(SPLIT, (400, 280), 4, 0, 3, lambda sm: 20 * 64 - 11, False, id='split-l2-e3'),
    pytest.param(SPLIT, (260, 140, 300), 4, 1, 2, lambda sm: 24 * 64 + 5, False, id='split-l3-e2-cat'),
    pytest.param(CLUSTER, (150, 100, 60), 5, 2, 5, lambda sm: (sm // 2 + 1) * 64 + 9, False, id='cluster-l3-e5-cat'),
    pytest.param(CLUSTER, (120, 70), 4, 0, 5, lambda sm: (sm // 2 + 3) * 64, False, id='cluster-l2-e5'),
    pytest.param(GENERAL, (60, 30), 3, 0, 3, lambda sm: 500, True, id='general-l2-e3-linear'),
    pytest.param(GENERAL, (70, 40, 25), 3, 0, 1, lambda sm: 700, True, id='general-l3-e1-linear'),
]


@pytest.mark.parametrize('route,sizes,d,dk,e,count,linear', CASES)
def test_stack_ensemble_score_matches_oracle(route, sizes, d, dk, e, count, linear):
  from vizier_b200 import gp
  stack, levels, rng, x_top, z_top = _build(sizes, d, e, 11 + e + len(sizes), dk, linear)
  try:
    sm = stack._lead().get_int('sm_count')
    mc = count(sm)
    xs = rng.uniform(-0.5, 1.5, size=(mc, d))
    xs[:5] = x_top[:5]
    zs = rng.integers(0, 3, size=(mc, dk)).astype(np.int32) if dk else None
    if dk:
      zs[:5] = z_top[:5]
    for l in range(1, len(sizes)):
      np.testing.assert_allclose(stack.alphas[l], so.level_alpha(levels, l), rtol=1e-14)
    seen_tr = False
    for use_tr, radius in ((False, 1.0), (True, 0.25), (True, 0.8)):
      acq = gp.Acquisition(1.8, use_tr, radius)
      out = stack.score(xs, acq, zs=zs, with_aux=True)
      stack.synchronize()
      for l, level in enumerate(stack.levels):
        for h in _members(level):
          assert h.get_int('score_route') == (GENERAL if linear else _route(sm, mc, sizes[l]))
      assert (GENERAL if linear else _route(sm, mc, sizes[-1])) == route
      want, mean, sd, dist = so.score(levels, xs, zs, coefficient=1.8, trust_radius_value=radius if use_tr else None)
      _close(out['mean'].cpu().numpy(), mean)
      _close(out['stddev'].cpu().numpy(), sd)
      _close(out['score'].cpu().numpy(), want)
      dist = go.min_linf_distance(xs, x_top, np.ones(d, bool))
      np.testing.assert_array_equal(out['linf_distance'].cpu().numpy(), dist)
      if use_tr and radius <= 0.5:
        assert np.any(want < -1e3) and np.any(want > -1e3)
        seen_tr = True
    assert seen_tr
  finally:
    stack.close()


@pytest.mark.parametrize('e,linear', [(3, False), (4, True)])
def test_mixture_of_the_device_member_moments_at_full_precision(e, linear):
  """The top level in high-noise mode (noise 1e-10): at its trials each member's stddev is ~1e-5 while |mean| ~ 1,
  where a one-pass mixture variance loses about six digits.  The combined stddev must be the two-pass mixture and stack
  of the device's own member moments to 1e-12."""
  from vizier_b200 import gp
  stack, levels, rng, x_top, _ = _build((80, 40), 3, e, 5, linear=linear, high_noise_top=True)
  try:
    xs = np.concatenate([x_top[:20], rng.uniform(size=(200, 3))])
    acq0 = gp.Acquisition(0.0, False, 1.0)
    out = stack.score(xs, acq0, with_aux=True)
    stack.synchronize()
    lead = stack._lead()
    mus, sds = [], []
    for level in stack.levels:
      lm, ls = [], []
      for h in _members(level):
        o = {k: torch.empty(len(xs), dtype=torch.float64, device=h.device) for k in ('score', 'mean', 'stddev')}
        if h is lead:
          o['linf_distance'] = torch.empty(len(xs), dtype=torch.float64, device=h.device)
        torch.cuda.synchronize()
        h.score(xs, acq0, out=o)
        h.synchronize()
        lm.append(o['mean'].cpu().numpy()); ls.append(o['stddev'].cpu().numpy())
      mus.append(np.stack(lm)); sds.append(np.stack(ls))
    mean, sd = so.mixture(mus[0], sds[0])
    for l in range(1, len(mus)):
      a = stack.alphas[l]
      mean_l, sd_l = so.mixture(mus[l], sds[l])
      mean, sd = mean + mean_l, sd_l ** a * sd ** (1.0 - a)
    got = out['stddev'].cpu().numpy()
    assert np.min(np.stack(sds[-1])[:, :20]) < 1e-3
    assert np.max(np.abs(got - sd) / sd) < 1e-12
    np.testing.assert_allclose(out['mean'].cpu().numpy(), mean, rtol=1e-14, atol=1e-15)
  finally:
    stack.close()


@pytest.mark.parametrize('m', [300, 20000])
def test_single_member_entry_is_bit_identical_to_score_stack(m):
  from vizier_b200 import _lib, gp
  stack, _, rng, _, _ = _build((120, 60), 4, 1, 2, dk=1)
  try:
    xs = torch.from_numpy(rng.uniform(size=(m, 4))).cuda()
    zs = torch.from_numpy(rng.integers(0, 3, size=(m, 1)).astype(np.int32)).cuda()
    acq = gp.Acquisition(1.8, True, 0.3)
    want = stack.score(xs, acq, zs=zs, with_aux=True)
    got = {k: torch.empty(m, dtype=torch.float64, device=xs.device) for k in ('score', 'mean', 'stddev', 'linf')}
    a, keep = acq._c()
    torch.cuda.synchronize()
    lib = stack._lib
    _lib.check('vzgp_score_stack_ensemble', lib.vzgp_score_stack_ensemble(
        stack._handles(), 2, 1, stack._alphas(), C.c_void_p(xs.data_ptr()), C.c_void_p(zs.data_ptr()), m, C.byref(a),
        *[C.c_void_p(got[k].data_ptr()) for k in ('score', 'mean', 'stddev', 'linf')]))
    stack.synchronize()
    for k, w in (('score', 'score'), ('mean', 'mean'), ('stddev', 'stddev'), ('linf', 'linf_distance')):
      assert torch.equal(got[k], want[w]), k
    del keep
  finally:
    stack.close()


def test_entry_point_checks():
  from vizier_b200 import _lib, gp
  stack, _, rng, x, _ = _build((40, 20), 2, 2, 3)
  try:
    lib, hs, al = stack._lib, stack._handles(), stack._alphas()
    acq, _keep = gp.Acquisition(1.8, False, 1.0)._c()
    out = torch.empty(4, dtype=torch.float64, device='cuda')
    xs = torch.zeros((4, 2), dtype=torch.float64, device='cuda')
    args = (C.c_void_p(xs.data_ptr()), None, 4, C.byref(acq), C.c_void_p(out.data_ptr()), None, None, None)
    for L, E in ((0, 2), (17, 2), (2, 0), (2, 9), (1, 3)):
      st = lib.vzgp_score_stack_ensemble(hs, L, E, al, *args)
      assert st == _lib.VZGP_ERR_ARG, (L, E)                 # (1, 3): members of one level on different trials
    bad = (C.c_double * 2)(0.0, 1.5)
    assert lib.vzgp_score_stack_ensemble(hs, 2, 2, bad, *args) == _lib.VZGP_ERR_ARG
    lone = gp.EnsembleGP(0, 2, stream=stack.stream)          # never fitted
    hs2 = (C.c_void_p * 4)(*[m._h for m in stack.levels[0].members + lone.members])
    assert lib.vzgp_score_stack_ensemble(hs2, 2, 2, al, *args) == _lib.VZGP_ERR_STATE
    # the multi-metric entry refuses single-metric levels
    sc, _k2 = gp.ScalarizedUcbAcquisition(np.ones((1, 2)) / np.sqrt(2), np.zeros(2))._c()
    single = (C.c_void_p * 2)(*[stack.levels[0].members[0]._h, stack.levels[1].members[0]._h])
    assert lib.vzgp_score_stack_multi(single, 2, al, C.c_void_p(xs.data_ptr()), None, 4, C.byref(sc),
                                      C.c_void_p(out.data_ptr()), None, None) == _lib.VZGP_ERR_ARG
    lone.close()
  finally:
    stack.close()


def _scalarization(rng, levels, n_metrics, s=24):
  from vizier_b200 import gp
  w = np.abs(rng.normal(size=(s, n_metrics)))
  w /= np.linalg.norm(w, axis=1, keepdims=True)
  labels = levels[0][0].chol @ (levels[0][0].chol.T @ levels[0][0].alpha)
  ref = go.hv_reference_point(labels, 0.01)
  best = go.hv_max_scalarized(labels, w, ref)
  return gp.ScalarizedUcbAcquisition(w, ref, best, 1.8)


@pytest.mark.parametrize('sizes,d,dk,n_metrics,count', [
    ((60, 30), 3, 0, 2, lambda sm: 300), ((90, 50, 30), 4, 1, 3, lambda sm: 500),
    ((200, 130), 4, 0, 2, lambda sm: 20 * 64 - 11), ((150, 80, 40), 3, 2, 3, lambda sm: (sm // 2 + 1) * 64 + 9)])
def test_stack_multi_score_matches_oracle(sizes, d, dk, n_metrics, count):
  stack, levels, rng, _, _ = _build(sizes, d, 1, 31 + n_metrics, dk, n_metrics=n_metrics)
  try:
    assert stack.n_metrics == n_metrics
    mc = count(stack._lead().get_int('sm_count'))
    xs = rng.uniform(size=(mc, d))
    zs = rng.integers(0, 3, size=(mc, dk)).astype(np.int32) if dk else None
    sc = _scalarization(rng, levels, n_metrics)
    out = stack.score_multi(xs, sc, zs=zs, with_aux=True)
    stack.synchronize()
    want, mean, sd = so.scalarized_score(levels, xs, sc.weights, sc.reference_point, sc.max_scalarized, 1.8, zs=zs)
    _close(out['mean'].cpu().numpy(), mean.T)
    _close(out['stddev'].cpu().numpy(), sd)
    _close(out['score'].cpu().numpy(), want)
    assert np.ptp(want) > 0
    m2, s2 = stack.predict(xs, zs)
    _close(m2, mean)
    _close(s2, sd)
  finally:
    stack.close()


def _eagle_cfgs(pool, batch, steps):
  from vizier_b200 import _lib
  cfg_o = eo.EagleConfig()
  cfg = _lib.EagleConfig(cfg_o.visibility, cfg_o.gravity, cfg_o.negative_gravity, cfg_o.perturbation,
                         cfg_o.perturbation_lower_bound, cfg_o.penalize_factor, cfg_o.normalization_scale,
                         cfg_o.prior_trials_pool_pct, pool, batch, steps * batch)
  return cfg_o, cfg


@pytest.mark.parametrize('e,linear', [(3, False), (2, True)])
def test_stack_ensemble_eagle_and_random_search_match_oracle(e, linear):
  from vizier_b200 import gp
  d, pool, batch, steps = 4, 50, 25, 8
  stack, levels, _, x_top, _ = _build((90, 35), d, e, 23, linear=linear)
  try:
    radius = go.trust_radius(35, d, 0)

    def score_fn(q):
      return so.score(levels, q, coefficient=1.8, trust_radius_value=radius)[0]

    cfg_o, cfg = _eagle_cfgs(pool, batch, steps)
    wx, wr, _ = eo.run_eagle_optimizer(score_fn, dim=d, pool_size=pool, batch_size=batch, max_evaluations=steps * batch,
                                       count=2, seed=5, cfg=cfg_o, prior_features=x_top)
    acq = gp.Acquisition(1.8, True, radius)
    bx, _, br = stack.eagle_run(cfg, acq, count=2, seed=5, prior=x_top)
    assert stack._lead().get_int('eagle_route') == GRAPH
    np.testing.assert_allclose(br, wr, atol=1e-9)
    np.testing.assert_allclose(bx, wx, atol=1e-9)
    rx, _, rs, _ = stack.random_search(3000, acq, 2, seed=9)
    wrx, wrs, _ = eo.run_random_optimizer(score_fn, dim=d, num_candidates=3000, count=2, seed=9)
    np.testing.assert_allclose(rs, wrs, atol=1e-9)
    np.testing.assert_allclose(rx, wrx, atol=0)
  finally:
    stack.close()


def test_stack_multi_eagle_matches_oracle():
  d, pool, batch, steps = 3, 50, 25, 8
  stack, levels, rng, x_top, _ = _build((80, 30), d, 1, 41, n_metrics=2)
  try:
    sc = _scalarization(rng, levels, 2)

    def score_fn(q):
      return so.scalarized_score(levels, q, sc.weights, sc.reference_point, sc.max_scalarized, 1.8)[0]

    cfg_o, cfg = _eagle_cfgs(pool, batch, steps)
    wx, wr, _ = eo.run_eagle_optimizer(score_fn, dim=d, pool_size=pool, batch_size=batch, max_evaluations=steps * batch,
                                       count=2, seed=7, cfg=cfg_o, prior_features=x_top)
    bx, _, br = stack.eagle_run(cfg, sc, count=2, seed=7, prior=x_top)
    assert stack._lead().get_int('eagle_route') == GRAPH
    np.testing.assert_allclose(br, wr, atol=1e-9 * max(1.0, np.max(np.abs(wr))))
    np.testing.assert_allclose(bx, wx, atol=1e-9)
  finally:
    stack.close()


def test_stepped_loop_with_zero_prior_equals_device_loop():
  """VectorizedOptimizer with a zero prior_acquisition (host-stepped loop on the lead handle, the stack scoring every
  batch) finds what the device loop finds."""
  from vizier_b200 import gp
  from vizier_b200 import optimizers as vb
  d, dk = 3, 1
  stack, _, _, x_top, z_top = _build((70, 30), d, 3, 51, dk=dk)
  try:
    opt = vb.VectorizedOptimizer(vb.VectorizedEagleStrategyFactory(), d, dk, 25, 1000, (3,))
    calls = []

    def zero(xc, xz):
      calls.append(xc.shape[0])
      return np.zeros(xc.shape[0])

    acq = gp.Acquisition(1.8, True, 0.3)
    dev = opt(stack, acq, count=2, prior_features=x_top, prior_categorical=z_top, seed=5)
    host = opt(stack, acq, count=2, prior_features=x_top, prior_categorical=z_top, seed=5, prior_acquisition=zero)
    assert stack._lead().get_int('eagle_route') == 3
    np.testing.assert_allclose(host.rewards, dev.rewards, rtol=0, atol=1e-12)
    np.testing.assert_allclose(host.features, dev.features, rtol=0, atol=1e-12)
    np.testing.assert_array_equal(host.categorical, dev.categorical)
    assert calls
  finally:
    stack.close()


# ---- the reference's StackedResidualGPTest (gp/gp_models_test.py:148-350) ------------------------------------------
def _lambda_data(f, n, offset=0):
  """_setup_lambda_search's data: quasi-random points of [-5, 5) (a base-2 van der Corput sequence here), raw labels,
  features scaled to [0, 1] as the converter does."""
  def vdc(i):
    r, denom = 0.0, 1.0
    while i:
      denom *= 2
      i, rem = divmod(i, 2)
      r += rem / denom
    return r
  u = np.array([vdc(i + 1 + offset) for i in range(n)])
  return u[:, None], np.array([f(-5.0 + 10.0 * v) for v in u])


def _train(datasets, linear_coef, e, seed=0):
  """train_gp([specs], [data]) (gp_models.py:302-347): one level per dataset, each trained with ARD on its residuals
  against the levels below; a single dataset is the plain model."""
  from vizier_b200 import ard, gp
  stack = gp.StackedGP(0)
  for x, y in datasets:
    resid = y - stack.mean(x) if stack.levels else y
    level = stack.new_level(e)
    ard_dev = level.members[0] if e > 1 else level
    best, _ = ard.train_gp(ard_dev, x, resid, None, rng=np.random.default_rng(seed),
                           random_restarts=max(ard.DEFAULT_RANDOM_RESTARTS, e), ensemble_size=e,
                           linear_coef=linear_coef or None)
    level.fit(x, resid, list(best) if e > 1 else best[0])
    stack.push(level, x.shape[0])
  return stack


def _mse(stack, data):
  """_compute_mse: the SUM of squared errors of the predictive mean."""
  x, y = data
  out = float(np.sum((stack.mean(x) - y) ** 2))
  stack.close()
  return out


MATRIX = [(0.0, 1), (0.4, 1), (0.0, 5), (0.4, 5)]


@pytest.mark.parametrize('linear_coef,e', MATRIX)
def test_sequential_base_accuracy(linear_coef, e):
  f = lambda x: -((x - 0.5) ** 2)  # noqa: E731
  base, top, test = _lambda_data(f, 100), _lambda_data(f, 5), _lambda_data(f, 100, offset=5)
  seq = _mse(_train([base, top], linear_coef, e), test)
  alone = _mse(_train([top], linear_coef, e), test)
  assert seq < alone, (seq, alone)


@pytest.mark.parametrize('linear_coef,e', MATRIX[:3])   # (0.4, 5) is commented out upstream as flaky
def test_multi_base(linear_coef, e):
  f = lambda x: -((x - 0.5) ** 2)  # noqa: E731
  top, base, test = _lambda_data(f, 5), _lambda_data(f, 100), _lambda_data(f, 100, offset=100)
  seq = _mse(_train([base, base, top], linear_coef, e), test)
  good = _mse(_train([base], linear_coef, e), test)
  assert round(seq - good, 4) == 0, (seq, good)
  assert good < 2e-2, good


@pytest.mark.parametrize('linear_coef,e', MATRIX)
def test_bad_base_resilience(linear_coef, e):
  f = lambda x: -((x - 0.5) ** 2)  # noqa: E731
  fake = lambda x: x ** 5  # noqa: E731
  bad, top, test = _lambda_data(fake, 100), _lambda_data(f, 100), _lambda_data(f, 100, offset=100)
  seq = _mse(_train([bad, top], linear_coef, e), test)
  fake_only = _mse(_train([_lambda_data(fake, 100)], linear_coef, e), test)
  assert seq < fake_only, (seq, fake_only)


# ---- the designer end to end (gp_bandit_test.py:597-621, test_run_with_priors) -------------------------------------
def _designer(n_metrics, **kw):
  from vizier_b200 import vz
  from vizier_b200 import optimizers as vb
  from vizier_b200.designers import gp_bandit
  p = vz.ProblemStatement()
  p.search_space.root.add_float_param('x0', -5.0, 5.0)
  p.search_space.root.add_float_param('x1', 0.0, 1.0)
  for m in range(n_metrics):
    p.metric_information.append(vz.MetricInformation(name=f'obj{m}', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  fac = vb.VectorizedOptimizerFactory(strategy_factory=vb.VectorizedEagleStrategyFactory(), max_evaluations=1000,
                                      suggestion_batch_size=25)
  return gp_bandit.VizierGPBandit(p, acquisition_optimizer_factory=fac, rng=1, **kw)


def _trials(n, n_metrics, seed, start=1):
  from vizier_b200 import vz
  rng = np.random.default_rng(seed)
  out = []
  for i in range(n):
    x0, x1 = rng.uniform(-5.0, 5.0), rng.uniform()
    t = vz.Trial(parameters={'x0': float(x0), 'x1': float(x1)}, id=start + i)
    v = -((x0 / 5.0 - 0.5) ** 2) - 0.3 * (x1 - 0.4) ** 2
    t.complete(vz.Measurement({f'obj{m}': float(v * (1 + m) + 0.1 * m * x1) for m in range(n_metrics)}))
    out.append(t)
  return out


@pytest.mark.parametrize('kw,n_metrics', [({'ensemble_size': 3}, 1), ({'linear_coef': 0.4}, 1),
                                          ({'ensemble_size': 3, 'linear_coef': 0.4}, 1), ({}, 2)],
                         ids=['e3', 'linear', 'e3-linear', 'two-metrics'])
def test_run_with_priors(kw, n_metrics):
  from vizier_b200 import vz
  des = _designer(n_metrics, **kw)
  des.set_priors([vz.CompletedTrials(_trials(60, n_metrics, 3)), vz.CompletedTrials(_trials(30, n_metrics, 4, 100))])
  assert len(des._stack.levels) == 2
  rng = np.random.default_rng(1)
  tid = 1000
  for batch in (3, 1, 2):
    sugg = des.suggest(batch)
    assert len(sugg) == batch
    done = []
    for s in sugg:
      assert -5.0 <= s.parameters['x0'].value <= 5.0 and 0.0 <= s.parameters['x1'].value <= 1.0
      tid += 1
      t = s.to_trial(tid)
      t.complete(vz.Measurement({f'obj{m}': float(rng.uniform(-1.0, 1.0)) for m in range(n_metrics)}))
      done.append(t)
    des.update(vz.CompletedTrials(done), vz.ActiveTrials())
  stack = des._stack
  assert len(stack.levels) == 3 and (stack.ensemble_size, stack.n_metrics) == (kw.get('ensemble_size', 1), n_metrics)
  test = [vz.Trial(parameters={'x0': float(a), 'x1': float(b)}) for a, b in zip(np.linspace(-4, 4, 7), np.linspace(0, 1, 7))]
  pred = des.predict(test, rng=3, num_samples=200)
  s = des.sample(test, rng=3, num_samples=50)
  assert s.shape == ((50, 7) if n_metrics == 1 else (50, 7, n_metrics))
  assert np.all(np.isfinite(pred.mean)) and np.all(np.isfinite(pred.stddev)) and np.all(pred.stddev > 0)
  assert np.asarray(pred.mean).shape == ((7,) if n_metrics == 1 else (7, n_metrics))
