"""MaxValueEntropySearch on the device against tests/mes_oracle.py: the max-value fit (vzgp_mes_fit), the MES value
on every scoring route, in every acquisition optimiser and in vzgp_score_grad, the state rules of the handle, and the
designer.

Stage-wise parity: the device's samples are held to the oracle's fit of the device's own trial moments (1e-12 b
max(1, N/100), b the Gumbel scale), and its scores to the oracle's MES of the device's own (mu, sd) (1e-12 relative); against the oracle's
own moments the bound is 1e-10 (1 + |dMES/dmu| + |dMES/dsd|), the moments' 1e-10 carried through the MES slopes."""
import ctypes as C
import json

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

import lbfgsb_oracle as lo  # noqa: E402
import mes_oracle as mo  # noqa: E402
from oracle import eagle_oracle as eo  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402

TOL = 1e-10
SMALL, SPLIT, CLUSTER, I8, GENERAL = 0, 1, 2, 3, 4


def _mods():
  from vizier_b200 import _lib, acquisitions, gp
  return _lib, acquisitions, gp


def _model(n, dc, linear=False, seed=0, noise=1e-3):
  _, _, gp = _mods()
  rng = np.random.default_rng(seed)
  x, y, params = lo.make_model(rng, n, dc, linear=linear, noise=noise)
  pred = lo.predictive(x, y, params)
  dev = gp.DeviceGP(0)
  dev.fit(x, y, lo.device_params(params))
  return x, y, pred, dev


def _device_trial_moments(dev, x):
  _, _, gp = _mods()
  out = dev.score(x, gp.Acquisition(0.0, False, 1.0), with_aux=True)
  dev.synchronize()
  return out['mean'].cpu().numpy(), out['stddev'].cpu().numpy()


# left: the label the fit starts from.  'median' keeps P(left) small (the Gumbel branch); 'max' is what the designer
# passes, and with small noise the posterior at the trials sits below the best label, so P(left) >= 0.25 (the
# authors' degenerate branch); with large noise the trials' spread takes it back to the Gumbel branch.
FIT_CASES = [(5, 3, False, 1e-3, 'median', False), (64, 4, False, 1e-3, 'median', False),
             (65, 4, False, 1e-3, 'median', False), (1000, 8, False, 1e-3, 'median', False),
             (64, 4, True, 1e-3, 'median', False), (300, 6, True, 1e-3, 'median', False),
             (65, 4, False, 1e-3, 'max', True), (50, 3, False, 4.0, 'max', False)]


@pytest.mark.parametrize('n,dc,linear,noise,left,degenerate', FIT_CASES,
                         ids=[f'N{n}-D{d}{"-linear" if lin else ""}-{lf}-noise{s:g}' for n, d, lin, s, lf, _ in FIT_CASES])
def test_mes_fit_against_oracle(n, dc, linear, noise, left, degenerate):
  x, y, pred, dev = _model(n, dc, linear, seed=n, noise=noise)
  best = float(np.max(y) if left == 'max' else np.median(y))
  got = dev.mes_fit(best, 100, 123).cpu().numpy()
  mu_d, sd_d = _device_trial_moments(dev, x)
  want = mo.fit(mu_d, sd_d, best, noise, 100, 123)
  want_own = mo.fit_predictive(pred, best)
  assert want['degenerate'] == want_own['degenerate'] == degenerate
  if want['degenerate']:
    np.testing.assert_array_equal(got, np.full(100, best + 5.0 * np.sqrt(noise)))
  else:
    b = want['b']
    assert b > 0
    # log P sums N terms, each within a few ulps between the device's erfcx / log1p and SciPy's: the quartiles move by
    # O(N eps) of the Gumbel scale
    np.testing.assert_allclose(got, want['samples'], rtol=0, atol=1e-12 * b * max(1.0, n / 100))
    np.testing.assert_allclose(got, want_own['samples'], rtol=0, atol=1e-9 * b)
    assert np.all(got >= want['floor'])
  dev.close()


def _tiles(dev, route):
  sm = dev.get_int('sm_count')
  return {'small': 4, 'split': min(9, sm // 2), 'cluster': sm // 2 + 1, 'i8': sm + 1, 'general': 3}[route]


def _check_scores(out, ys, pred, xs, tr, radius, mu, sd):
  """Device outputs against the oracle on the device's own moments and on the oracle's."""
  got = {k: out[k].cpu().numpy() for k in ('score', 'mean', 'stddev', 'linf_distance') if k in out}
  np.testing.assert_allclose(got['mean'], mu, rtol=0, atol=TOL)
  np.testing.assert_allclose(got['stddev'], sd, rtol=0, atol=TOL)
  own, _ = mo.score_with_aux(pred, xs, ys, use_trust_region=tr, radius=radius, moments=(got['mean'], got['stddev']))
  np.testing.assert_allclose(got['score'], own, rtol=1e-12, atol=1e-300)   # subnormal MES values lose digits
  ref, aux = mo.score_with_aux(pred, xs, ys, use_trust_region=tr, radius=radius)
  _, s_mu, s_sd = mo.value_and_slopes(ys, mu, sd)
  assert np.all(np.abs(got['score'] - ref) <= TOL * (1 + np.abs(s_mu) + np.abs(s_sd)))
  if tr:
    np.testing.assert_array_equal(got['linf_distance'], aux['linf_distance'])


@pytest.mark.parametrize('tr', [True, False], ids=['tr', 'no-tr'])
@pytest.mark.parametrize('route', ['small', 'split', 'cluster', 'i8', 'general'])
def test_scoring_routes(route, tr):
  _, _, gp = _mods()
  x, y, pred, dev = _model(300, 6, linear=route == 'general', seed=5)
  dev.set_int('score_i8', 1 if route == 'i8' else 0)
  ys = dev.mes_fit(float(np.max(y))).cpu().numpy()
  m = _tiles(dev, route) * 64 - 5
  xs = np.random.default_rng(6).uniform(size=(m, 6))
  radius = 0.3
  a = gp.Acquisition(1.8, tr, radius, acq_fn=gp.MES)
  out = dev.score(xs, a, with_aux=True)
  dev.synchronize()
  assert dev.get_int('score_route') == {'small': SMALL, 'split': SPLIT, 'cluster': CLUSTER, 'i8': I8,
                                        'general': GENERAL}[route]
  mu, sd = go.predict(pred, xs)
  _check_scores(out, ys, pred, xs, tr, radius, mu, sd)
  # without the aux outputs (the pre-scaled variant of the kernels when no distance is needed): other moments in the
  # last bits, carried through the MES slopes
  fast = dev.score(xs, a)
  dev.synchronize()
  _, s_mu, s_sd = mo.value_and_slopes(ys, mu, sd)
  assert np.all(np.abs(fast['score'].cpu().numpy() - out['score'].cpu().numpy()) <= TOL * (1 + np.abs(s_mu) + np.abs(s_sd)))
  dev.close()


def test_injected_extremes():
  """Samples far below and far above the mean (gamma from -1e3 to 40, where log(normcdf) is -inf) and one at it."""
  _, _, gp = _mods()
  x, y, pred, dev = _model(40, 3, seed=3)
  xs = np.random.default_rng(4).uniform(size=(50, 3))
  mu, sd = _device_trial_moments(dev, xs)
  i = 0
  ys = mu[i] + sd[i] * np.array([-1e3, -500.0, -40.0, -39.0, -38.0, -37.0, -12.0, -1.0, 0.0, 1.0, 37.0, 40.0])
  dev.set_mes(ys)
  out = dev.score(xs, gp.Acquisition(1.8, False, 1.0, acq_fn=gp.MES), with_aux=True)
  dev.synchronize()
  got = out['score'].cpu().numpy()
  want = mo.value(ys, out['mean'].cpu().numpy(), out['stddev'].cpu().numpy())
  assert np.all(np.isfinite(got))
  np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
  dev.close()


@pytest.mark.parametrize('below', [False, True], ids=['samples-above', 'one-sample-below'])
def test_clamped_variance(below):
  """Candidates on well-separated trials with noise 1e-20: the variance is round-off around 0 and is clamped at some of
  them.  There MES takes its sd = 0 limits (0 for samples above the mean, +inf for one below) on the small-pool, split
  and general routes, and vzgp_score_grad gives it no gradient."""
  _, _, gp = _mods()
  x = np.stack(np.meshgrid(np.linspace(0.1, 0.9, 4), np.linspace(0.1, 0.9, 4)), -1).reshape(-1, 2)
  y = np.sin(3 * x[:, 0]) + x[:, 1]
  params = go.GPParams(1.0, np.full(2, 0.02), 1e-20)
  pred = lo.predictive(x, y, params)
  dev = gp.DeviceGP(0)
  dev.fit(x, y, lo.device_params(params))
  xs = np.concatenate([x, x + 1e-9, x - 1e-9])
  ys = np.array([3.0, 4.0, 5.0] + ([-5.0] if below else []))
  mes = gp.Acquisition(1.8, False, 1.0, acq_fn=gp.MES)
  seen = 0
  for tiles in (8, 0):                      # small-pool route, then k_score (split / cluster)
    dev.set_int('small_tiles', tiles)
    dev.set_mes(ys)
    out = dev.score(xs, mes, with_aux=True)
    dev.synchronize()
    sd = out['stddev'].cpu().numpy()
    got = out['score'].cpu().numpy()
    want = mo.value(ys, out['mean'].cpu().numpy(), sd)
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
    clamped = sd == 0
    seen += int(clamped.sum())
    assert np.all(got[clamped] == (np.inf if below else 0.0))
  g = dev.score_grad(xs, mes, with_aux=True)
  dev.synchronize()
  clamped = g['stddev'].cpu().numpy() == 0
  assert seen > 0 and clamped.any()
  assert np.all(g['grad'].cpu().numpy()[clamped] == 0.0)
  assert np.all(g['score'].cpu().numpy()[clamped] == (np.inf if below else 0.0))
  dev.close()


def _mes_score_fn(pred, ys, radius, d):
  return lambda q: go.apply_trust_region(mo.value(ys, *go.predict(pred, q)),
                                         go.min_linf_distance(q, pred.x, np.ones(d, bool), pred.row_valid), radius)


def _cfg(pool, batch, steps):
  _lib, _, _ = _mods()
  c = eo.EagleConfig()
  return c, _lib.EagleConfig(c.visibility, c.gravity, c.negative_gravity, c.perturbation, c.perturbation_lower_bound,
                             c.penalize_factor, c.normalization_scale, c.prior_trials_pool_pct, pool, batch,
                             steps * batch)


EAGLE_FORMS = [('persistent', 40, 4, 25, 25, 6), ('grid', 130, 3, 50, 25, 7), ('graph', 700, 12, 1200, 600, 3)]
EAGLE_ROUTE = {'persistent': 0, 'grid': 1, 'graph': 2}   # vzgp_eagle_route


@pytest.mark.parametrize('form,n,d,pool,batch,steps', EAGLE_FORMS, ids=[f[0] for f in EAGLE_FORMS])
def test_eagle_forms(form, n, d, pool, batch, steps):
  _, _, gp = _mods()
  x, y, pred, dev = _model(n, d, seed=21)
  ys = dev.mes_fit(float(np.max(y))).cpu().numpy()
  radius = go.trust_radius(n, d, 0)
  score_fn = _mes_score_fn(pred, ys, radius, d)
  cfg_o, cfg = _cfg(pool, batch, steps)
  wx, wr, _ = eo.run_eagle_optimizer(score_fn, dim=d, pool_size=pool, batch_size=batch,
                                     max_evaluations=steps * batch, count=3, seed=7, cfg=cfg_o, prior_features=x)
  bx, _, br = dev.eagle_run(cfg, gp.Acquisition(1.8, True, radius, acq_fn=gp.MES), count=3, seed=7, prior=x)
  assert dev.get_int('eagle_route') == EAGLE_ROUTE[form]
  if form != 'graph':
    np.testing.assert_allclose(br, wr, atol=1e-9)
    np.testing.assert_allclose(bx, wx, atol=1e-9)
  else:
    np.testing.assert_allclose(br, score_fn(bx), rtol=1e-10, atol=1e-10)
  dev.close()


def test_stepped_loop_matches_eagle_run():
  _, _, gp = _mods()
  n, d, pool, batch, steps = 120, 4, 50, 25, 6
  x, y, pred, dev = _model(n, d, seed=31)
  dev.mes_fit(float(np.max(y)))
  acq = gp.Acquisition(1.8, True, go.trust_radius(n, d, 0), acq_fn=gp.MES)
  _, cfg = _cfg(pool, batch, steps)
  bx0, _, br0 = dev.eagle_run(cfg, acq, count=3, seed=7, prior=x)
  se = gp.SteppedEagle(dev, cfg, 3, 7, n_prior=n)
  se.seed(x, None, dev.score(torch.from_numpy(x).cuda(), acq)['score'])
  for _ in range(steps):
    xs, _, rewards = se.ask()
    r = dev.score(xs, acq)['score']
    with torch.cuda.stream(dev._stream):
      rewards.copy_(r)
    se.tell()
  bx1, _, br1 = se.end()
  np.testing.assert_allclose(br1, br0, atol=1e-9)
  dev.close()


def test_random_search_indices():
  _, _, gp = _mods()
  n, d, m = 120, 6, 5000
  x, y, pred, dev = _model(n, d, seed=31)
  ys = dev.mes_fit(float(np.max(y))).cpu().numpy()
  radius = go.trust_radius(n, d, 0)
  bx, _, bs, bi = dev.random_search(m, gp.Acquisition(1.8, True, radius, acq_fn=gp.MES), 3, 99)
  wx, ws, wi = eo.run_random_optimizer(_mes_score_fn(pred, ys, radius, d), dim=d, num_candidates=m, count=3, seed=99)
  np.testing.assert_array_equal(bi, wi)
  np.testing.assert_array_equal(bx, wx)
  np.testing.assert_allclose(bs, ws, rtol=1e-10, atol=1e-10)
  dev.close()


GRAD_CASES = [(n, dc, lin) for n in (5, 65, 1000) for dc in (1, 20) for lin in (False, True)]


@pytest.mark.parametrize('n,dc,linear', GRAD_CASES, ids=[f'N{n}-D{d}{"-linear" if l else ""}' for n, d, l in GRAD_CASES])
def test_score_grad(n, dc, linear):
  _, _, gp = _mods()
  x, y, pred, dev = _model(n, dc, linear, seed=n + dc)
  ys = dev.mes_fit(float(np.max(y))).cpu().numpy()
  xs = np.random.default_rng(8).uniform(size=(300, dc))
  for tr in (False, True):
    acq = gp.Acquisition(1.8, tr, 0.3 if tr else 1.0, acq_fn=gp.MES)
    out = dev.score_grad(xs, acq, with_aux=True)
    dev.synchronize()
    want = mo.score_and_grad(pred, xs, acq, ys)
    _, s_mu, s_sd = mo.value_and_slopes(ys, want['mean'], want['stddev'])
    got = out['score'].cpu().numpy()
    assert np.all(np.abs(got - want['score']) <= TOL * (1 + np.abs(s_mu) + np.abs(s_sd)))
    np.testing.assert_allclose(out['mean'].cpu().numpy(), want['mean'], rtol=0, atol=TOL)
    np.testing.assert_allclose(out['stddev'].cpu().numpy(), want['stddev'], rtol=0, atol=TOL)
    # the MES slopes at the device's own moments: near the trials sd is small and the slopes change fast with
    # (mu, sd), so the moments' round-off would otherwise dominate the comparison
    want = mo.score_and_grad(pred, xs, acq, ys, slopes_at=(out['mean'].cpu().numpy(), out['stddev'].cpu().numpy()))
    g = out['grad'].cpu().numpy()
    scale = max(np.max(np.abs(want['grad'])), 1e-300)
    assert np.max(np.abs(g - want['grad'])) <= 1e-9 * scale, np.max(np.abs(g - want['grad'])) / scale
  dev.close()


def test_state_rules():
  _lib, _, gp = _mods()
  x, y, pred, dev = _model(60, 3, seed=9)
  params = pred.params
  xs = np.random.default_rng(1).uniform(size=(200, 3))
  ucb = gp.Acquisition(1.8, True, 0.3)
  base = dev.score(xs, ucb)['score'].cpu().numpy()
  dev.mes_fit(float(np.max(y)))
  mes = gp.Acquisition(1.8, True, 0.3, acq_fn=gp.MES)
  dev.score(xs, mes)
  # refit without mes_fit: the library refuses to score with the stale samples
  dev.fit(x, y, lo.device_params(params))
  xt = torch.from_numpy(xs).cuda()
  out = torch.empty(200, dtype=torch.float64, device='cuda')
  a, _ = mes._c()
  rc = dev._lib.vzgp_score(dev._h, C.c_void_p(xt.data_ptr()), None, 200, C.byref(a), C.c_void_p(out.data_ptr()),
                           None, None, None)
  assert rc == _lib.VZGP_ERR_ARG
  with pytest.raises(RuntimeError):
    dev.score(xs, mes)
  # back to UCB: bit-identical to before
  again = dev.score(xs, ucb)['score'].cpu().numpy()
  np.testing.assert_array_equal(again, base)
  dev.set_mes([0.5, 1.0, 1.5])
  np.testing.assert_allclose(dev.score(xs, mes, with_aux=True)['score'].cpu().numpy(),
                             mo.score_with_aux(pred, xs, [0.5, 1.0, 1.5], radius=0.3)[0], rtol=1e-9, atol=1e-9)
  # ensembles and stacks take the acquisition of hs[0] and refuse MES
  ens = gp.EnsembleGP(0, 2)
  ens.fit(x, y, [lo.device_params(params)] * 2)
  ens.members[0].set_mes([1.0])
  with pytest.raises(_lib.VzgpError):
    ens.score(xs, mes)
  with pytest.raises(_lib.VzgpError):
    ens.score_grad(xs, mes)
  stack = gp.StackedGP(0)
  l0 = stack.new_level(); l0.fit(x, y, lo.device_params(params)); stack.push(l0, 60)
  l0.set_mes([1.0])
  with pytest.raises(_lib.VzgpError):
    stack.score(xs, mes)
  # GP-UCB-PE ignores the handle's acquisition
  other = gp.DeviceGP(0, stream=dev.stream)
  other.fit(x, y, lo.device_params(params))
  pe = gp.UcbPeAcquisition(mode=1, threshold=0.0, trust_radius=0.3)
  dev.set_acquisition(None)
  before = dev.score_pe(other, xs, pe)['score'].cpu().numpy()
  dev.set_mes([1.0, 2.0])
  np.testing.assert_array_equal(dev.score_pe(other, xs, pe)['score'].cpu().numpy(), before)
  for h in (dev, other, ens, stack):
    h.close()


def _designer_problem(d=3):
  from vizier_b200 import vz
  p = vz.ProblemStatement()
  for i in range(d):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='obj', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  return p


@pytest.mark.parametrize('optimizer', ['eagle', 'lbfgsb'])
def test_designer_loop(optimizer):
  from vizier_b200 import optimizers as vb, vz
  from vizier_b200.designers import gp_bandit
  _, acq, _ = _mods()
  opt = (vb.LBFGSBOptimizerFactory() if optimizer == 'lbfgsb' else
         vb.VectorizedOptimizerFactory(strategy_factory=vb.VectorizedEagleStrategyFactory(), max_evaluations=1000,
                                       suggestion_batch_size=25))
  des = gp_bandit.VizierGPBandit.from_problem(_designer_problem(), seed=2, acquisition_optimizer_factory=opt,
                                             scoring_function_factory=acq.MaxValueEntropySearch.scoring_fn_factory)
  f = lambda v: -np.sum((v - 0.3) ** 2)
  tid = 1
  for _ in range(20):
    s = des.suggest(1)[0]
    t = s.to_trial(tid); tid += 1
    v = np.array([t.parameters[k].value for k in sorted(t.parameters)])
    t.complete(vz.Measurement({'obj': float(f(v))}))
    des.update(vz.CompletedTrials([t]), vz.ActiveTrials())
  info = json.loads(s.metadata.ns('devinfo')['acquisition_optimization'])
  cont, _, labels = des._trials_to_data(des._trials[:-1])
  xw, _ = des._converter.to_features([t])
  q = des._last_params
  pred = go.precompute_predictive(go.GPParams(q.signal_variance, q.continuous_length_scale_squared,
                                              q.observation_noise_variance), cont, labels[:, 0])
  ys = mo.fit_predictive(pred, float(np.max(labels)), 100, 123)['samples']
  mu, sd = go.predict(pred, xw)
  raw = float(mo.value(ys, mu, sd)[0])
  assert abs(info['raw_acquisition'] - raw) < 1e-10 * max(1.0, abs(raw))
  assert abs(info['mean'] - float(mu[0])) < 1e-10 and abs(info['stddev'] - float(sd[0])) < 1e-10
  dist = go.min_linf_distance(xw, cont, np.ones(3, bool), np.ones(len(cont), bool))
  want = float(go.apply_trust_region(np.array([raw]), dist, info['radius'])[0])
  assert abs(info['acquisition'] - want) < 1e-10 * max(1.0, abs(want))
