"""Acquisition functions other than UCB (LCB, EI, PI and the AcquisitionTrustRegion presets) on every scoring route
and in every acquisition optimiser, against tests/acq_oracle.py: score, mean and stddev within 1e-10, the L-inf
distance bit for bit.  Candidates whose thresholding value lies within 1e-12 of the threshold are left out of the
score comparison (either side is right there).  Also: switching acquisitions on one handle, and the GP-UCB-PE and
multi-metric calls ignoring the handle's acquisition."""
import json

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

import acq_oracle as ao  # noqa: E402
from oracle import eagle_oracle as eo  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402

TOL = 1e-10
SMALL, SPLIT, CLUSTER, I8, GENERAL = 0, 1, 2, 3, 4


def _mods():
  from vizier_b200 import _lib, acquisitions, gp
  return _lib, acquisitions, gp


def _data(y):
  _, acq, _ = _mods()
  return acq.ModelData(features=None, labels=acq.PaddedArray.as_padded(np.asarray(y, np.float64).reshape(-1, 1)))


def _acq_fns(y):
  _, acq, _ = _mods()
  d = _data(y)
  best = acq.get_best_labels(d.labels)
  return {
      'LCB': acq.LCB(1.3), 'EI': acq.EI(best), 'PI': acq.PI(best),
      'ucb_pi': acq.AcquisitionTrustRegion.default_ucb_pi(d), 'ucb_lcb': acq.AcquisitionTrustRegion.default_ucb_lcb(d),
      'ucb_lcb_wide': acq.AcquisitionTrustRegion.default_ucb_lcb_wide(d),
      'ucb_lcb_delay_tr': acq.AcquisitionTrustRegion.default_ucb_lcb_delay_tr(d),
  }


KINDS = ['LCB', 'EI', 'PI', 'ucb_pi', 'ucb_lcb', 'ucb_lcb_wide', 'ucb_lcb_delay_tr']


def _problem(n, d, seed, dk=0):
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, d))
  y = np.sin(3 * x[:, 0]) - np.sum((x - 0.4) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  z = rng.integers(0, 3, size=(n, dk)).astype(np.int32) if dk else None
  return x, y, z


def _near_threshold(fn, mu, sd):
  """Candidates whose thresholding value is within 1e-12 of the lowered threshold."""
  _, acq, gp = _mods()
  spec = acq.lower_acquisition(fn)
  if spec.thresholding is None:
    return np.zeros(mu.shape, bool)
  t = ao.evaluate_spec(gp.AcqFnSpec(spec.thresholding), mu, sd)
  return np.abs(t - spec.threshold) < 1e-12


def _compare(out, fn, mu, sd, want, dist=None):
  got = {k: out[k].cpu().numpy() for k in ('score', 'mean', 'stddev', 'linf_distance') if k in out}
  np.testing.assert_allclose(got['mean'], mu, rtol=0, atol=TOL)
  np.testing.assert_allclose(got['stddev'], sd, rtol=0, atol=TOL)
  keep = ~_near_threshold(fn, mu, sd)
  assert keep.mean() > 0.99
  np.testing.assert_allclose(got['score'][keep], want[keep], rtol=0, atol=TOL)
  if dist is not None:
    np.testing.assert_array_equal(got['linf_distance'], dist)


def _tiles(dev, route):
  sm = dev.get_int('sm_count')
  return {'small': 4, 'split': min(9, sm // 2), 'cluster': sm // 2 + 1, 'i8': sm + 1}[route]


ROUTE_CASES = [('small', 300, 6, 0), ('split', 300, 6, 0), ('cluster', 300, 6, 0), ('i8', 300, 6, 0),
               ('small', 200, 4, 2), ('cluster', 200, 4, 2)]


@pytest.mark.parametrize('tr', [True, False], ids=['tr', 'no-tr'])
@pytest.mark.parametrize('route,n,d,dk', ROUTE_CASES, ids=[f'{r}-N{n}-dk{k}' for r, n, _, k in ROUTE_CASES])
def test_single_model_routes(route, n, d, dk, tr):
  _lib, acq, gp = _mods()
  x, y, z = _problem(n, d, 5, dk)
  ls2 = 0.4 * (1 + np.arange(d) / d)
  lk = np.linspace(0.7, 1.3, dk) if dk else None
  po, pg = go.GPParams(1.0, ls2, 1e-3, lk), gp.GPHyperParams(1.0, ls2, 1e-3, lk)
  pred = go.precompute_predictive(po, x, y, z)
  dev = gp.DeviceGP(0)
  dev.fit(x, y, pg, z=z)
  dev.set_int('score_i8', 1 if route == 'i8' else 0)
  m = _tiles(dev, route) * 64 - 5
  rng = np.random.default_rng(6)
  xs = rng.uniform(size=(m, d))
  zs = rng.integers(0, 3, size=(m, dk)).astype(np.int32) if dk else None
  radius = 0.3
  mu, sd = go.predict(pred, xs, zs)
  dist = go.min_linf_distance(xs, x, np.ones(d, bool), pred.row_valid)
  for kind, fn in _acq_fns(y).items():
    a = gp.Acquisition(1.8, tr, radius, acq_fn=acq.lower_acquisition(fn))
    out = dev.score(xs, a, zs=zs, with_aux=True)
    dev.synchronize()
    assert dev.get_int('score_route') == {'small': SMALL, 'split': SPLIT, 'cluster': CLUSTER, 'i8': I8}[route], kind
    want = ao.evaluate(fn, mu, sd)
    if tr:
      want = go.apply_trust_region(want, dist, radius)
    _compare(out, fn, mu, sd, want, dist)
    # without the aux outputs (the pre-scaled variant of the kernels when no distance is needed)
    fast = dev.score(xs, a, zs=zs)
    dev.synchronize()
    keep = ~_near_threshold(fn, mu, sd)
    np.testing.assert_allclose(fast['score'].cpu().numpy()[keep], want[keep], rtol=0, atol=TOL)
  dev.close()


@pytest.mark.parametrize('tr', [True, False], ids=['tr', 'no-tr'])
def test_general_route_linear_model(tr):
  _lib, acq, gp = _mods()
  n, d = 90, 4
  x, y, _ = _problem(n, d, 8)
  ls2 = 0.5 * (1 + np.arange(d) / d)
  po = go.GPParams(0.8, ls2, 2e-3, None, go.LinearParams(0.1, 0.9, 0.3, -0.4))
  pg = gp.GPHyperParams(0.8, ls2, 2e-3, None, 0.1, 0.9, 0.3, -0.4)
  pred = go.precompute_predictive(po, x, y)
  dev = gp.DeviceGP(0)
  dev.fit(x, y, pg)
  xs = np.random.default_rng(9).uniform(size=(777, d))
  mu, sd = go.predict(pred, xs)
  dist = go.min_linf_distance(xs, x, np.ones(d, bool), pred.row_valid)
  for kind, fn in _acq_fns(y).items():
    out = dev.score(xs, gp.Acquisition(1.8, tr, 0.3, acq_fn=acq.lower_acquisition(fn)), with_aux=True)
    dev.synchronize()
    assert dev.get_int('score_route') == GENERAL
    want = ao.evaluate(fn, mu, sd)
    _compare(out, fn, mu, sd, go.apply_trust_region(want, dist, 0.3) if tr else want, dist)
  dev.close()


@pytest.mark.parametrize('m', [200, 20_000])
def test_ensemble_and_stack(m):
  _lib, acq, gp = _mods()
  n, d = 120, 5
  x, y, _ = _problem(n, d, 11)
  xs = np.random.default_rng(12).uniform(size=(m, d))
  plist = [(0.9, np.full(d, 0.4), 1e-3), (1.3, np.linspace(0.2, 0.9, d), 3e-3), (0.6, np.full(d, 0.7), 2e-3)]
  preds = [go.precompute_predictive(go.GPParams(*p), x, y) for p in plist]
  ens = gp.EnsembleGP(0, 3)
  ens.fit(x, y, [gp.GPHyperParams(*p) for p in plist])
  mu, sd = go.predict_ensemble(preds, xs)
  dist = go.min_linf_distance(xs, x, np.ones(d, bool), preds[0].row_valid)
  for kind, fn in _acq_fns(y).items():
    out = ens.score(xs, gp.Acquisition(1.8, True, 0.3, acq_fn=acq.lower_acquisition(fn)), with_aux=True)
    ens.synchronize()
    _compare(out, fn, mu, sd, go.apply_trust_region(ao.evaluate(fn, mu, sd), dist, 0.3), dist)
  # stack of two levels: a prior study and the current one on its residuals
  x0, y0, _ = _problem(80, d, 13)
  stack = gp.StackedGP(0)
  p0 = go.precompute_predictive(go.GPParams(*plist[0]), x0, y0)
  l0 = stack.new_level(); l0.fit(x0, y0, gp.GPHyperParams(*plist[0])); stack.push(l0, 80)
  resid = go.stack_residual_labels([p0], x, y)
  p1 = go.precompute_predictive(go.GPParams(*plist[1]), x, resid)
  l1 = stack.new_level(); l1.fit(x, resid, gp.GPHyperParams(*plist[1])); stack.push(l1, n)
  mu, sd = go.predict_stack([p0, p1], xs)
  for kind, fn in _acq_fns(y).items():
    out = stack.score(xs, gp.Acquisition(1.8, True, 0.3, acq_fn=acq.lower_acquisition(fn)), with_aux=True)
    stack.synchronize()
    _compare(out, fn, mu, sd, go.apply_trust_region(ao.evaluate(fn, mu, sd), dist, 0.3), dist)
  ens.synchronize()
  stack.close()


def _eagle(dev, pred, fn, x, d, pool, batch, steps, a, trajectory=True):
  cfg_o = eo.EagleConfig()
  radius = a.trust_radius
  score_fn = lambda q: go.apply_trust_region(ao.evaluate(fn, *go.predict(pred, q)),
                                             go.min_linf_distance(q, pred.x, np.ones(d, bool), pred.row_valid), radius)
  wx, wr, _ = eo.run_eagle_optimizer(score_fn, dim=d, pool_size=pool, batch_size=batch, max_evaluations=steps * batch,
                                     count=3, seed=7, cfg=cfg_o, prior_features=x)
  _lib, _, _ = _mods()
  cfg = _lib.EagleConfig(cfg_o.visibility, cfg_o.gravity, cfg_o.negative_gravity, cfg_o.perturbation,
                         cfg_o.perturbation_lower_bound, cfg_o.penalize_factor, cfg_o.normalization_scale,
                         cfg_o.prior_trials_pool_pct, pool, batch, steps * batch)
  bx, _, br = dev.eagle_run(cfg, a, count=3, seed=7, prior=x)
  if trajectory:
    np.testing.assert_allclose(br, wr, atol=1e-9)
    np.testing.assert_allclose(bx, wx, atol=1e-9)
  else:
    # the winners' rewards are the acquisition at the winners, and as good as the oracle's run up to 1e-4
    np.testing.assert_allclose(br, score_fn(bx), rtol=0, atol=1e-10)
    assert br[0] >= wr[0] - 1e-4 * max(1.0, abs(wr[0]))


# persistent (N <= 64, batch <= 64), grid (batch <= 512), graph (batch > 512).  The graph form scores its 600-candidate
# batches with k_score, whose sums round differently from the oracle's in the last bits; over 1200 flies with EI's
# nearly flat values that is enough to flip a pool comparison and part the two trajectories, so there the test checks
# the winners' rewards against the oracle's acquisition at the winners instead of the whole trajectory.
EAGLE_FORMS = [('persistent', 40, 4, 25, 25, 6), ('grid', 130, 3, 50, 25, 7), ('graph', 700, 12, 1200, 600, 4)]


@pytest.mark.parametrize('form,n,d,pool,batch,steps', EAGLE_FORMS, ids=[f[0] for f in EAGLE_FORMS])
def test_eagle_forms_and_switching(form, n, d, pool, batch, steps):
  _lib, acq, gp = _mods()
  x, y, _ = _problem(n, d, 21)
  ls2 = np.full(d, 0.3)
  pred = go.precompute_predictive(go.GPParams(1.0, ls2, 1e-3), x, y)
  dev = gp.DeviceGP(0)
  dev.fit(x, y, gp.GPHyperParams(1.0, ls2, 1e-3))
  radius = go.trust_radius(n, d, 0)
  fns = _acq_fns(y)
  ucb = acq.UCB(1.8)
  # EI, UCB, the ucb_pi preset and EI again on one handle: each run matches the oracle of its own acquisition
  for fn in (fns['EI'], ucb, fns['ucb_pi'], fns['EI']):
    spec = None if fn is ucb else acq.lower_acquisition(fn)
    _eagle(dev, pred, fn, x, d, pool, batch, steps, gp.Acquisition(1.8, True, radius, acq_fn=spec), form != 'graph')
  dev.close()


@pytest.mark.parametrize('kind', ['EI', 'ucb_pi'])
def test_random_search(kind):
  _lib, acq, gp = _mods()
  n, d, m = 120, 6, 5000
  x, y, _ = _problem(n, d, 31)
  ls2 = np.full(d, 0.5)
  pred = go.precompute_predictive(go.GPParams(1.0, ls2, 1e-3), x, y)
  dev = gp.DeviceGP(0)
  dev.fit(x, y, gp.GPHyperParams(1.0, ls2, 1e-3))
  fn = _acq_fns(y)[kind]
  radius = go.trust_radius(n, d, 0)
  bx, _, bs, bi = dev.random_search(m, gp.Acquisition(1.8, True, radius, acq_fn=acq.lower_acquisition(fn)), 3, 99)
  score_fn = lambda q: go.apply_trust_region(ao.evaluate(fn, *go.predict(pred, q)),
                                             go.min_linf_distance(q, x, np.ones(d, bool), pred.row_valid), radius)
  wx, ws, wi = eo.run_random_optimizer(score_fn, dim=d, num_candidates=m, count=3, seed=99)
  np.testing.assert_array_equal(bi, wi)
  np.testing.assert_array_equal(bx, wx)
  np.testing.assert_allclose(bs, ws, atol=TOL)
  dev.close()


def test_pe_and_multi_ignore_the_handle_acquisition():
  _lib, acq, gp = _mods()
  n, d, m = 100, 4, 3000
  x, y, _ = _problem(n, d, 41)
  xs = np.random.default_rng(42).uniform(size=(m, d))
  ls2 = np.full(d, 0.4)
  a = gp.DeviceGP(0)
  b = gp.DeviceGP(0, stream=a.stream)
  a.fit(x, y, gp.GPHyperParams(1.0, ls2, 1e-3))
  b.fit(np.vstack([x, xs[:10]]), np.concatenate([y, np.zeros(10)]), gp.GPHyperParams(1.0, ls2, 1e-3))
  ei = acq.lower_acquisition(_acq_fns(y)['EI'])
  pe = gp.UcbPeAcquisition(mode=1, threshold=0.1, trust_radius=0.3)
  before = {k: v.cpu().numpy() for k, v in a.score_pe(b, xs, pe).items()}
  a.set_acquisition(ei); b.set_acquisition(ei)
  after = {k: v.cpu().numpy() for k, v in a.score_pe(b, xs, pe).items()}
  for k in before:
    np.testing.assert_array_equal(after[k], before[k])
  # multi-metric model on the same handle
  y2 = np.stack([y, np.cos(x[:, 1])], axis=1)
  a.set_acquisition(None)
  a.fit(x, y2, gp.GPHyperParams(1.0, ls2, 1e-3))
  w = np.abs(np.random.default_rng(43).normal(size=(16, 2)))
  sc = gp.ScalarizedUcbAcquisition(w / np.linalg.norm(w, axis=1, keepdims=True), np.array([-2.0, -2.0]))
  before = a.score_multi(xs, sc, with_aux=True)
  a.synchronize()
  before = {k: before[k].cpu().numpy() for k in ('score', 'mean', 'stddev')}
  a.set_acquisition(ei)
  after = a.score_multi(xs, sc, with_aux=True)
  a.synchronize()
  for k in before:
    np.testing.assert_array_equal(after[k].cpu().numpy(), before[k])
  a.close(); b.close()


def test_set_acquisition_validates():
  _lib, acq, gp = _mods()
  dev = gp.DeviceGP(0)
  with pytest.raises(_lib.VzgpError):
    dev.set_acquisition(gp.AcqFnSpec(gp.AcqTermSpec(7)))
  with pytest.raises(_lib.VzgpError):
    dev.set_acquisition(gp.AcqFnSpec(gp.AcqTermSpec(_lib.ACQ_EI, best_label=-np.inf)))
  dev.set_acquisition(gp.AcqFnSpec(gp.AcqTermSpec(_lib.ACQ_PI, best_label=0.5)))
  dev.set_acquisition(None)
  dev.close()


def _designer_problem(d=3):
  from vizier_b200 import vz
  p = vz.ProblemStatement()
  for i in range(d):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='obj', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  return p


@pytest.mark.parametrize('preset,extra', [('EI', {}), ('ucb_pi', {}), ('EI', {'ensemble_size': 3, 'linear_coef': 0.1})],
                         ids=['EI', 'ucb_pi', 'EI-ensemble3-linear'])
def test_designer_loop(preset, extra):
  from vizier_b200 import optimizers as vb, vz
  from vizier_b200.designers import gp_bandit
  _lib, acq, gp = _mods()
  factory = acq.bayesian_scoring_function_factory(
      (lambda dd: acq.EI(acq.get_best_labels(dd.labels))) if preset == 'EI' else acq.AcquisitionTrustRegion.default_ucb_pi)
  opt = vb.VectorizedOptimizerFactory(strategy_factory=vb.VectorizedEagleStrategyFactory(), max_evaluations=1000,
                                      suggestion_batch_size=25)
  p = _designer_problem()
  des = gp_bandit.VizierGPBandit.from_problem(p, seed=2, acquisition_optimizer_factory=opt, scoring_function_factory=factory,
                                             **extra)
  f = lambda v: -np.sum((v - 0.3) ** 2)
  tid = 1
  for _ in range(20):
    s = des.suggest(1)[0]
    t = s.to_trial(tid); tid += 1
    v = np.array([t.parameters[k].value for k in sorted(t.parameters)])
    t.complete(vz.Measurement({'obj': float(f(v))}))
    des.update(vz.CompletedTrials([t]), vz.ActiveTrials())
  info = json.loads(s.metadata.ns('devinfo')['acquisition_optimization'])
  # the acquisition at the winner, recomputed by the oracle from the designer's own data and model
  cont, cat, labels = des._trials_to_data(des._trials[:-1])
  xw, _ = des._converter.to_features([t])
  fn = des._scoring_function(acq.ModelData(None, acq.PaddedArray.as_padded(labels))).acquisition_fn
  params = des._last_params if isinstance(des._last_params, list) else [des._last_params]
  preds = [go.precompute_predictive(go.GPParams(q.signal_variance, q.continuous_length_scale_squared,
                                                q.observation_noise_variance, None,
                                                go.LinearParams(q.linear_coef, q.linear_slope_amplitude, q.linear_shift,
                                                                q.mean_constant) if q.linear_coef else None),
                                    cont, labels[:, 0]) for q in params]
  mu, sd = go.predict_ensemble(preds, xw) if len(preds) > 1 else go.predict(preds[0], xw)
  raw = float(ao.evaluate(fn, mu, sd)[0])
  assert abs(info['raw_acquisition'] - raw) < 1e-10 * max(1.0, abs(raw))
  assert abs(info['mean'] - float(mu[0])) < 1e-10 and abs(info['stddev'] - float(sd[0])) < 1e-10
  dist = go.min_linf_distance(xw, cont, np.ones(3, bool), np.ones(len(cont), bool))
  want = float(go.apply_trust_region(np.array([raw]), dist, info['radius'])[0])
  assert abs(info['acquisition'] - want) < 1e-10 * max(1.0, abs(want))
