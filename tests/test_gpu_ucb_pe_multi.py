"""Multi-metric GP-UCB-PE on the GPU against the tests-side oracle (pe_multi_oracle.py): vzgp_score_pe_multi on every
scoring route, the Eagle loop with that scorer, the host-stepped loop, and VizierGPUCBPEBandit end to end with two
metrics (gp_ucb_pe_test.py:144-360)."""
import ast
import copy

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from oracle import eagle_oracle as eo  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402
import pe_multi_oracle as pmo  # noqa: E402

SMALL, SPLIT, CLUSTER = 0, 1, 2   # vzgp_score_route
AGGS = (pmo.AVERAGE, pmo.UNION, pmo.INTERSECTION)


def _models(n, n_pending, d, dk, m, seed, sm=None):
  """Model A (independent multi-task GP, m metrics) on n trials, model B on n + n_pending trials with zero labels;
  oracle predictives and device handles on one stream."""
  from vizier_b200 import gp
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, d))
  z = rng.integers(0, 3, size=(n, dk)).astype(np.int32) if dk else None
  y = np.stack([np.sin(3 * x[:, k % d] + k) - np.sum((x - 0.15 * k) ** 2, axis=1) + 0.05 * rng.normal(size=n)
                for k in range(m)], axis=1)
  xb = np.concatenate([x, rng.uniform(size=(n_pending, d))])
  zb = np.concatenate([z, rng.integers(0, 3, size=(n_pending, dk)).astype(np.int32)]) if dk else None
  ls2 = 0.5 * (1 + np.arange(d) / d)
  lk = np.linspace(0.7, 1.3, dk) if dk else None
  po = go.GPParams(1.2, ls2, 1e-3, lk)
  pg = gp.GPHyperParams(1.2, ls2, 1e-3, lk)
  pred_a = go.precompute_predictive(po, x, y, z)
  pred_b = go.precompute_predictive(po, xb, np.zeros(n + n_pending), zb)
  dev_a = gp.DeviceGP(0)
  dev_b = gp.DeviceGP(0, stream=dev_a.stream)
  for h in (dev_a, dev_b):
    h.set_int('score_i8', 0)
    h.set_int('small_tiles', -1)
  assert dev_a.fit(x, y, pg, z=z) == 0
  assert dev_b.fit(xb, np.zeros(n + n_pending), pg, z=zb) == 0
  return rng, x, y, xb, pred_a, pred_b, dev_a, dev_b


def _route(sm, m, n):
  """The route launch_score takes for m candidates on n trials (default small_tiles, no integer split)."""
  tiles = -(-m // 64)
  if tiles <= 8:
    return SMALL
  nblocks = -(-(-(-n // 64) * 64) // 128)
  nsplit = (nblocks + 1) // 2 if (2 * tiles <= sm and nblocks >= 2) else 1
  return SPLIT if nsplit > 1 else CLUSTER


def _close(got, want):
  want = np.asarray(want, np.float64)
  err = np.abs(np.asarray(got) - want)
  tol = 1e-10 * np.maximum(1.0, np.abs(want))
  assert np.all(err <= tol), (float(np.max(err / tol)), np.unravel_index(np.argmax(err / tol), err.shape))


# route, n, n_pending, d, dk, metrics, candidates (a callable of the SM count)
CASES = [
    pytest.param(SMALL, 40, 5, 3, 1, 2, lambda sm: 300, id='small-m2-cat'),
    pytest.param(SPLIT, 300, 8, 4, 0, 3, lambda sm: 20 * 64 - 11, id='split-m3'),
    pytest.param(CLUSTER, 150, 10, 5, 2, 8, lambda sm: (sm // 2 + 1) * 64 + 9, id='cluster-m8-cat'),
]


@pytest.mark.parametrize('route,n,n_pending,d,dk,m,count', CASES)
def test_score_pe_multi_matches_oracle(route, n, n_pending, d, dk, m, count):
  from vizier_b200 import gp
  rng, x, y, xb, pred_a, pred_b, dev_a, dev_b = _models(n, n_pending, d, dk, m, 7 + m)
  try:
    sm = dev_a.get_int('sm_count')
    mc = count(sm)
    xs = rng.uniform(size=(mc, d))
    xs[:5] = x[:5]
    zs = rng.integers(0, 3, size=(mc, dk)).astype(np.int32) if dk else None
    mu, sd = go.predict(pred_a, xs, zs)
    mu = mu.reshape(mc, m)
    _, sd_b = go.predict(pred_b, xs, zs)
    thr = pmo.ucb_thresholds_multi(pred_a, pred_b)
    w = np.abs(rng.normal(size=(1000, m))); w /= np.linalg.norm(w, axis=1, keepdims=True)
    ref = go.hv_reference_point(y)
    best = go.hv_max_scalarized(y, w, ref)
    mask = np.ones(d, bool); mask[d - 1] = False
    tr_rows = n + n_pending - 3
    dist = go.min_linf_distance(xs, xb[:tr_rows], mask)
    seen_tr = False
    for use_tr, radius in ((False, 1.0), (True, 0.2), (True, 0.7)):
      configs = [dict(mode=0, floor=floor) for floor in (best, None)] + [dict(mode=1, agg=a) for a in AGGS]
      for c in configs:
        sc = gp.ScalarizedUcbAcquisition(w, ref, c.get('floor'), 1.8) if c['mode'] == 0 else None
        pe = gp.UcbPeMultiAcquisition(n_metrics=m, mode=c['mode'], thresholds=thr, region_penalty=c.get('agg', 0),
                                      scalarization=sc, use_trust_region=use_tr, trust_radius=radius, tr_dim_mask=mask,
                                      tr_rows=tr_rows)
        out = dev_a.score_pe_multi(dev_b, xs, pe, zs=zs)
        assert dev_a.get_int('score_route') == _route(sm, mc, n) == route
        assert dev_b.get_int('score_route') == _route(sm, mc, n + n_pending)
        want = pmo.combine(mu, sd, sd_b, mode=c['mode'], thresholds=thr, region_penalty=c.get('agg', 0), weights=w,
                           reference_point=ref, max_scalarized=c.get('floor'),
                           dist=dist if use_tr else None, trust_radius_value=radius)
        _close(out['mean'].cpu().numpy().T, mu)
        _close(out['stddev'].cpu().numpy(), sd)
        _close(out['stddev_from_all'].cpu().numpy(), sd_b)
        _close(out['score'].cpu().numpy(), want)
        if use_tr and radius <= 0.5:
          assert np.any(want < -1e3) and np.any(want > -1e3)
          seen_tr = True
    assert seen_tr
  finally:
    dev_b.close(); dev_a.close()


def _eagle_cfgs(pool, batch, steps):
  from vizier_b200 import _lib
  from vizier_b200.designers import gp_ucb_pe
  c = gp_ucb_pe.default_eagle_config
  cfg_o = eo.EagleConfig(visibility=c.visibility, gravity=c.gravity, negative_gravity=c.negative_gravity,
                         perturbation=c.perturbation, perturbation_lower_bound=c.perturbation_lower_bound,
                         penalize_factor=c.penalize_factor, normalization_scale=c.normalization_scale,
                         prior_trials_pool_pct=c.prior_trials_pool_pct, mutate_normalization_type=1)
  cfg = _lib.EagleConfig(cfg_o.visibility, cfg_o.gravity, cfg_o.negative_gravity, cfg_o.perturbation,
                         cfg_o.perturbation_lower_bound, cfg_o.penalize_factor, cfg_o.normalization_scale,
                         cfg_o.prior_trials_pool_pct, pool, batch, steps * batch, 1.0, 30.0, 0.98, 1)
  return cfg_o, cfg


def test_eagle_run_pe_multi_matches_oracle():
  """vzgp_eagle_run_pe_multi against the oracle optimiser with the oracle score (GP-UCB-PE's Eagle configuration,
  RANDOM force normalisation), both modes."""
  from vizier_b200 import gp
  n, n_pending, d, m = 40, 3, 3, 2
  rng, x, y, xb, pred_a, pred_b, dev_a, dev_b = _models(n, n_pending, d, 0, m, 21)
  try:
    mask = np.ones(d, bool)
    rows = n + n_pending
    radius = go.trust_radius(rows, d, 0)
    thr = pmo.ucb_thresholds_multi(pred_a, pred_b)
    w = np.abs(rng.normal(size=(1000, m))); w /= np.linalg.norm(w, axis=1, keepdims=True)
    ref = go.hv_reference_point(y); best = go.hv_max_scalarized(y, w, ref)
    pool, batch, steps = 25, 25, 7
    cfg_o, cfg = _eagle_cfgs(pool, batch, steps)
    for mode, agg in ((0, 0), (1, pmo.UNION), (1, pmo.AVERAGE)):
      def score_fn(xc, xz, mode=mode, agg=agg):
        return pmo.ucb_pe_multi_score(pred_a, pred_b, xc, mode=mode, thresholds=thr, region_penalty=agg, weights=w,
                                      reference_point=ref, max_scalarized=best, tr_dim_mask=mask, tr_rows=rows,
                                      trust_radius_value=radius)[0]
      wc, _, wr = eo.run_eagle_optimizer_mixed(score_fn, dim=d, sizes=np.zeros(0, int), pool_size=pool, batch_size=batch,
                                               max_evaluations=steps * batch, count=2, seed=13, cfg=cfg_o, prior_c=x,
                                               prior_z=np.zeros((n, 0), np.int32))
      pe = gp.UcbPeMultiAcquisition(n_metrics=m, mode=mode, thresholds=thr, region_penalty=agg,
                                    scalarization=gp.ScalarizedUcbAcquisition(w, ref, best, 1.8), trust_radius=radius,
                                    tr_dim_mask=mask)
      bx, _, br = dev_a.eagle_run(cfg, pe, 2, 13, prior=x, other=dev_b)
      np.testing.assert_allclose(br, wr, atol=1e-9 * max(1.0, np.max(np.abs(wr))), rtol=0)
      np.testing.assert_allclose(bx, wc, atol=1e-9, rtol=0)
  finally:
    dev_b.close(); dev_a.close()


def test_stepped_loop_with_zero_prior_equals_device_loop():
  """VectorizedOptimizer with a zero prior_acquisition (host-stepped loop, vzgp_score_pe_multi per batch) finds what
  the graph-replayed device loop finds."""
  from vizier_b200 import gp
  from vizier_b200 import optimizers as vb
  from vizier_b200.designers import gp_ucb_pe
  n, n_pending, d, dk, m = 60, 4, 3, 1, 2
  rng, x, y, xb, pred_a, pred_b, dev_a, dev_b = _models(n, n_pending, d, dk, m, 31)
  try:
    thr = pmo.ucb_thresholds_multi(pred_a, pred_b)
    w = np.abs(rng.normal(size=(1000, m))); w /= np.linalg.norm(w, axis=1, keepdims=True)
    ref = go.hv_reference_point(y); best = go.hv_max_scalarized(y, w, ref)
    opt = vb.VectorizedOptimizer(vb.VectorizedEagleStrategyFactory(eagle_config=gp_ucb_pe.default_eagle_config), d, dk,
                                 25, 1000, (3,))
    calls = []

    def zero(xc, xz):
      calls.append(xc.shape[0])
      return np.zeros(xc.shape[0])

    for mode in (0, 1):
      pe = gp.UcbPeMultiAcquisition(n_metrics=m, mode=mode, thresholds=thr, region_penalty=pmo.INTERSECTION,
                                    scalarization=gp.ScalarizedUcbAcquisition(w, ref, best, 1.8), trust_radius=0.3,
                                    tr_dim_mask=np.ones(d, bool), tr_rows=n + n_pending)
      zp = np.zeros((n, dk), np.int32)
      dev = opt(dev_a, pe, count=2, prior_features=x, prior_categorical=zp, seed=5, other=dev_b)
      host = opt(dev_a, pe, count=2, prior_features=x, prior_categorical=zp, seed=5, other=dev_b, prior_acquisition=zero)
      np.testing.assert_array_equal(host.features, dev.features)
      np.testing.assert_array_equal(host.categorical, dev.categorical)
      np.testing.assert_array_equal(host.rewards, dev.rewards)
      assert dev.aux['mean'].shape == (2, m) and dev.aux['stddev_from_all'].shape == (2,)
      np.testing.assert_array_equal(host.aux['prior_acq_values'], np.zeros(2))
    assert calls
    with pytest.raises(NotImplementedError):
      vb.VectorizedOptimizer(vb.random_strategy_factory, d, dk, 100, 100, (3,))(dev_a, pe, other=dev_b)
  finally:
    dev_b.close(); dev_a.close()


def _predictions(md):
  pred = md.ns('prediction_in_warped_y_space')
  vec = {k: np.asarray(ast.literal_eval(pred[k]), np.float64) for k in ('mean', 'stddev', 'stddev_from_all')}
  return vec, float(pred['acquisition']), pred['use_ucb'] == 'True'


def _problem():
  from vizier_b200 import vz
  p = vz.ProblemStatement()
  p.search_space.root.add_float_param('x0', -2.0, 2.0)
  p.search_space.root.add_float_param('x1', 0.1, 10.0, scale_type=vz.ScaleType.LOG)
  p.search_space.root.add_float_param('x2', 0.0, 1.0)
  for k in range(2):
    goal = vz.ObjectiveMetricGoal.MAXIMIZE if k == 0 else vz.ObjectiveMetricGoal.MINIMIZE
    p.metric_information.append(vz.MetricInformation(name=f'metric{k}', goal=goal))
  return p


@pytest.mark.parametrize('penalty,high_noise', [('UNION', False), ('INTERSECTION', False), ('AVERAGE', False),
                                                ('AVERAGE', True)])
def test_designer_two_metrics(penalty, high_noise):
  """gp_ucb_pe_test.py:144-360 with two metrics (metric1 minimised): two batches on active trials only, then the
  oldest batch completes before each new one; sample / predict shapes, the use_ucb pattern, PE acquisition = stddev
  of B with a zero penalty, per-metric metadata vectors."""
  from vizier_b200 import optimizers as vb
  from vizier_b200 import vz
  from vizier_b200.designers import gp_ucb_pe
  p = _problem()
  ns = 'gp_ucb_pe_bandit_test'
  iters, batch = 5, 2
  cfg = gp_ucb_pe.UCBPEConfig(
      ucb_coefficient=10.0, explore_region_ucb_coefficient=0.5, cb_violation_penalty_coefficient=0.0,
      ucb_overwrite_probability=0.0, pe_overwrite_probability=0.0, pe_overwrite_probability_in_high_noise=1.0,
      signal_to_noise_threshold=np.inf if high_noise else 0.0,
      multimetric_promising_region_penalty_type=gp_ucb_pe.MultimetricPromisingRegionPenaltyType[penalty])
  fac = vb.VectorizedOptimizerFactory(strategy_factory=vb.VectorizedEagleStrategyFactory(eagle_config=gp_ucb_pe.default_eagle_config),
                                      max_evaluations=500, suggestion_batch_size=25)
  d = gp_ucb_pe.VizierGPUCBPEBandit(p, acquisition_optimizer_factory=fac, metadata_ns=ns, config=cfg, rng=1)
  label_rng = np.random.default_rng(1)
  test_trials = [vz.Trial(parameters={'x0': v, 'x1': 1.0 + 3 * abs(v), 'x2': 0.5}) for v in (-1.0, 0.3, 1.5)]
  active, all_trials, tid = [], [], 1
  last_pred = last_samples = None
  for idx in range(iters + 2):
    sugg = d.suggest(batch)
    assert len(sugg) == batch
    for s in sugg:
      assert p.search_space.contains(s.parameters)
      active.append(s.to_trial(tid)); tid += 1
      all_trials.append(copy.deepcopy(active[-1]))
    done = []
    if 0 < idx < iters:
      for _ in range(batch):
        t = active.pop(0)
        t.complete(vz.Measurement({f'metric{k}': float(label_rng.uniform(-10, 10)) for k in range(2)}))
        done.append(t)
    d.update(vz.CompletedTrials(done), vz.ActiveTrials(active))
    if len(done) > 1:
      samples = d.sample(test_trials, num_samples=5)
      assert samples.shape == (5, 3, 2) and not np.isnan(samples).any()
      other = d.sample(test_trials, num_samples=5, rng=7)
      assert not np.isnan(other).any() and not (np.abs(samples - other) <= 1e-6).all()
      pred = d.predict(test_trials)
      assert pred.mean.shape == (3, 2) and pred.stddev.shape == (3, 2)
      assert not np.isnan(pred.mean).any() and not np.isnan(pred.stddev).any()
      if last_pred is not None:
        assert not (np.abs(last_pred.mean - pred.mean) <= 1e-6).all()
        assert not (np.abs(last_samples - samples) <= 1e-6).all()
      last_pred, last_samples = pred, samples
  assert len(all_trials) == (iters + 2) * batch
  # the second batch (the first is the seeds) comes from pure exploration on active trials only
  for jdx in range(batch, 2 * batch):
    vec, acq, use_ucb = _predictions(all_trials[jdx].metadata.ns(ns))
    assert not use_ucb and acq >= 0.0
    assert all(v.shape == (2,) for v in vec.values())
  n_ucb = n_pe = 0
  for idx in range(2, iters + 2):
    for jdx in range(batch):
      vec, acq, use_ucb = _predictions(all_trials[idx * batch + jdx].metadata.ns(ns))
      assert all(v.shape == (2,) for v in vec.values()), vec
      assert vec['stddev_from_all'][0] == vec['stddev_from_all'][1]
      if jdx == 0 and idx < iters + 1 and not high_noise:
        assert use_ucb
        n_ucb += 1
        continue
      assert not use_ucb
      # zero penalty: the PE acquisition is the stddev of model B (inside the trust region); the metadata vectors
      # carry np.array2string's 8 decimals
      assert acq >= 0.0
      assert abs(acq - vec['stddev_from_all'][0]) <= 1e-8 * max(1.0, acq)
      n_pe += 1
  assert n_pe > 0 and (n_ucb > 0) == (not high_noise)


def test_designer_predicts_each_metric_on_its_own_scale():
  """Each metric has its own output warper: predictions at observed points come back near each metric's labels even
  when the two metrics live on very different scales (the MINIMIZE metric sign-flipped by the converter)."""
  from vizier_b200 import vz
  from vizier_b200.designers import gp_ucb_pe
  p = _problem()
  d = gp_ucb_pe.VizierGPUCBPEBandit(p, rng=4)
  rng = np.random.default_rng(6)

  def f(params):
    x0, x2 = params['x0'].value, params['x2'].value
    return {'metric0': 0.01 * np.sin(x0) + 0.02 * x2, 'metric1': 500.0 + 300.0 * (x0 ** 2 + x2)}

  trials = []
  for i in range(25):
    t = vz.Trial(parameters={'x0': float(rng.uniform(-2, 2)), 'x1': float(rng.uniform(0.1, 10)),
                             'x2': float(rng.uniform())}, id=i + 1)
    t.complete(vz.Measurement({k: float(v) for k, v in f(t.parameters).items()}))
    trials.append(t)
  d.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  pred = d.predict(trials[:6], rng=1, num_samples=500)
  truth = np.array([[f(t.parameters)['metric0'], -f(t.parameters)['metric1']] for t in trials[:6]])
  spread = np.ptp(np.array([[f(t.parameters)['metric0'], f(t.parameters)['metric1']] for t in trials]), axis=0)
  assert pred.mean.shape == (6, 2)
  assert np.all(np.abs(pred.mean - truth) < 0.2 * spread[None, :]), (pred.mean, truth)


def test_designer_two_metrics_with_prior_acquisition():
  """A prior_acquisition on a two-metric study runs through the host-stepped Eagle loop and lands in the metadata."""
  from vizier_b200 import optimizers as vb
  from vizier_b200 import vz
  from vizier_b200.designers import gp_ucb_pe
  p = _problem()
  fac = vb.VectorizedOptimizerFactory(strategy_factory=vb.VectorizedEagleStrategyFactory(eagle_config=gp_ucb_pe.default_eagle_config),
                                      max_evaluations=500, suggestion_batch_size=25)

  def prior(xc, xz):
    return -5.0 * np.sum((xc - 0.8) ** 2, axis=-1)

  d = gp_ucb_pe.VizierGPUCBPEBandit(p, acquisition_optimizer_factory=fac, prior_acquisition=prior, rng=3)
  rng = np.random.default_rng(2)
  trials = []
  for i in range(8):
    t = vz.Trial(parameters={'x0': float(rng.uniform(-2, 2)), 'x1': float(rng.uniform(0.1, 10)),
                             'x2': float(rng.uniform())}, id=i + 1)
    t.complete(vz.Measurement({'metric0': float(rng.normal()), 'metric1': float(rng.normal())}))
    trials.append(t)
  d.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  out = d.suggest(3)
  assert len(out) == 3
  for s in out:
    assert p.search_space.contains(s.parameters)
    md = s.metadata.ns('google_gp_ucb_pe_bandit')
    assert np.isfinite(float(md.ns('prior_acquisition')['value']))
    assert np.asarray(ast.literal_eval(md.ns('prediction_in_warped_y_space')['mean'])).shape == (2,)
