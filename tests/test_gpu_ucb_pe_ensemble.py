"""GP-UCB-PE over uniform ensembles on the GPU against the tests-side oracle (pe_ensemble_oracle.py):
vzgp_score_pe_ensemble on every scoring route, the cooperative and replayed-graph Eagle loops, the host-stepped loop,
the designer's model B and threshold, and VizierGPUCBPEBandit(ensemble_size=3) end to end (gp_ucb_pe_test.py:63,
:88-95)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from oracle import eagle_oracle as eo  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402
import pe_ensemble_oracle as peo  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, 'tests')
SMALL, SPLIT, CLUSTER, GENERAL = 0, 1, 2, 4   # vzgp_score_route
COOPERATIVE, GRAPH = 1, 2                     # vzgp_eagle_route


def _params(e, d, dk, linear, high_noise_b=False):
  """Member e's hyper-parameters as (oracle, device) pairs; distinct members so their means spread."""
  from vizier_b200 import gp
  out = []
  for k in range(e):
    sf2, sn2 = 1.0 + 0.3 * k, 1e-3 * (1 + k)
    ls2 = 0.4 * (1 + np.arange(d) / d) * (1 + 0.25 * k)
    lk = np.linspace(0.7, 1.3, dk) * (1 + 0.1 * k) if dk else None
    if high_noise_b:
      sn2 = 1e-10
    if linear:
      lp = (1.0, 0.6 + 0.1 * k, 0.2, 0.1 * k)
      out.append((go.GPParams(sf2, ls2, sn2, lk, go.LinearParams(*lp)),
                  gp.GPHyperParams(sf2, ls2, sn2, lk, linear_coef=lp[0], linear_slope_amplitude=lp[1],
                                   linear_shift=lp[2], mean_constant=lp[3])))
    else:
      out.append((go.GPParams(sf2, ls2, sn2, lk), gp.GPHyperParams(sf2, ls2, sn2, lk)))
  return out


def _models(n, n_pending, d, dk, e, seed, linear=False, high_noise=False):
  """E members of A on n trials and of B on n + n_pending trials (real labels, then 0; noise 1e-10 in high-noise
  mode): oracle predictives and two EnsembleGPs on one stream."""
  from vizier_b200 import gp
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, d))
  z = rng.integers(0, 3, size=(n, dk)).astype(np.int32) if dk else None
  y = np.sin(3 * x[:, 0]) - np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  xb = np.concatenate([x, rng.uniform(size=(n_pending, d))])
  xb[n:n + 1] = 1.3                  # a pending trial far from the completed ones
  zb = np.concatenate([z, rng.integers(0, 3, size=(n_pending, dk)).astype(np.int32)]) if dk else None
  yb = np.concatenate([y, np.zeros(n_pending)])
  pa, pb = _params(e, d, dk, linear), _params(e, d, dk, linear, high_noise)
  pred_a = [go.precompute_predictive(po, x, y, z) for po, _ in pa]
  pred_b = [go.precompute_predictive(po, xb, yb, zb) for po, _ in pb]
  dev_a = gp.EnsembleGP(0, e)
  dev_b = gp.EnsembleGP(0, e, stream=dev_a.stream)
  for h in dev_a.members + dev_b.members:
    h.set_int('score_i8', 0)
    h.set_int('small_tiles', -1)
  assert dev_a.fit(x, y, [p for _, p in pa], z=z) == 0
  assert dev_b.fit(xb, yb, [p for _, p in pb], z=zb) == 0
  return rng, x, z, y, xb, pred_a, pred_b, dev_a, dev_b


def _route(sm, m, n):
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


# route, n, n_pending, d, dk, E, candidates (a callable of the SM count), linear kernel, high-noise mode
CASES = [
    pytest.param(SMALL, 40, 5, 3, 1, 2, lambda sm: 300, False, False, id='small-e2-cat'),
    pytest.param(SMALL, 50, 0, 3, 0, 3, lambda sm: 200, False, True, id='small-e3-highnoise-nopending'),
    pytest.param(SPLIT, 300, 8, 4, 0, 3, lambda sm: 20 * 64 - 11, False, True, id='split-e3-highnoise'),
    pytest.param(CLUSTER, 150, 10, 5, 2, 5, lambda sm: (sm // 2 + 1) * 64 + 9, False, False, id='cluster-e5-cat'),
    pytest.param(GENERAL, 60, 4, 3, 0, 3, lambda sm: 500, True, False, id='general-e3-linear'),
]


@pytest.mark.parametrize('route,n,n_pending,d,dk,e,count,linear,high_noise', CASES)
def test_score_pe_ensemble_matches_oracle(route, n, n_pending, d, dk, e, count, linear, high_noise):
  from vizier_b200 import gp
  rng, x, z, y, xb, pred_a, pred_b, dev_a, dev_b = _models(n, n_pending, d, dk, e, 7 + e, linear, high_noise)
  try:
    sm = dev_a.members[0].get_int('sm_count')
    mc = count(sm)
    xs = rng.uniform(-1.0, 2.0, size=(mc, d))   # many candidates far from every trial: the region must bite
    xs[:5] = x[:5]                     # at trials: model B's stddev is tiny in high-noise mode
    xs[5:5 + n_pending] = xb[n:] + 0.01   # next to pending trials: inside B's trust region, not all inside A's
    zs = rng.integers(0, 3, size=(mc, dk)).astype(np.int32) if dk else None
    if dk:
      zs[5:5 + n_pending] = np.concatenate([z, np.zeros((n_pending, dk), np.int32)])[n:] if n_pending else zs[5:5]
    thr = peo.ucb_threshold(pred_a, pred_b)
    mask = np.ones(d, bool); mask[d - 1] = False
    tr_rows = n + n_pending
    dist = go.min_linf_distance(xs, xb[:tr_rows], mask)
    # a radius equal to one candidate's distance: the strict region leaves that candidate out
    edge = int(np.argmax(np.where((dist > 0.1) & (dist < 0.45), 1, 0)))
    assert 0.1 < dist[edge] < 0.45
    seen_tr = False
    for use_tr, radius in ((False, 1.0), (True, 0.2), (True, float(dist[edge])), (True, 0.7)):
      for mode in (0, 1):
        pe = gp.UcbPeAcquisition(mode=mode, threshold=thr, use_trust_region=use_tr, trust_radius=radius,
                                 tr_dim_mask=mask, tr_rows=tr_rows)
        out = dev_a.score_pe(dev_b, xs, pe, zs=zs)
        for h in dev_a.members:
          assert h.get_int('score_route') == (GENERAL if linear else _route(sm, mc, n)) == route
        for h in dev_b.members:
          assert h.get_int('score_route') == (GENERAL if linear else _route(sm, mc, n + n_pending))
        want, aux = peo.ucb_pe_ensemble_score(pred_a, pred_b, xs, zs, mode=mode, threshold=thr, tr_dim_mask=mask,
                                              tr_rows=tr_rows, trust_radius_value=radius, use_trust_region=use_tr)
        _close(out['mean'].cpu().numpy(), aux['mean'])
        _close(out['stddev'].cpu().numpy(), aux['stddev'])
        _close(out['stddev_from_all'].cpu().numpy(), aux['stddev_from_all'])
        _close(out['score'].cpu().numpy(), want)
        if use_tr and radius <= 0.5:
          assert np.any(want < -1e3) and np.any(want > -1e3)
          if n_pending and radius == 0.2:   # next to the far pending trial: inside B's region only
            assert want[5] > -1e3 and go.min_linf_distance(xs[5:6], x, mask)[0] > radius
          if radius == dist[edge]:
            assert want[edge] < -1e3
          seen_tr = True
    assert seen_tr
    # the mixture of the device's own member moments, at full relative precision: in high-noise mode B's stddev at
    # the trials is ~1e-5 while |mean| ~ 1, where a one-pass variance loses about six digits
    pe = gp.UcbPeAcquisition(mode=0, use_trust_region=False)
    out = dev_a.score_pe(dev_b, xs, pe, zs=zs)
    mus, sds = [], []
    for h in dev_b.members:      # the kernel variant score_pe runs: no distance output
      o = {k: torch.empty(mc, dtype=torch.float64, device=h.device) for k in ('score', 'mean', 'stddev')}
      torch.cuda.synchronize()
      h.score(xs, gp.Acquisition(0.0, False, 1.0), zs=zs, out=o)
      h.synchronize()
      mus.append(o['mean'].cpu().numpy()); sds.append(o['stddev'].cpu().numpy())
    _, sd_mix = peo.mixture(np.stack(mus), np.stack(sds))
    got = out['stddev_from_all'].cpu().numpy()
    assert np.max(np.abs(got - sd_mix) / sd_mix) < 1e-12
    if high_noise:
      assert np.min(sd_mix[:5]) < 1e-3
    # repeated calls are bit-identical
    again = dev_a.score_pe(dev_b, xs, pe, zs=zs)
    assert torch.equal(again['score'], out['score']) and torch.equal(again['stddev_from_all'], out['stddev_from_all'])
  finally:
    dev_b.close(); dev_a.close()


@pytest.mark.parametrize('route,m', [(SMALL, 300), (CLUSTER, 20000)])
def test_single_member_matches_score_pe(route, m):
  """E = 1 through the ensemble entry computes what vzgp_score_pe computes."""
  from vizier_b200 import gp
  rng, x, z, y, xb, pred_a, pred_b, dev_a, dev_b = _models(120, 6, 4, 1, 1, 3)
  try:
    xs = rng.uniform(size=(m, 4))
    zs = rng.integers(0, 3, size=(m, 1)).astype(np.int32)
    for mode, radius in ((0, 0.3), (1, 0.3), (1, 0.8)):
      pe = gp.UcbPeAcquisition(mode=mode, threshold=0.2, trust_radius=radius, tr_rows=123)
      got = dev_a.score_pe(dev_b, xs, pe, zs=zs)
      want = dev_a.members[0].score_pe(dev_b.members[0], xs, pe, zs=zs)
      for k in ('score', 'mean', 'stddev', 'stddev_from_all'):
        g, w = got[k].cpu().numpy(), want[k].cpu().numpy()
        assert np.all(np.abs(g - w) <= 1e-15 * np.abs(w)), k
  finally:
    dev_b.close(); dev_a.close()


def test_entry_point_checks():
  from vizier_b200 import _lib
  from vizier_b200 import gp
  _, x, z, y, xb, _, _, dev_a, dev_b = _models(30, 2, 2, 0, 2, 5)
  other = gp.EnsembleGP(0, 2)                          # its own stream
  lone = gp.EnsembleGP(0, 2, stream=dev_a.stream)      # never fitted
  try:
    pe = gp.UcbPeAcquisition()
    with pytest.raises(_lib.VzgpError, match='stream'):
      other.fit(x, y, [p for _, p in _params(2, 2, 0, False)])
      dev_a.score_pe(other, x, pe)
    with pytest.raises(_lib.VzgpError) as err:
      dev_a.score_pe(lone, x, pe)
    assert err.value.status == _lib.VZGP_ERR_STATE
    lone.fit(x[:20], y[:20], [p for _, p in _params(2, 2, 0, False)])
    lone.members[1].fit(x, y, _params(2, 2, 0, False)[1][1])
    with pytest.raises(_lib.VzgpError, match='same trials'):
      dev_a.score_pe(lone, x, pe)
  finally:
    for g in (lone, other, dev_b, dev_a):
      g.close()


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


# n, n_pending, d, dk, E, high-noise mode
EAGLE_CASES = [(40, 3, 3, 0, 2, False), (150, 5, 4, 1, 3, True), (90, 4, 3, 0, 7, False), (90, 4, 3, 0, 8, False)]


def eagle_case(n, n_pending, d, dk, e, high_noise):
  """Runs one Eagle case against the oracle optimiser; returns the route the device took."""
  from vizier_b200 import gp
  _, x, z, y, xb, pred_a, pred_b, dev_a, dev_b = _models(n, n_pending, d, dk, e, 21 + e, False, high_noise)
  try:
    mask = np.ones(d, bool)
    rows = n + n_pending
    radius = go.trust_radius(rows, d, dk)
    thr = peo.ucb_threshold(pred_a, pred_b)
    pool, batch, steps = 25, 25, 7
    cfg_o, cfg = _eagle_cfgs(pool, batch, steps)
    sizes = np.full(dk, 3, int)
    zp = z if dk else np.zeros((n, 0), np.int32)
    routes = set()
    for mode in (0, 1):
      def score_fn(xc, xz, mode=mode):
        return peo.ucb_pe_ensemble_score(pred_a, pred_b, xc, xz if dk else None, mode=mode, threshold=thr,
                                         tr_dim_mask=mask, tr_rows=rows, trust_radius_value=radius)[0]
      wc, wz, wr = eo.run_eagle_optimizer_mixed(score_fn, dim=d, sizes=sizes, pool_size=pool, batch_size=batch,
                                                max_evaluations=steps * batch, count=2, seed=13, cfg=cfg_o, prior_c=x,
                                                prior_z=zp)
      pe = gp.UcbPeAcquisition(mode=mode, threshold=thr, trust_radius=radius, tr_dim_mask=mask)
      bx, bz, br = dev_a.eagle_run(cfg, pe, 2, 13, prior=x, prior_z=z, cat_sizes=list(sizes), other=dev_b)
      np.testing.assert_allclose(br, wr, atol=1e-9 * max(1.0, np.max(np.abs(wr))), rtol=0)
      np.testing.assert_allclose(bx, wc, atol=1e-9, rtol=0)
      if dk:
        np.testing.assert_array_equal(bz, wz)
      routes.add(dev_a.members[0].get_int('eagle_route'))
    assert len(routes) == 1
    return routes.pop()
  finally:
    dev_b.close(); dev_a.close()


@pytest.mark.parametrize('case', EAGLE_CASES, ids=lambda c: f'n{c[0]}-e{c[4]}')
def test_eagle_run_pe_ensemble_cooperative_matches_oracle(case):
  """The cooperative form for E <= 7; E = 8 exceeds its kernel-parameter budget and replays the graph."""
  assert eagle_case(*case) == (COOPERATIVE if case[4] <= 7 else GRAPH)


_CHILD = """
import json, sys
import test_gpu_ucb_pe_ensemble as t
print('RESULT ' + json.dumps([t.eagle_case(*c) for c in json.loads(sys.argv[1])]))
"""


def test_eagle_run_pe_ensemble_graph_form_matches_oracle():
  """VZGP_EAGLE_GRID=0 (read once per process, so in a child): the replayed-graph form."""
  env = dict(os.environ)
  env['VZGP_EAGLE_GRID'] = '0'
  env['PYTHONPATH'] = os.pathsep.join([ROOT, TESTS] + ([env['PYTHONPATH']] if env.get('PYTHONPATH') else []))
  cases = EAGLE_CASES[:2]
  proc = subprocess.run([sys.executable, '-c', _CHILD, json.dumps(cases)], cwd=ROOT, env=env, capture_output=True,
                        text=True, timeout=900)
  assert proc.returncode == 0, proc.stderr[-4000:]
  line = [ln for ln in proc.stdout.splitlines() if ln.startswith('RESULT ')][-1]
  assert json.loads(line[len('RESULT '):]) == [GRAPH] * len(cases)


def test_stepped_loop_with_zero_prior_equals_device_loop():
  """VectorizedOptimizer with a zero prior_acquisition (host-stepped loop, vzgp_score_pe_ensemble per batch) finds what
  the device loop finds."""
  from vizier_b200 import gp
  from vizier_b200 import optimizers as vb
  from vizier_b200.designers import gp_ucb_pe
  n, n_pending, d, dk, e = 60, 4, 3, 1, 3
  _, x, z, y, xb, pred_a, pred_b, dev_a, dev_b = _models(n, n_pending, d, dk, e, 31)
  try:
    opt = vb.VectorizedOptimizer(vb.VectorizedEagleStrategyFactory(eagle_config=gp_ucb_pe.default_eagle_config), d, dk,
                                 25, 1000, (3,))
    calls = []

    def zero(xc, xz):
      calls.append(xc.shape[0])
      return np.zeros(xc.shape[0])

    for mode in (0, 1):
      pe = gp.UcbPeAcquisition(mode=mode, threshold=0.1, trust_radius=0.3, tr_dim_mask=np.ones(d, bool),
                               tr_rows=n + n_pending)
      dev = opt(dev_a, pe, count=2, prior_features=x, prior_categorical=z, seed=5, other=dev_b)
      host = opt(dev_a, pe, count=2, prior_features=x, prior_categorical=z, seed=5, other=dev_b, prior_acquisition=zero)
      np.testing.assert_allclose(host.rewards, dev.rewards, rtol=0, atol=1e-12)
      np.testing.assert_allclose(host.features, dev.features, rtol=0, atol=1e-12)
      np.testing.assert_array_equal(host.categorical, dev.categorical)
      np.testing.assert_array_equal(host.aux['prior_acq_values'], np.zeros(2))
    assert calls
  finally:
    dev_b.close(); dev_a.close()


def _data(n, n_pending, d, seed):
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, d))
  y = np.sin(3 * x[:, 0]) - np.sum((x - 0.3) ** 2, axis=1)
  return x, y, rng.uniform(size=(n_pending, d))


def test_designer_model_b_and_threshold_match_oracle():
  """The designer fits model B's members on completed + pending trials with the real labels then 0, and takes the
  UCB threshold on the mixture of A's members."""
  from vizier_b200.designers import gp_ucb_pe
  d = gp_ucb_pe.VizierGPUCBPEBandit(_problem(), ensemble_size=3, rng=1)
  n, n_pending, dd = 30, 4, 3
  x, y, pend = _data(n, n_pending, dd, 8)
  pairs = _params(3, dd, 0, False)
  params = [p for _, p in pairs]
  dev_a, dev_b = d._devices()
  dev_a.fit(x, y, params)
  xc_all, _ = d._fit_all_features(params, x, np.zeros((n, 0), np.int32), y[:, None], pend,
                                  np.zeros((n_pending, 0), np.int32), False)
  pred_a = [go.precompute_predictive(po, x, y) for po, _ in pairs]
  pred_b = [go.precompute_predictive(po, xc_all, np.concatenate([y, np.zeros(n_pending)])) for po, _ in pairs]
  xs = np.random.default_rng(2).uniform(size=(200, dd))
  from vizier_b200 import gp
  out = dev_a.score_pe(dev_b, xs, gp.UcbPeAcquisition(mode=0, use_trust_region=False))
  _, aux = peo.ucb_pe_ensemble_score(pred_a, pred_b, xs, mode=0, use_trust_region=False)
  _close(out['stddev_from_all'].cpu().numpy(), aux['stddev_from_all'])
  want = peo.ucb_threshold(pred_a, pred_b)
  assert abs(d._ucb_threshold(xc_all, None) - want) <= 1e-10 * max(1.0, abs(want))
  # member 0's threshold differs here: the test can tell the mixture from one member
  assert abs(go.ucb_threshold(pred_a[0], pred_b[0]) - want) > 1e-6


def _problem(linear_cat=False):
  from vizier_b200 import vz
  p = vz.ProblemStatement()
  p.search_space.root.add_float_param('x0', -2.0, 2.0)
  p.search_space.root.add_float_param('x1', 0.1, 10.0, scale_type=vz.ScaleType.LOG)
  p.search_space.root.add_float_param('x2', 0.0, 1.0)
  if linear_cat:
    p.search_space.root.add_categorical_param('c0', ['a', 'b', 'c'])
  p.metric_information.append(vz.MetricInformation(name='metric', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  return p


def _factory():
  from vizier_b200 import optimizers as vb
  from vizier_b200.designers import gp_ucb_pe
  return vb.VectorizedOptimizerFactory(strategy_factory=vb.VectorizedEagleStrategyFactory(
      eagle_config=gp_ucb_pe.default_eagle_config), max_evaluations=500, suggestion_batch_size=25)


@pytest.mark.parametrize('high_noise', [False, True])
def test_designer_ensemble_like_the_reference_test(high_noise):
  """gp_ucb_pe_test.py:63 and :88-95 with ensemble_size 3: batches on active trials, then completions; UCB
  acquisition = mean + 10 stddev_from_all, PE acquisition = stddev_from_all (zero penalty); sample / predict shapes, no
  NaN, and they change as trials complete."""
  from vizier_b200 import vz
  from vizier_b200.designers import gp_ucb_pe
  p = _problem()
  ns = 'gp_ucb_pe_bandit_test'
  iters, batch = 4, 2
  cfg = gp_ucb_pe.UCBPEConfig(
      ucb_coefficient=10.0, explore_region_ucb_coefficient=0.5, cb_violation_penalty_coefficient=0.0,
      ucb_overwrite_probability=0.0, pe_overwrite_probability=0.0, pe_overwrite_probability_in_high_noise=1.0,
      signal_to_noise_threshold=np.inf if high_noise else 0.0)
  d = gp_ucb_pe.VizierGPUCBPEBandit(p, acquisition_optimizer_factory=_factory(), metadata_ns=ns, config=cfg, rng=1,
                                    ensemble_size=3)
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
      all_trials.append(active[-1])
    done = []
    if 0 < idx < iters:
      for _ in range(batch):
        t = active.pop(0)
        t.complete(vz.Measurement({'metric': float(label_rng.uniform(-10, 10))}))
        done.append(t)
    d.update(vz.CompletedTrials(done), vz.ActiveTrials(active))
    if len(d._all_completed_trials) > 1:
      samples = d.sample(test_trials, num_samples=5)
      assert samples.shape == (5, 3) and not np.isnan(samples).any()
      other = d.sample(test_trials, num_samples=5, rng=7)
      assert not np.isnan(other).any() and not (np.abs(samples - other) <= 1e-6).all()
      pred = d.predict(test_trials)
      assert pred.mean.shape == (3,) and pred.stddev.shape == (3,)
      assert not np.isnan(pred.mean).any() and not np.isnan(pred.stddev).any()
      if last_pred is not None and done:
        assert not (np.abs(last_pred.mean - pred.mean) <= 1e-6).all()
        assert not (np.abs(last_samples - samples) <= 1e-6).all()
      last_pred, last_samples = pred, samples
  n_ucb = n_pe = 0
  for t in all_trials[batch:]:
    md = t.metadata.ns(ns)
    pred = md.ns('prediction_in_warped_y_space')
    mean, sda, acq = (float(pred[k]) for k in ('mean', 'stddev_from_all', 'acquisition'))
    assert pred['params'].count('GPHyperParams(') == 3
    if pred['use_ucb'] == 'True':
      assert abs(mean + 10.0 * sda - acq) <= 1e-6 * max(1.0, abs(acq))
      n_ucb += 1
    else:
      assert acq >= 0.0 and abs(acq - sda) <= 1e-6 * max(1.0, acq)
      n_pe += 1
  assert n_pe > 0 and (n_ucb > 0) == (not high_noise)


@pytest.mark.parametrize('kind', ['linear', 'categorical', 'prior_acquisition'])
def test_designer_ensemble_variants(kind):
  """One suggest each with the Matern + linear kernel (general route members), a categorical feature, and a
  prior_acquisition (host-stepped loop)."""
  from vizier_b200 import vz
  from vizier_b200.designers import gp_ucb_pe
  p = _problem(linear_cat=kind == 'categorical')
  kw = {}
  if kind == 'linear':
    kw['mixes_linear_kernel'] = True
  if kind == 'prior_acquisition':
    kw['prior_acquisition'] = lambda xc, xz: -5.0 * np.sum((xc - 0.8) ** 2, axis=-1)
  d = gp_ucb_pe.VizierGPUCBPEBandit(p, acquisition_optimizer_factory=_factory(), ensemble_size=3, rng=3, **kw)
  rng = np.random.default_rng(2)
  trials = []
  for i in range(10):
    params = {'x0': float(rng.uniform(-2, 2)), 'x1': float(rng.uniform(0.1, 10)), 'x2': float(rng.uniform())}
    if kind == 'categorical':
      params['c0'] = ['a', 'b', 'c'][i % 3]
    t = vz.Trial(parameters=params, id=i + 1)
    t.complete(vz.Measurement({'metric': float(rng.normal())}))
    trials.append(t)
  d.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  out = d.suggest(2)
  assert len(out) == 2
  for s in out:
    assert p.search_space.contains(s.parameters)
    md = s.metadata.ns('google_gp_ucb_pe_bandit')
    pred = md.ns('prediction_in_warped_y_space')
    assert all(np.isfinite(float(pred[k])) for k in ('mean', 'stddev', 'stddev_from_all', 'acquisition'))
    if kind == 'prior_acquisition':
      assert np.isfinite(float(md.ns('prior_acquisition')['value']))
  assert d.sample(trials[:3], num_samples=4).shape == (4, 3)


def test_designer_ensemble_prior_only_suggestions():
  """Only active trials: the mixture stddev of B's members on zero labels is maximised; the metadata stddev is the
  mixture prior sqrt(mean_e(sf2_e + sn2_e)) of the first E initial points."""
  from vizier_b200 import vz
  from vizier_b200.designers import gp_ucb_pe
  p = _problem()
  d = gp_ucb_pe.VizierGPUCBPEBandit(p, acquisition_optimizer_factory=_factory(), ensemble_size=3, rng=5)
  active = [s.to_trial(i + 1) for i, s in enumerate(d.suggest(2))]       # seeds
  d.update(vz.CompletedTrials(), vz.ActiveTrials(active))
  seen = []
  fit = d._build_gp_model_and_optimize_parameters
  d._build_gp_model_and_optimize_parameters = lambda *a: seen.append(fit(*a)) or seen[-1]
  out = d.suggest(2)
  params = seen[-1]
  assert isinstance(params, list) and len(params) == 3
  want_sd = float(np.sqrt(np.mean([q.signal_variance + q.observation_noise_variance for q in params])))
  for s in out:
    assert p.search_space.contains(s.parameters)
    pred = s.metadata.ns('google_gp_ucb_pe_bandit').ns('prediction_in_warped_y_space')
    assert float(pred['mean']) == 0.0
    assert abs(float(pred['stddev']) - want_sd) <= 1e-12 * want_sd
    assert float(pred['stddev_from_all']) > 0.0


def test_set_pe_with_an_ensemble_raises():
  from vizier_b200 import vz
  from vizier_b200.designers import gp_ucb_pe
  d = gp_ucb_pe.VizierGPUCBPEBandit(_problem(), acquisition_optimizer_factory=_factory(), ensemble_size=2, rng=1,
                                    config=gp_ucb_pe.UCBPEConfig(optimize_set_acquisition_for_exploration=True))
  rng = np.random.default_rng(3)
  trials = []
  for i in range(6):
    t = vz.Trial(parameters={'x0': float(rng.uniform(-2, 2)), 'x1': 1.0, 'x2': float(rng.uniform())}, id=i + 1)
    t.complete(vz.Measurement({'metric': float(rng.normal())}))
    trials.append(t)
  d.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  with pytest.raises(ValueError, match='ensemble'):
    d.suggest(3)
  assert len(d.suggest(1)) == 1        # one suggestion at a time does not take the set path
