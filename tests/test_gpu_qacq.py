"""Parallel (q-) acquisitions on the device against the oracle: the Monte Carlo kernel on given moments
(`vzgp_qacq_from_moments`), the set scorer on fitted models (`vzgp_score_qsets`: k_qset_moments + k_qacq_mc behind the
general route's K* and W), the set optimisers, and the designer with `scoring_function_is_parallel=True`.

Every case asserts the route it took.  Scores agree with tests/qacq_oracle.py::qacq_score to rtol 1e-9: the oracle
draws the same Philox normals and members and sums the samples in the kernel's order."""
import math

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from oracle import eagle_oracle as eo  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402

import qacq_oracle as qo  # noqa: E402

ROUTE_GENERAL = 4
KINDS = (qo.QACQ_QEI, qo.QACQ_QPI, qo.QACQ_QUCB)


@pytest.fixture(scope='module')
def dev():
  from vizier_b200 import gp
  d = gp.DeviceGP(0)
  yield d
  d.close()


def _spd_moments(rng, e, n, q):
  a = rng.normal(size=(e, n, q, q)) * 0.4
  cov = a @ np.swapaxes(a, -1, -2) + 0.05 * np.eye(q)
  mean = rng.normal(size=(e, n, q)) * 0.5
  return mean, cov


def _qacq(kind, **kw):
  from vizier_b200 import gp
  return gp.QAcquisition(kind, **kw)


# ---------------------------------------------------------------- Monte Carlo stage on given moments
@pytest.mark.parametrize('q', [1, 3, 16])
@pytest.mark.parametrize('s', [1, 100, 5000])
@pytest.mark.parametrize('e', [1, 3])
@pytest.mark.parametrize('kind', KINDS)
def test_from_moments_matches_oracle(dev, q, s, e, kind):
  rng = np.random.default_rng(q * 1000 + s + 7 * e + kind)
  n = 7
  mean, cov = _spd_moments(rng, e, n, q)
  best = 0.2
  got = dev.qacq_from_moments(mean, cov, _qacq(kind, best_label=best, coefficient=1.3, num_samples=s), seed=99,
                              period=3).cpu().numpy()
  want = qo.qacq_from_moments(mean, cov, kind=kind, best_label=best, coefficient=1.3, num_samples=s, seed=99,
                              period=3)[0]
  np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)


@pytest.mark.parametrize('kind', KINDS)
def test_from_moments_jitter_ladder_and_exhaustion(dev, kind):
  retry = np.array([[1.0, 1.0], [1.0, 1.0 - 5e-5]])
  hopeless = np.array([[1.0, 0.0], [0.0, -10.0]])
  cov = np.stack([retry, hopeless, np.eye(2)])[None]
  mean = np.array([[[0.1, 0.2], [0.0, 0.0], [-0.3, 0.4]]])
  qa = _qacq(kind, best_label=0.0, num_samples=300)
  got = dev.qacq_from_moments(mean, cov, qa, seed=5).cpu().numpy()
  want = qo.qacq_from_moments(mean, cov, kind=kind, best_label=0.0, num_samples=300, seed=5)[0]
  assert np.isnan(got[1]) and np.isnan(want[1])
  np.testing.assert_allclose(got[[0, 2]], want[[0, 2]], rtol=0, atol=1e-12)
  # the retried factor is that of Sigma + 1e-4 I: scoring Sigma + 1e-4 I directly gives the same value
  direct = dev.qacq_from_moments(mean[:, :1], (retry + 1e-4 * np.eye(2))[None, None], qa, seed=5, period=3).cpu().numpy()
  np.testing.assert_allclose(direct[0], got[0], rtol=0, atol=1e-12)


def test_from_moments_reference_known_answers(dev):
  """acquisitions_test.py:279-335 on tfd.Normal moments."""
  qei = dev.qacq_from_moments([[[0.1]]], [[[[1.0]]]], _qacq(qo.QACQ_QEI, best_label=0.2, num_samples=5000), seed=0)
  assert abs(float(qei[0]) - 0.346) < 2e-2
  from scipy import stats
  mu, sd, best = np.array([0.3, -0.2, 1.1]), np.array([0.9, 0.5, 0.3]), 0.1
  mean, cov = mu[None, :, None], (sd ** 2)[None, :, None, None]
  qpi = dev.qacq_from_moments(mean, cov, _qacq(qo.QACQ_QPI, best_label=best, num_samples=5000), seed=1).cpu().numpy()
  np.testing.assert_allclose(qpi, stats.norm.cdf((mu - best) / sd), atol=2.5e-2)
  qucb = dev.qacq_from_moments(mean, cov, _qacq(qo.QACQ_QUCB, coefficient=1.8 * math.sqrt(math.pi / 2), num_samples=5000),
                               seed=2, period=1).cpu().numpy()
  np.testing.assert_allclose(qucb, mu + 1.8 * sd, atol=4 * 1.8 * sd.max() * math.sqrt(math.pi / 2 - 1) / math.sqrt(5000))


# ---------------------------------------------------------------- fitted models
def _models(n, d, dk=0, linear=False, e=1, seed=0):
  from vizier_b200 import gp
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, d))
  z = rng.integers(0, 3, size=(n, dk)).astype(np.int32) if dk else None
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n) + (0.1 * z.sum(axis=1) if dk else 0.0)
  devs, preds = [], []
  first = None
  for m in range(e):
    ls2 = 0.5 * (1 + np.arange(d) / d) * (1 + 0.3 * m)
    cls2 = np.full(dk, 0.7 + 0.2 * m) if dk else None
    sf2, sn2 = 1.0 + 0.2 * m, 1e-3 * (1 + m)
    lin = go.LinearParams(0.1, 0.8, 0.2, 0.3) if linear else None
    po = go.GPParams(sf2, ls2, sn2, cls2, linear=lin)
    pg = gp.GPHyperParams(sf2, ls2, sn2, cls2, **(dict(linear_coef=0.1, linear_slope_amplitude=0.8, linear_shift=0.2,
                                                        mean_constant=0.3) if linear else {}))
    dv = gp.DeviceGP(0) if first is None else gp.DeviceGP(0, stream=first.stream)
    first = first or dv
    dv.fit(x, y, pg, z=z)
    devs.append(dv)
    preds.append(go.precompute_predictive(po, x, y, z))
  return devs, preds, x, z


def _score(devs, sets, zsets, qa, seed, period=0, with_cov=True):
  from vizier_b200 import gp
  n, q, d = sets.shape
  out = gp._score_qsets(devs, sets.reshape(n * q, d), q, qa, seed, zs=None if zsets is None else zsets.reshape(n * q, -1),
                        period=period, with_aux=True, with_cov=with_cov)
  devs[0].synchronize()
  for dv in devs:
    assert dv.get_int('score_route') == ROUTE_GENERAL
  return {k: v.cpu().numpy() for k, v in out.items() if k != '_inputs'}


def _check(devs, preds, sets, zsets, kind, *, tr=False, radius=0.35, period=0, seed=17, s=64):
  best = 0.0
  qa = _qacq(kind, best_label=best, coefficient=1.8, num_samples=s, use_trust_region=tr, trust_radius=radius)
  got = _score(devs, sets, zsets, qa, seed, period)
  want, aux = qo.qacq_score(preds, sets, zsets, kind=kind, best_label=best, coefficient=1.8, num_samples=s, seed=seed,
                            period=period, use_trust_region=tr, trust_radius_value=radius)
  np.testing.assert_allclose(got['cov'], aux['cov'], rtol=0, atol=1e-10)
  np.testing.assert_allclose(got['mean'], aux['mean'], rtol=0, atol=1e-10)
  np.testing.assert_allclose(got['stddev'], aux['stddev'], rtol=0, atol=1e-9)
  np.testing.assert_array_equal(got['linf_distance'], aux['linf_distance'])
  np.testing.assert_allclose(got['score'], want, rtol=1e-9, atol=1e-12)
  return got


@pytest.mark.parametrize('n,d,q', [(50, 2, 1), (63, 6, 2), (64, 2, 4), (65, 20, 2), (300, 6, 5), (1000, 2, 16),
                                   (300, 20, 1), (1000, 6, 4)])
@pytest.mark.parametrize('kind', KINDS)
def test_score_qsets_matches_oracle(n, d, q, kind):
  devs, preds, _, _ = _models(n, d, seed=n + d)
  rng = np.random.default_rng(q)
  sets = rng.uniform(size=(11, q, d))
  _check(devs, preds, sets, None, kind)
  for dv in devs:
    dv.close()


@pytest.mark.parametrize('variant', ['categorical', 'linear', 'ensemble', 'trust_region', 'all'])
def test_score_qsets_variants_match_oracle(variant):
  dk = 2 if variant in ('categorical', 'all') else 0
  linear = variant in ('linear', 'all')
  e = 3 if variant in ('ensemble', 'all') else 1
  tr = variant in ('trust_region', 'all')
  devs, preds, x, z = _models(120, 4, dk=dk, linear=linear, e=e, seed=3)
  rng = np.random.default_rng(4)
  q = 4
  sets = rng.uniform(size=(9, q, 4))
  sets[0] = x[:q] + 0.01                      # near the trials: inside the trust region
  zsets = rng.integers(0, 3, size=(9, q, dk)).astype(np.int32) if dk else None
  for kind in KINDS:
    _check(devs, preds, sets, zsets, kind, tr=tr, radius=0.3)
  for dv in devs:
    dv.close()


@pytest.mark.parametrize('q,n_sets', [(5, 819), (5, 830), (3, 1400), (16, 257)])
def test_score_qsets_chunk_edges(q, n_sets):
  """Chunks hold whole sets: q = 5 gives 4095-row chunks; n_sets * q crosses 4096."""
  devs, preds, _, _ = _models(64, 2, seed=q)
  sets = np.random.default_rng(n_sets).uniform(size=(n_sets, q, 2))
  _check(devs, preds, sets, None, qo.QACQ_QEI, period=25, s=16)
  devs[0].close()


def test_score_qsets_duplicate_and_observed_points():
  """A set with a repeated point (a rank-deficient K** block; the noise keeps Sigma definite) and a set of observed
  trials."""
  devs, preds, x, _ = _models(80, 3, seed=8)
  sets = np.stack([np.stack([x[5], x[5], x[7]]), x[:3], np.random.default_rng(1).uniform(size=(3, 3))])
  for kind in KINDS:
    _check(devs, preds, sets, None, kind)
  devs[0].close()


def test_common_random_numbers_and_repeatability():
  devs, _, _, _ = _models(100, 3, seed=9)
  rng = np.random.default_rng(2)
  base = rng.uniform(size=(4, 3, 3))
  sets = np.concatenate([base, base])                # set i and i + 4 share contents
  qa = _qacq(qo.QACQ_QEI, best_label=0.0, num_samples=100)
  a = _score(devs, sets, None, qa, 7, period=4)['score']
  b = _score(devs, sets, None, qa, 7, period=4)['score']
  np.testing.assert_array_equal(a, b)                # bit-identical repeat
  np.testing.assert_array_equal(a[:4], a[4:])        # same position (mod period) -> same draws
  c = _score(devs, sets, None, qa, 7, period=8)['score']
  assert not np.array_equal(c[:4], c[4:])            # other positions -> other draws
  devs[0].close()


# ---------------------------------------------------------------- set optimisers
def test_eagle_qsets_trajectory_matches_oracle():
  """The n_parallel Eagle optimiser through the stepped loop with the q-scorer, against the oracle's optimiser driven
  by qacq_score (same Philox draws for the optimiser and the Monte Carlo)."""
  from vizier_b200 import gp
  from vizier_b200 import _lib
  n, d, q, pool, batch, steps = 40, 3, 4, 50, 25, 8
  devs, preds, x, _ = _models(n, d, seed=21)
  dv = devs[0]
  cfg_o = eo.EagleConfig()
  cfg = _lib.EagleConfig(cfg_o.visibility, cfg_o.gravity, cfg_o.negative_gravity, cfg_o.perturbation,
                         cfg_o.perturbation_lower_bound, cfg_o.penalize_factor, cfg_o.normalization_scale,
                         cfg_o.prior_trials_pool_pct, pool, batch, steps * batch)
  cfg.n_parallel = q
  qa = _qacq(qo.QACQ_QEI, best_label=-0.05, num_samples=50)
  acq_seed = 1234
  score = lambda xs: dv.score_qsets(xs.reshape(-1, d), q, qa, acq_seed, period=batch)['score']
  n_sets = n // q
  prior_sets = x[: n_sets * q].reshape(n_sets, q * d)
  se = gp.SteppedEagle(dv, cfg, 2, 11, n_prior=n_sets)
  se.seed(prior_sets, None, score(torch.from_numpy(prior_sets).cuda()))
  for _ in range(steps):
    xs, _, rewards = se.ask()
    r = score(xs)
    with torch.cuda.stream(dv._stream):
      rewards.copy_(r)
    se.tell()
  bx, _, br = se.end()
  assert dv.get_int('score_route') == ROUTE_GENERAL
  score_fn = lambda s: qo.qacq_score(preds, s, kind=qo.QACQ_QEI, best_label=qa.best_label, num_samples=50,
                                     seed=acq_seed, period=batch)[0]
  wx, wr, _ = eo.run_eagle_optimizer_sets(score_fn, dim=d, n_parallel=q, pool_size=pool, batch_size=batch,
                                          max_evaluations=steps * batch, count=2, seed=11, cfg=cfg_o, prior_features=x)
  np.testing.assert_allclose(br, wr, rtol=1e-8, atol=1e-9)
  np.testing.assert_allclose(bx.reshape(2, q, d), wx, atol=1e-8)
  dv.close()


def test_random_strategy_sets_pick_the_oracle_top_set():
  from vizier_b200 import optimizers as vb
  d, q, batch, max_eval = 3, 2, 25, 400
  devs, preds, _, _ = _models(60, d, seed=31)
  dv = devs[0]
  opt = vb.VectorizedOptimizer(vb.random_strategy_factory, d, 0, batch, max_eval)
  qa = _qacq(qo.QACQ_QUCB, coefficient=1.8, num_samples=40)
  res = opt.optimize_qsets(dv, qa, n_parallel=q, seed=77, acq_seed=5)
  assert dv.get_int('score_route') == ROUTE_GENERAL
  n_sets = max_eval
  pool = eo.philox_uniform(77, eo.STREAM_RANDOM_POOL, 0, n_sets * q * d).reshape(n_sets, q, d)
  want = qo.qacq_score(preds, pool, kind=qo.QACQ_QUCB, coefficient=1.8, num_samples=40, seed=5, period=batch)[0]
  top = int(go.top_k(want, 1)[0])
  np.testing.assert_allclose(res.features, pool[top], atol=0)
  final = qo.qacq_score(preds, pool[top:top + 1], kind=qo.QACQ_QUCB, coefficient=1.8, num_samples=40, seed=5,
                        period=batch)[0]
  np.testing.assert_allclose(res.rewards, np.full(q, final[0]), rtol=1e-9)
  dv.close()


# ---------------------------------------------------------------- designer
def _designer_problem(cat=False):
  from vizier_b200 import vz
  p = vz.ProblemStatement()
  p.search_space.root.add_float_param('x1', 0.0, 1.0)
  p.search_space.root.add_float_param('x2', 0.0, 1.0)
  if cat:
    p.search_space.root.add_categorical_param('c', ['a', 'b', 'c'])
  p.metric_information.append(vz.MetricInformation(name='obj', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  return p


def test_parallel_qei_designer_mirrors_reference_test():
  """gp_bandit_test.py:430-474: QEI (100 samples), n_parallel = 4, no trust region, 4 seed trials, an ensemble of 3,
  linear_coef 0.1, ARD with maxiter 5, the test's 10-evaluation Eagle optimiser: three rounds of suggest(4), each
  completed with random metrics, give 12 trials with valid parameters."""
  from vizier_b200 import acquisitions as acq
  from vizier_b200 import ard
  from vizier_b200 import optimizers as vb
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit
  problem = vz.ProblemStatement()
  problem.search_space.root.add_float_param('lineardouble', -1., 2.)
  problem.search_space.root.add_float_param('logdouble', 1e-4, 1e2, scale_type=vz.ScaleType.LOG)
  problem.metric_information.append(vz.MetricInformation(name='metric', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  designer = gp_bandit.VizierGPBandit(
      problem, scoring_function_factory=acq.bayesian_scoring_function_factory(
          lambda d: acq.QEI(acq.get_best_labels(d.labels), num_samples=100)),
      acquisition_optimizer_factory=vb.VectorizedOptimizerFactory(
          strategy_factory=vb.VectorizedEagleStrategyFactory(), max_evaluations=10),
      scoring_function_is_parallel=True, use_trust_region=False, num_seed_trials=4, ensemble_size=3,
      linear_coef=0.1, ard_optimizer=ard.ScipyLbfgsB(ard.LbfgsBOptions(maxiter=5, num_line_search_steps=5)), rng=0)
  rng = np.random.default_rng(1)
  trials = []
  for _ in range(3):
    sugg = designer.suggest(4)
    assert len(sugg) == 4
    done = []
    for s in sugg:
      assert problem.search_space.contains(s.parameters)
      t = s.to_trial(len(trials) + len(done) + 1)
      t.complete(vz.Measurement({'metric': float(rng.uniform())}))
      done.append(t)
    designer.update(vz.CompletedTrials(done), vz.ActiveTrials())
    trials.extend(done)
  assert len(trials) == 12
  assert all(dv.get_int('score_route') == ROUTE_GENERAL for dv in designer._dev.members)


@pytest.mark.parametrize('factory', ['qucb', 'qpi'])
def test_parallel_designer_with_trust_region(factory):
  import json
  from vizier_b200 import acquisitions as acq
  from vizier_b200 import ard
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit
  fn = (lambda d: acq.QUCB()) if factory == 'qucb' else (lambda d: acq.QPI(acq.get_best_labels(d.labels)))
  designer = gp_bandit.VizierGPBandit(
      _designer_problem(), scoring_function_factory=acq.bayesian_scoring_function_factory(fn),
      scoring_function_is_parallel=True, num_seed_trials=3, ard_optimizer=ard.ScipyLbfgsB(ard.LbfgsBOptions(maxiter=5, num_line_search_steps=5)), rng=3,
      acquisition_optimizer_factory=gp_bandit.vb.VectorizedOptimizerFactory(max_evaluations=2000))
  rng = np.random.default_rng(1)
  done = []
  for i, s in enumerate(designer.suggest(3)):
    t = s.to_trial(i + 1)
    t.complete(vz.Measurement({'obj': float(rng.uniform())}))
    done.append(t)
  designer.update(vz.CompletedTrials(done), vz.ActiveTrials())
  sugg = designer.suggest(3)
  assert len(sugg) == 3
  pts = np.array([[s.parameters['x1'].value, s.parameters['x2'].value] for s in sugg])
  assert ((pts >= 0) & (pts <= 1)).all()
  assert len({tuple(p) for p in pts}) == 3
  values = {json.loads(s.metadata.ns('devinfo')['acquisition_optimization'])['acquisition'] for s in sugg}
  assert len(values) == 1 and np.isfinite(list(values)[0])
  assert designer._dev.get_int('score_route') == ROUTE_GENERAL
  one = designer.suggest(1)
  assert len(one) == 1


def test_parallel_designer_eagle_rejects_categorical_random_accepts():
  from vizier_b200 import acquisitions as acq
  from vizier_b200 import ard
  from vizier_b200 import optimizers as vb
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit
  f = acq.bayesian_scoring_function_factory(lambda d: acq.QEI(acq.get_best_labels(d.labels)))
  rng = np.random.default_rng(2)

  def run(factory):
    designer = gp_bandit.VizierGPBandit(_designer_problem(cat=True), scoring_function_factory=f,
                                        scoring_function_is_parallel=True, num_seed_trials=3, rng=4,
                                        ard_optimizer=ard.ScipyLbfgsB(ard.LbfgsBOptions(maxiter=5, num_line_search_steps=5)), acquisition_optimizer_factory=factory)
    done = []
    for i, s in enumerate(designer.suggest(3)):
      t = s.to_trial(i + 1)
      t.complete(vz.Measurement({'obj': float(rng.uniform())}))
      done.append(t)
    designer.update(vz.CompletedTrials(done), vz.ActiveTrials())
    return designer, designer.suggest(2)

  with pytest.raises(NotImplementedError):
    run(gp_bandit.default_acquisition_optimizer_factory)
  designer, sugg = run(vb.VectorizedOptimizerFactory(strategy_factory=vb.random_strategy_factory, max_evaluations=1000))
  assert len(sugg) == 2 and all(s.parameters['c'].value in ('a', 'b', 'c') for s in sugg)
  assert designer._dev.get_int('score_route') == ROUTE_GENERAL
