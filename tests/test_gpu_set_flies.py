"""Set flies of up to 1024 coordinates in the Eagle optimiser (n_parallel = q points of Dc continuous features).

k_eagle_suggest_wide walks a fly in 64-column chunks.  These tests hold it to the oracle's set optimiser at widths that end
a chunk early (80, 66), fill chunks exactly (128, 1024) and take many chunks (640), in MEAN and RANDOM normalisation,
with and without prior sets, at pool sizes 50, 100 and 3000; they drive the q-acquisitions through optimize_qsets,
both designers at 20 dimensions, and require flies of at most 64 coordinates to reproduce, bit for bit, the runs
recorded by tools/make_set_flies_golden.py before wide flies existed."""
import dataclasses
import importlib.util
import json
import os

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from oracle import eagle_oracle as eo  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402

import qacq_oracle as qo  # noqa: E402
import set_flies_oracle as so  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEPPED = 3     # vzgp_eagle_route
BATCH = 25


def _config(cfg_o, pool, steps, q):
  from vizier_b200 import _lib
  return _lib.EagleConfig(cfg_o.visibility, cfg_o.gravity, cfg_o.negative_gravity, cfg_o.perturbation,
                          cfg_o.perturbation_lower_bound, cfg_o.penalize_factor, cfg_o.normalization_scale,
                          cfg_o.prior_trials_pool_pct, pool, BATCH, steps * BATCH, cfg_o.categorical_perturbation_factor,
                          cfg_o.pure_categorical_perturbation_factor, cfg_o.prob_same_category_without_perturbation,
                          cfg_o.mutate_normalization_type, q)


def _run_stepped(dev, cfg, count, seed, score, prior_sets=None):
  from vizier_b200 import gp
  se = gp.SteppedEagle(dev, cfg, count, seed, n_prior=0 if prior_sets is None else len(prior_sets))
  assert dev.get_int('eagle_route') == STEPPED
  if prior_sets is not None:
    se.seed(prior_sets, None, score(torch.from_numpy(prior_sets).cuda()))
  for _ in range((cfg.max_evaluations - 1) // cfg.batch_size + 1):
    xs, _, rewards = se.ask()
    r = score(xs)
    with torch.cuda.stream(dev.stream):
      rewards.copy_(r)
    se.tell()
  return se.end()


# ---------------------------------------------------------------------------------------------------------------------
# 1. set-PE trajectories against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class SetCase:
  name: str
  dc: int
  q: int
  pool: int
  norm: int               # mutate_normalization_type
  prior: bool
  extra_steps: int = 6    # steps after the pool's first pass

  @property
  def steps(self):
    return self.pool // BATCH + self.extra_steps


SET_CASES = [
    SetCase('w80-mean-prior', 20, 4, 50, 0, True),
    SetCase('w80-random', 20, 4, 100, 1, False),
    SetCase('w66-random-prior', 33, 2, 50, 1, True),
    SetCase('w66-mean', 33, 2, 100, 0, False),
    SetCase('w128-mean', 64, 2, 100, 0, False),
    SetCase('w128-random-prior', 64, 2, 50, 1, True),
    SetCase('w640-mean-prior', 40, 16, 50, 0, True),
    SetCase('w640-random', 40, 16, 100, 1, False),
    SetCase('w1024-random-prior', 64, 16, 50, 1, True),
    SetCase('w1024-mean', 64, 16, 100, 0, False),
    SetCase('w1024-P3000', 64, 16, 3000, 0, False, extra_steps=3),
]


def _two_models(d, n_done=50, n_pend=4, seed=5):
  from vizier_b200 import gp
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n_done + n_pend, d))
  y = -np.sum((x[:n_done] - 0.3) ** 2, axis=1) / d + 0.05 * rng.normal(size=n_done)
  ls2 = 0.3 * d * (1 + np.arange(d) / d) / 4
  po, pg = go.GPParams(1.1, ls2, 1e-3), gp.GPHyperParams(1.1, ls2, 1e-3)
  pred_a = go.precompute_predictive(po, x[:n_done], y)
  pred_b = go.precompute_predictive(po, x, np.r_[y, np.zeros(n_pend)])
  dev_a = gp.DeviceGP(0)
  dev_b = gp.DeviceGP(0, stream=dev_a.stream)     # vzgp_score_set_pe needs both models on one stream
  dev_a.fit(x[:n_done], y, pg)
  dev_b.fit(x, np.r_[y, np.zeros(n_pend)], pg)
  return x, pred_a, pred_b, dev_a, dev_b


@pytest.mark.parametrize('c', SET_CASES, ids=lambda c: c.name)
def test_set_pe_trajectory_matches_oracle(c):
  from vizier_b200 import gp
  n_done, n_pend = 50, 4
  x, pred_a, pred_b, dev_a, dev_b = _two_models(c.dc, n_done, n_pend)
  try:
    kw = dict(explore_coefficient=0.5, penalty_coefficient=10.0, threshold=-0.1)
    pe = gp.UcbPeAcquisition(mode=1, use_trust_region=True, trust_radius=0.45, tr_rows=n_done + n_pend, **kw)
    cfg_o = eo.EagleConfig(mutate_normalization_type=c.norm)
    n_sets = n_done // c.q
    prior_sets = x[: n_sets * c.q].reshape(n_sets, c.q * c.dc) if c.prior else None
    score = lambda xs: dev_a.score_set_pe(dev_b, xs.reshape(-1, c.dc), c.q, pe)['score']
    bx, _, br = _run_stepped(dev_a, _config(cfg_o, c.pool, c.steps, c.q), 2, 11, score, prior_sets)
    score_fn = lambda s: go.set_pe_score(pred_a, pred_b, s, tr_rows=n_done + n_pend, trust_radius_value=0.45, **kw)[0]
    wx, wr = so.run_sets(score_fn, dim=c.dc, n_parallel=c.q, pool_size=c.pool, batch_size=BATCH,
                         max_evaluations=c.steps * BATCH, count=2, seed=11, cfg=cfg_o,
                         prior_features=x[:n_done] if c.prior else None)
    assert np.all(np.isfinite(wr))
    np.testing.assert_allclose(br, wr, rtol=1e-8, atol=1e-6)
    np.testing.assert_allclose(bx.reshape(2, c.q, c.dc), wx, atol=1e-8)
  finally:
    dev_a.close()
    dev_b.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. q-acquisitions through optimize_qsets
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dc,q', [(20, 4), (64, 16)])
@pytest.mark.parametrize('kind', [qo.QACQ_QEI, qo.QACQ_QUCB])
def test_optimize_qsets_wide_sets_match_oracle(dc, q, kind):
  from vizier_b200 import gp
  from vizier_b200 import optimizers as vb
  n, max_eval, seed, acq_seed = 60, 250, 21, 1234
  rng = np.random.default_rng(dc + q)
  x = rng.uniform(size=(n, dc))
  y = -np.sum((x - 0.3) ** 2, axis=1) / dc + 0.05 * rng.normal(size=n)
  ls2 = 0.3 * dc * (1 + np.arange(dc) / dc) / 4
  pred = go.precompute_predictive(go.GPParams(1.0, ls2, 1e-3), x, y)
  dev = gp.DeviceGP(0)
  try:
    dev.fit(x, y, gp.GPHyperParams(1.0, ls2, 1e-3))
    qa = gp.QAcquisition(kind, best_label=float(np.max(y)), coefficient=1.8, num_samples=50)
    opt = vb.VectorizedOptimizer(vb.VectorizedEagleStrategyFactory(), dc, 0, BATCH, max_eval)
    res = opt.optimize_qsets(dev, qa, n_parallel=q, prior_features=x, seed=seed, acq_seed=acq_seed)
    assert dev.get_int('eagle_route') == STEPPED
    pool = vb.VectorizedEagleStrategyFactory().pool_size(dc, BATCH)
    score_fn = lambda s: qo.qacq_score([pred], s, kind=kind, best_label=qa.best_label, coefficient=1.8, num_samples=50,
                                       seed=acq_seed, period=BATCH)[0]
    wx, _, _ = eo.run_eagle_optimizer_sets(score_fn, dim=dc, n_parallel=q, pool_size=pool, batch_size=BATCH,
                                           max_evaluations=max_eval, count=1, seed=seed, cfg=eo.EagleConfig(),
                                           prior_features=x)
    np.testing.assert_allclose(res.features, wx[0], atol=1e-8)
    final = qo.qacq_score([pred], wx[:1], kind=kind, best_label=qa.best_label, coefficient=1.8, num_samples=50,
                          seed=acq_seed, period=BATCH)[0]
    np.testing.assert_allclose(res.rewards, np.full(q, final[0]), rtol=1e-9, atol=1e-12)
  finally:
    dev.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. flies of at most 64 coordinates: bit-identical to the runs recorded before the chunked form
# ---------------------------------------------------------------------------------------------------------------------
def _golden_tool():
  spec = importlib.util.spec_from_file_location('make_set_flies_golden',
                                                os.path.join(ROOT, 'tools', 'make_set_flies_golden.py'))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


GOLDEN = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'eagle_narrow_flies.json')))


@pytest.mark.parametrize('name', sorted(GOLDEN['cases']))
def test_narrow_flies_are_bit_identical_to_the_recorded_runs(name):
  tool = _golden_tool()
  case = {c.name: c for c in tool.CASES}[name]
  want = GOLDEN['cases'][name]
  bc, bz, br = tool.run(case)
  assert [float(v).hex() for v in br.ravel()] == want['rewards']
  assert [float(v).hex() for v in bc.ravel()] == want['features']
  assert [int(v) for v in bz.ravel()] == want['categorical']


# ---------------------------------------------------------------------------------------------------------------------
# 4. designers at 20 continuous dimensions
# ---------------------------------------------------------------------------------------------------------------------
def _problem_and_trials(d, n):
  from vizier_b200 import vz
  p = vz.ProblemStatement()
  for i in range(d):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='obj', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  rng = np.random.default_rng(0)
  trials = []
  for i in range(n):
    xv = rng.uniform(size=d)
    t = vz.Trial(parameters={f'x{j}': float(xv[j]) for j in range(d)}, id=i + 1)
    t.complete(vz.Measurement({'obj': float(-np.sum((xv - 0.3) ** 2))}))
    trials.append(t)
  return p, trials


def _points(sugg, d):
  return np.array([[s.parameters[f'x{j}'].value for j in range(d)] for s in sugg])


def test_ucb_pe_set_batches_in_20_dimensions():
  import dataclasses as dc_
  from vizier_b200 import optimizers as vb
  from vizier_b200 import vz
  from vizier_b200.designers import gp_ucb_pe
  d = 20
  p, trials = _problem_and_trials(d, 40)
  fac = vb.VectorizedOptimizerFactory(strategy_factory=vb.VectorizedEagleStrategyFactory(eagle_config=gp_ucb_pe.default_eagle_config),
                                      max_evaluations=3000, suggestion_batch_size=25)
  cfg = dc_.replace(gp_ucb_pe.UCBPEConfig(), optimize_set_acquisition_for_exploration=True)
  des = gp_ucb_pe.VizierGPUCBPEBandit(p, acquisition_optimizer_factory=fac, config=cfg, rng=2)
  des.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  ns = 'google_gp_ucb_pe_bandit'

  def check_set(sugg):
    pts = _points(sugg, d)
    assert np.all((pts >= 0) & (pts <= 1))
    preds = [s.metadata.ns(ns).ns('prediction_in_warped_y_space') for s in sugg]
    assert [pr['use_ucb'] for pr in preds] == ['False'] * len(sugg)      # the set part is pure exploration
    assert len({pr['acquisition'] for pr in preds}) == 1                 # one acquisition value for the whole set
    dmin = min(np.linalg.norm(pts[i] - pts[j]) for i in range(len(pts)) for j in range(i + 1, len(pts)))
    assert dmin > 0.05                                                   # log-det repels the members

  sugg = des.suggest(6)
  assert len(sugg) == 6
  check_set(sugg[1:])                                 # one UCB / PE suggestion, then a set of 5
  des.update(vz.CompletedTrials(), vz.ActiveTrials([s.to_trial(41 + i) for i, s in enumerate(sugg)]))
  again = des.suggest(6)                              # nothing completed since: one set of 6
  assert len(again) == 6
  check_set(again)


@pytest.mark.parametrize('ensemble_size', [1, 2])
def test_parallel_qei_designer_in_20_dimensions(ensemble_size):
  from vizier_b200 import acquisitions as acq
  from vizier_b200 import ard
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit
  d = 20
  p, trials = _problem_and_trials(d, 30)
  des = gp_bandit.VizierGPBandit(
      p, scoring_function_factory=acq.bayesian_scoring_function_factory(
          lambda data: acq.QEI(acq.get_best_labels(data.labels), num_samples=50)),
      scoring_function_is_parallel=True, ensemble_size=ensemble_size, rng=5,
      ard_optimizer=ard.ScipyLbfgsB(ard.LbfgsBOptions(maxiter=5, num_line_search_steps=5)),
      acquisition_optimizer_factory=gp_bandit.vb.VectorizedOptimizerFactory(max_evaluations=2000))
  des.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  sugg = des.suggest(4)
  assert len(sugg) == 4
  pts = _points(sugg, d)
  assert np.all((pts >= 0) & (pts <= 1))
  assert len({tuple(x) for x in pts}) == 4
  values = {json.loads(s.metadata.ns('devinfo')['acquisition_optimization'])['acquisition'] for s in sugg}
  assert len(values) == 1 and np.isfinite(list(values)[0])


# ---------------------------------------------------------------------------------------------------------------------
# 5. refused set flies
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dc,dk,q', [(4, 0, 17), (64, 0, 17), (3, 1, 2)])
def test_eagle_begin_refuses_set_flies_outside_its_limits(dc, dk, q):
  from vizier_b200 import _lib, gp
  rng = np.random.default_rng(1)
  x = rng.uniform(size=(8, dc))
  z = rng.integers(0, 3, size=(8, dk)).astype(np.int32) if dk else None
  dev = gp.DeviceGP(0)
  try:
    dev.fit(x, rng.normal(size=8), gp.GPHyperParams(1.0, np.full(dc, 0.5), 1e-3, np.ones(dk) if dk else None), z=z)
    with pytest.raises(_lib.VzgpError) as err:
      gp.SteppedEagle(dev, _config(eo.EagleConfig(), 50, 2, q), 1, 3, cat_sizes=[3] * dk or None)
    assert err.value.status == _lib.VZGP_ERR_ARG
    assert 'n_parallel <= 16 and n_parallel * Dc <= 1024' in str(err.value)
    if not dk:     # the largest accepted fly on the same handle
      gp.SteppedEagle(dev, _config(eo.EagleConfig(), 50, 2, min(16, 1024 // dc)), 1, 3).end()
  finally:
    dev.close()
