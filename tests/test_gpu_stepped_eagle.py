"""Host-stepped Eagle loop (vzgp_eagle_begin / seed / ask / tell / end) and `prior_acquisition`.

The stepped loop shares state, kernels and Philox draws with `vzgp_eagle_run`; the caller scores each batch.  With
the library's own acquisition as the scorer it must reproduce `vzgp_eagle_run`; with an extra host-side term it is
compared with the oracle's optimiser driven by the same composite score function (gp_ucb_pe.py:376-379, :487-490).
"""
import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from oracle import eagle_oracle as eo  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402


@pytest.fixture()
def dev():
  from vizier_b200 import gp
  d = gp.DeviceGP(0)
  yield d
  d.close()


def _problem(n, d, seed):
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, d))
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  return x, y


def _cfg(cfg_o, pool, batch, steps):
  from vizier_b200 import _lib
  return _lib.EagleConfig(cfg_o.visibility, cfg_o.gravity, cfg_o.negative_gravity, cfg_o.perturbation,
                          cfg_o.perturbation_lower_bound, cfg_o.penalize_factor, cfg_o.normalization_scale,
                          cfg_o.prior_trials_pool_pct, pool, batch, steps * batch)


def _prior_term(xc):
  """A smooth user prior over the features (what `prior_acquisition` would return)."""
  return -0.7 * np.sum((np.asarray(xc) - 0.8) ** 2, axis=1)


@pytest.mark.parametrize('n,d,pool,batch,steps', [(120, 4, 50, 25, 12), (300, 6, 100, 50, 6)])
def test_stepped_loop_reproduces_eagle_run_and_oracle_with_prior_term(dev, n, d, pool, batch, steps):
  from vizier_b200 import gp
  x, y = _problem(n, d, 31)
  ls2 = 0.5 * (1 + np.arange(d) / d)
  po, pg = go.GPParams(1.0, ls2, 1e-3), gp.GPHyperParams(1.0, ls2, 1e-3)
  pred = go.precompute_predictive(po, x, y)
  dev.fit(x, y, pg)
  radius = go.trust_radius(n, d, 0)
  acq = gp.Acquisition(1.8, True, radius)
  cfg_o = eo.EagleConfig()
  cfg = _cfg(cfg_o, pool, batch, steps)

  def run_stepped(extra):
    se = gp.SteppedEagle(dev, cfg, 3, 7, n_prior=n)

    def score(xs):
      out = dev.score(xs, acq)['score']
      if extra:
        with torch.cuda.stream(dev._stream):
          out = out + torch.as_tensor(_prior_term(xs.cpu().numpy()), device=dev.device)
      return out

    se.seed(x, None, score(torch.from_numpy(x).cuda()))
    for _ in range(steps):
      xs, _, rewards = se.ask()
      r = score(xs)
      with torch.cuda.stream(dev._stream):
        rewards.copy_(r)
      se.tell()
    return se.end()

  # 1. the library's acquisition as the scorer: the same run as vzgp_eagle_run (the cooperative form at these sizes)
  bx0, _, br0 = dev.eagle_run(cfg, acq, count=3, seed=7, prior=x)
  assert dev.get_int('eagle_route') == 1          # vzgp_eagle_route: cooperative
  bx1, _, br1 = run_stepped(False)
  np.testing.assert_allclose(br1, br0, atol=1e-9)
  np.testing.assert_allclose(bx1, bx0, atol=1e-9)
  # 2. with the host-side prior term: the oracle's optimiser on the composite score
  score_fn = lambda q: go.score_with_aux(pred, q)[0] + _prior_term(q)
  wx, wr, _ = eo.run_eagle_optimizer(score_fn, dim=d, pool_size=pool, batch_size=batch, max_evaluations=steps * batch,
                                     count=3, seed=7, cfg=cfg_o, prior_features=x)
  bx2, _, br2 = run_stepped(True)
  np.testing.assert_allclose(br2, wr, atol=1e-9)
  np.testing.assert_allclose(bx2, wx, atol=1e-9)
  assert not np.allclose(bx2, bx0)     # the prior term moved the optimum


def test_stepped_loop_rejects_out_of_order_calls(dev):
  from vizier_b200 import _lib, gp
  x, y = _problem(40, 3, 5)
  dev.fit(x, y, gp.GPHyperParams(1.0, np.full(3, 0.5), 1e-3))
  cfg = _cfg(eo.EagleConfig(), 50, 25, 2)
  se = gp.SteppedEagle(dev, cfg, 1, 3)
  with pytest.raises(_lib.VzgpError):
    se.tell()                       # nothing asked yet
  se.ask()
  with pytest.raises(_lib.VzgpError):
    se.ask()                        # the previous batch has not been told
  se.tell()
  se.end()
  with pytest.raises(_lib.VzgpError):
    se.tell()                       # the run is over


def test_ucb_pe_designer_with_prior_acquisition(dev):
  """`VizierGPUCBPEBandit(prior_acquisition=...)`: suggestions are pulled towards the prior's optimum and carry the
  prior value in their metadata (gp_ucb_pe.py:1147-1150)."""
  del dev
  from vizier_b200 import vz
  from vizier_b200.designers import gp_ucb_pe
  from vizier_b200 import optimizers as vb
  p = vz.ProblemStatement()
  for i in range(3):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='obj', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  rng = np.random.default_rng(0)
  trials = []
  for i in range(30):
    xv = rng.uniform(size=3)
    t = vz.Trial(parameters={f'x{j}': float(xv[j]) for j in range(3)}, id=i + 1)
    t.complete(vz.Measurement({'obj': float(-np.sum((xv - 0.3) ** 2))}))
    trials.append(t)
  fac = vb.VectorizedOptimizerFactory(strategy_factory=vb.VectorizedEagleStrategyFactory(eagle_config=gp_ucb_pe.default_eagle_config),
                                      max_evaluations=2500, suggestion_batch_size=25)
  strong_prior = lambda xc, xz: -50.0 * np.sum((xc - 0.9) ** 2, axis=1)

  def suggest(prior):
    d = gp_ucb_pe.VizierGPUCBPEBandit(p, acquisition_optimizer_factory=fac, prior_acquisition=prior, rng=1)
    d.update(vz.CompletedTrials(trials), vz.ActiveTrials())
    return d.suggest(1)[0]

  s0, s1 = suggest(None), suggest(strong_prior)
  x0 = np.array([s0.parameters[f'x{j}'].value for j in range(3)])
  x1 = np.array([s1.parameters[f'x{j}'].value for j in range(3)])
  assert np.sum((x1 - 0.9) ** 2) < np.sum((x0 - 0.9) ** 2)
  assert np.max(np.abs(x1 - 0.9)) < 0.25
  val = float(s1.metadata.ns('google_gp_ucb_pe_bandit').ns('prior_acquisition')['value'])
  np.testing.assert_allclose(val, strong_prior(x1[None, :], None)[0], rtol=1e-6, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------------------
# Set-PE batches (gp_ucb_pe.py:510-594, :1157-1260): set scorer, n_parallel Eagle, designer
# ---------------------------------------------------------------------------------------------------------------------
def _two_models(n_done, n_pend, d, seed, sn2=1e-3):
  from vizier_b200 import gp
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n_done + n_pend, d))
  y = -np.sum((x[:n_done] - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n_done)
  ls2 = 0.3 * (1 + np.arange(d) / d)
  po, pg = go.GPParams(1.1, ls2, sn2), gp.GPHyperParams(1.1, ls2, sn2)
  pred_a = go.precompute_predictive(po, x[:n_done], y)
  y_all = np.r_[y, np.zeros(n_pend)]
  pred_b = go.precompute_predictive(po, x, y_all)
  dev_a = gp.DeviceGP(0)
  dev_b = gp.DeviceGP(0, stream=dev_a.stream)     # both models on one stream (vzgp_score_set_pe requires it)
  return x, y, y_all, pg, pred_a, pred_b, dev_a, dev_b


@pytest.mark.parametrize('n_done,n_pend,d,q,radius', [(60, 5, 4, 3, 0.25), (150, 0, 6, 5, 0.9), (40, 8, 2, 8, 0.3)])
def test_set_pe_score_matches_oracle(n_done, n_pend, d, q, radius):
  from vizier_b200 import gp
  x, y, y_all, pg, pred_a, pred_b, dev_a, dev_b = _two_models(n_done, n_pend, d, 3)
  dev_a.fit(x[:n_done], y, pg)
  dev_b.fit(x, y_all, pg)
  rng = np.random.default_rng(9)
  sets = rng.uniform(size=(37, q, d))
  sets[3, 1] = sets[3, 0]                      # a duplicated point: covariance singular up to the noise
  sets[5] = x[:q]                              # a set of observed points
  pe = gp.UcbPeAcquisition(mode=1, explore_coefficient=0.5, penalty_coefficient=10.0, threshold=-0.2,
                           use_trust_region=True, trust_radius=radius, tr_rows=n_done + max(n_pend - 2, 0))
  out = dev_a.score_set_pe(dev_b, sets.reshape(-1, d), q, pe)
  dev_a.synchronize()
  want, aux = go.set_pe_score(pred_a, pred_b, sets, explore_coefficient=0.5, penalty_coefficient=10.0, threshold=-0.2,
                              tr_rows=n_done + max(n_pend - 2, 0), trust_radius_value=radius)
  np.testing.assert_allclose(out['mean'].cpu().numpy(), aux['mean'], atol=1e-10)
  np.testing.assert_allclose(out['stddev'].cpu().numpy(), aux['stddev'], atol=1e-10)
  np.testing.assert_allclose(out['stddev_from_all'].cpu().numpy(), aux['stddev_from_all'], atol=1e-9)
  np.testing.assert_allclose(out['score'].cpu().numpy(), want, rtol=1e-9, atol=1e-7)
  dev_a.close(); dev_b.close()


def test_eagle_sets_trajectory_matches_oracle():
  """The n_parallel form of the optimiser (set flies) through the stepped loop against the oracle's, same Philox draws."""
  from vizier_b200 import gp
  n_done, n_pend, d, q, pool, batch, steps = 50, 4, 3, 4, 50, 25, 10
  x, y, y_all, pg, pred_a, pred_b, dev_a, dev_b = _two_models(n_done, n_pend, d, 5)
  dev_a.fit(x[:n_done], y, pg)
  dev_b.fit(x, y_all, pg)
  radius = 0.35
  pe = gp.UcbPeAcquisition(mode=1, explore_coefficient=0.5, penalty_coefficient=10.0, threshold=-0.1,
                           use_trust_region=True, trust_radius=radius, tr_rows=n_done + n_pend)
  cfg_o = eo.EagleConfig()
  cfg = _cfg(cfg_o, pool, batch, steps)
  cfg.n_parallel = q
  n_sets = n_done // q
  prior_sets = x[: n_sets * q].reshape(n_sets, q * d)
  score = lambda xs: dev_a.score_set_pe(dev_b, xs.reshape(-1, d), q, pe)['score']
  se = gp.SteppedEagle(dev_a, cfg, 2, 11, n_prior=n_sets)
  se.seed(prior_sets, None, score(torch.from_numpy(prior_sets).cuda()))
  for _ in range(steps):
    xs, _, rewards = se.ask()
    r = score(xs)
    with torch.cuda.stream(dev_a._stream):
      rewards.copy_(r)
    se.tell()
  bx, _, br = se.end()
  score_fn = lambda s: go.set_pe_score(pred_a, pred_b, s, explore_coefficient=0.5, penalty_coefficient=10.0, threshold=-0.1,
                                       tr_rows=n_done + n_pend, trust_radius_value=radius)[0]
  wx, wr, _ = eo.run_eagle_optimizer_sets(score_fn, dim=d, n_parallel=q, pool_size=pool, batch_size=batch,
                                          max_evaluations=steps * batch, count=2, seed=11, cfg=cfg_o, prior_features=x[:n_done])
  np.testing.assert_allclose(br, wr, rtol=1e-8, atol=1e-6)
  np.testing.assert_allclose(bx.reshape(2, q, d), wx, atol=1e-8)
  dev_a.close(); dev_b.close()


def test_ucb_pe_designer_set_batches(dev):
  """`optimize_set_acquisition_for_exploration=True`: a batch of 4 = one UCB/PE suggestion + a set of 3 (or a set of 4
  when nothing completed since the last suggestion); points of a set are spread out (log-det acquisition)."""
  del dev
  from vizier_b200 import vz
  from vizier_b200.designers import gp_ucb_pe
  from vizier_b200 import optimizers as vb
  import dataclasses
  p = vz.ProblemStatement()
  for i in range(3):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='obj', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  rng = np.random.default_rng(0)
  trials = []
  for i in range(40):
    xv = rng.uniform(size=3)
    t = vz.Trial(parameters={f'x{j}': float(xv[j]) for j in range(3)}, id=i + 1)
    t.complete(vz.Measurement({'obj': float(-np.sum((xv - 0.3) ** 2))}))
    trials.append(t)
  fac = vb.VectorizedOptimizerFactory(strategy_factory=vb.VectorizedEagleStrategyFactory(eagle_config=gp_ucb_pe.default_eagle_config),
                                      max_evaluations=3000, suggestion_batch_size=25)
  cfg = dataclasses.replace(gp_ucb_pe.UCBPEConfig(), optimize_set_acquisition_for_exploration=True)
  d = gp_ucb_pe.VizierGPUCBPEBandit(p, acquisition_optimizer_factory=fac, config=cfg, rng=2)
  d.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  sugg = d.suggest(4)
  assert len(sugg) == 4
  pts = np.array([[s.parameters[f'x{j}'].value for j in range(3)] for s in sugg])
  assert np.all((pts >= 0) & (pts <= 1))
  ns = 'google_gp_ucb_pe_bandit'
  flags = [s.metadata.ns(ns).ns('prediction_in_warped_y_space')['use_ucb'] for s in sugg]
  assert flags[1:] == ['False'] * 3                     # the set part is pure exploration
  acqs = {s.metadata.ns(ns).ns('prediction_in_warped_y_space')['acquisition'] for s in sugg[1:]}
  assert len(acqs) == 1                                 # one acquisition value for the whole set
  dmin = min(np.linalg.norm(pts[i] - pts[j]) for i in range(1, 4) for j in range(i + 1, 4))
  assert dmin > 0.05                                    # log-det repels the members from each other


@pytest.mark.parametrize('set_pe', [False, True])
def test_prior_acquisition_like_the_reference_test(set_pe):
  """gp_ucb_pe_test.py:476-607 (test_prior_acquisition), same configuration and assertions: a constant prior
  acquisition of 12345 appears in every suggestion's metadata; the first suggestion of a batch is UCB with
  acquisition = mean + 10 stddev + prior; the others are PE - per point  stddev_from_all (+ a non-positive penalty)
  + prior, or, with set optimisation, ONE value log det(cov) + prior for the whole set whose geometric mean of
  eigenvalues is below the arithmetic mean of the predictive variances."""
  import dataclasses
  from vizier_b200 import vz
  from vizier_b200.designers import gp_ucb_pe
  from vizier_b200 import optimizers as vb
  p = vz.ProblemStatement()
  for i in range(3):
    p.search_space.root.add_float_param(f'x{i}', -1.0 * (i + 1), 2.0 * (i + 1))
  p.metric_information.append(vz.MetricInformation(name='metric', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  fac = vb.VectorizedOptimizerFactory(strategy_factory=vb.VectorizedEagleStrategyFactory(), max_evaluations=100)
  cfg = gp_ucb_pe.UCBPEConfig(ucb_coefficient=10.0, explore_region_ucb_coefficient=0.5, cb_violation_penalty_coefficient=10.0,
                              ucb_overwrite_probability=0.0, pe_overwrite_probability=0.0, signal_to_noise_threshold=0.0,
                              optimize_set_acquisition_for_exploration=set_pe)
  ns = 'gp_ucb_pe_bandit_test'
  des = gp_ucb_pe.VizierGPUCBPEBandit(p, acquisition_optimizer_factory=fac, metadata_ns=ns, num_seed_trials=1, config=cfg,
                                      prior_acquisition=lambda xc, xz: np.ones(xc.shape[0]) * 12345.0, rng=1)
  rng = np.random.default_rng(1)
  batch, iters, trial_id, all_trials = 3, 2, 1, []
  for _ in range(iters):
    sugg = des.suggest(count=batch)
    assert len(sugg) == batch
    done = []
    for s in sugg:
      trial_id += 1
      t = s.to_trial(trial_id)
      t.complete(vz.Measurement({'metric': float(rng.uniform(-10.0, 10.0))}))
      done.append(t)
    all_trials.extend(done)
    des.update(vz.CompletedTrials(done), vz.ActiveTrials())
  assert len(all_trials) == iters * batch
  set_acq, sd_all = None, []
  for idx, t in enumerate(all_trials):
    if idx < batch:
      continue                      # seed suggestions
    md = t.metadata.ns(ns)
    pred = md.ns('prediction_in_warped_y_space')
    mean, sd, sda, acq = (float(pred[k]) for k in ('mean', 'stddev', 'stddev_from_all', 'acquisition'))
    prior = float(md.ns('prior_acquisition')['value'])
    assert prior == 12345.0
    if idx % batch == 0:
      assert pred['use_ucb'] == 'True'
      np.testing.assert_allclose(mean + 10.0 * sda + prior, acq, rtol=1e-9)
    else:
      assert pred['use_ucb'] == 'False'
      if set_pe:
        assert acq > 10000.0
        sd_all.append(sda)
        if set_acq is None:
          set_acq = acq - prior
        else:
          np.testing.assert_allclose(set_acq, acq - prior, rtol=1e-9)
      else:
        assert acq <= sda + prior + 1e-9      # PE: stddev_from_all + (penalty <= 0) + prior
  if set_pe:
    assert np.exp(set_acq / (batch - 1)) <= np.mean(np.square(sd_all)) + 1e-12
