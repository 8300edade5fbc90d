"""`vzgp_score_grad` / `vzgp_score_grad_ensemble` and the L-BFGS-B acquisition optimiser on the device.

Values, means and stddevs are held to the 1e-10 of test_gpu_score_routes.py; the trust-region distance bit for bit.
The gradient is held to 1e-9 of its max-norm over the points of a case: each entry is a sum over N trials of terms
as large as that max-norm, so round-off in a different summation order is ~N * 1e-16 of it (1e-13 at N = 1000), and
the bound leaves room for that while any formula error (a dropped term, a wrong factor) shows up in the leading
digits.  Sizes cross every batching boundary of the kernels: 64-row GEMM tiles (N = 64 / 65), one CTA per candidate
and the 4096-candidate chunks (M = 100 000), the lead member's distance planes, and the feature loop (Dc = 1 / 64)."""
import json

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

import lbfgsb_oracle as lo  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402
from vizier_b200 import gp, vz  # noqa: E402
from vizier_b200 import optimizers as vb  # noqa: E402
from vizier_b200.designers import gp_bandit  # noqa: E402

TOL = 1e-10
GRAD_TOL = 1e-9
ACQS = ['ucb', 'lcb', 'ei', 'pi', 'atr_ucb_pi', 'atr_ucb_lcb']


def _model(n, dc, E, linear, seed=0, n_valid=None, label_offset=0.0, noise=1e-3):
  rng = np.random.default_rng(seed)
  x, y, _ = lo.make_model(rng, n, dc, linear=linear)
  y = y + label_offset
  params = [lo.make_model(rng, 1, dc, linear=linear, seed_params=seed * 10 + e, noise=noise)[2] for e in range(E)]
  preds = [lo.predictive(x, y, p, n_valid) for p in params]
  if E == 1:
    dev = gp.DeviceGP(0)
    dev.fit(x, y, lo.device_params(params[0]), n_valid=n_valid)
  else:
    dev = gp.EnsembleGP(0, E)
    dev.fit(x, y, [lo.device_params(p) for p in params], n_valid=n_valid)
  return x, y, preds, dev


def _acq(name, best, radius):
  spec = lo.acquisitions(best)[name]
  return gp.Acquisition(1.8, radius is not None, 1.0 if radius is None else radius, acq_fn=spec)


def _check(dev, preds, xs, acq, rows=None):
  out = dev.score_grad(xs, acq, with_aux=True)
  ref = dev.score(xs, acq, with_aux=True)
  dev.synchronize()
  got = {k: out[k].cpu().numpy() for k in ('score', 'grad', 'mean', 'stddev', 'linf_distance')}
  sc = ref['score'].cpu().numpy()
  np.testing.assert_allclose(got['score'], sc, rtol=TOL if len(preds) == 1 else 1e-9, atol=TOL)
  sel = np.arange(len(xs)) if rows is None else rows
  want = lo.score_and_grad(preds, xs[sel], acq)
  for k in ('score', 'mean', 'stddev'):
    np.testing.assert_allclose(got[k][sel], want[k], rtol=TOL, atol=TOL, err_msg=k)
  if acq.use_trust_region and acq.trust_radius <= 0.5:
    np.testing.assert_array_equal(got['linf_distance'][sel], want['linf_distance'])
  scale = max(np.max(np.abs(want['grad'])), 1e-300)
  err = np.max(np.abs(got['grad'][sel] - want['grad']))
  assert err <= GRAD_TOL * scale, (err, scale)
  return got, want


# (N, Dc, M): every N in {5, 64, 65, 1000}, Dc in {1, 20, 64} and M in {1, 25, 200, 100 000} appears
CASES = [(5, 1, 1), (5, 20, 25), (64, 20, 200), (65, 64, 25), (65, 1, 100_000), (1000, 20, 25), (1000, 1, 200),
         (1000, 64, 1), (1000, 20, 100_000)]


@pytest.mark.parametrize('linear', [False, True])
@pytest.mark.parametrize('E', [1, 2, 3, 5])
@pytest.mark.parametrize('n,dc,m', CASES)
def test_score_grad_matches_oracle(n, dc, m, E, linear):
  """Every acquisition, the trust region active (radius 0.25 at small N: many points outside) and inactive."""
  if E == 5 and (n, m) != (65, 25) and (n, dc, m) != (1000, 20, 25):
    pytest.skip('E = 5 at two sizes')
  x, y, preds, dev = _model(n, dc, E, linear, seed=n + dc)
  rng = np.random.default_rng(m)
  xs = rng.uniform(size=(m, dc))
  rows = None if m <= 200 else np.sort(rng.choice(m, 200, replace=False))
  best = float(np.max(y))
  for name in ACQS:
    for radius in ((0.25, None) if n <= 65 else (None,)):
      _check(dev, preds, xs, _acq(name, best, radius), rows)
  dev.close()


def test_padded_trials():
  """n_valid < n: the padded rows take no part in mean, variance, gradient or distance."""
  x, y, preds, dev = _model(40, 6, 2, False, seed=4, n_valid=31)
  xs = np.random.default_rng(2).uniform(size=(50, 6))
  for radius in (0.3, None):
    _check(dev, preds, xs, _acq('ei', float(np.max(y[:31])), radius))
  dev.close()


def test_ensemble_members_with_different_padding():
  """Members that share their 31 valid trials but were fitted with 40 and 70 rows (padded sizes 64 and 128): each is
  scored with its own padded size, to the oracle."""
  rng = np.random.default_rng(6)
  x, y, _ = lo.make_model(rng, 70, 4)
  params = [lo.make_model(rng, 1, 4, seed_params=e)[2] for e in range(2)]
  dev = gp.EnsembleGP(0, 2)
  dev.members[0].fit(x[:40], y[:40], lo.device_params(params[0]), n_valid=31)
  dev.members[1].fit(x, y, lo.device_params(params[1]), n_valid=31)
  preds = [lo.predictive(x[:40], y[:40], params[0], 31), lo.predictive(x, y, params[1], 31)]
  xs = rng.uniform(size=(60, 4))
  for radius in (0.3, None):
    _check(dev, preds, xs, _acq('pi', float(np.max(y[:31])), radius))
  dev.close()


def test_clamped_variance():
  """Candidates on well-separated trials with noise 1e-20: the computed variance is round-off around 0 and goes
  negative at some of them.  There the device reports stddev 0, counts the clamp, and keeps only the mean part of the
  gradient with the sd = 0 slopes: UCB 1, EI [imp > 0], PI 0 (the oracle's dmu at the same points)."""
  rng = np.random.default_rng(8)
  x = np.stack(np.meshgrid(np.linspace(0.1, 0.9, 4), np.linspace(0.1, 0.9, 4)), -1).reshape(-1, 2)
  y = np.sin(3 * x[:, 0]) + x[:, 1]
  params = go.GPParams(1.0, np.full(2, 0.02), 1e-20)
  pred = lo.predictive(x, y, params)
  dev = gp.DeviceGP(0)
  dev.fit(x, y, lo.device_params(params))
  xs = np.concatenate([x, x + 1e-9, x - 1e-9])
  _, _, dmu, _ = lo.moment_grads(pred, xs)
  best = float(np.median(y))
  for name, slope in (('ucb', lambda imp: 1.0), ('ei', lambda imp: float(imp > 0)), ('pi', lambda imp: 0.0)):
    dev.clamped_count()                       # reset
    out = dev.score_grad(xs, _acq(name, best, None), with_aux=True)
    dev.synchronize()
    sd, mean = out['stddev'].cpu().numpy(), out['mean'].cpu().numpy()
    grad = out['grad'].cpu().numpy()
    clamped = sd == 0
    assert clamped.any() and dev.clamped_count() == int(clamped.sum())
    for m in np.flatnonzero(clamped):
      imp = mean[m] - best - (0.01 if name == 'ei' else 0.0)
      np.testing.assert_allclose(grad[m], slope(imp) * dmu[m], rtol=1e-9, atol=1e-9 * np.max(np.abs(dmu)))
  dev.close()


def test_mixture_against_device_member_moments():
  """In a cancellation regime (|mu| ~ 1000 > 1e3 stddev) the ensemble's stddev and its gradient equal the two-pass
  mixture of the members' own device moments: a one-pass variance mean(var + mu^2) - mean^2 loses ~6 digits here."""
  x, y, preds, dev = _model(30, 3, 3, False, seed=9, label_offset=1000.0, noise=1e-6)
  xs = x[:20] + 1e-3
  members = []
  for m in dev.members:
    a = m.score_grad(xs, gp.Acquisition(0.0, False, 1.0), with_aux=True)
    b = m.score_grad(xs, gp.Acquisition(1.0, False, 1.0))
    m.synchronize()
    mu, sd = a['mean'].cpu().numpy(), a['stddev'].cpu().numpy()
    dmu, dsd = a['grad'].cpu().numpy(), b['grad'].cpu().numpy() - a['grad'].cpu().numpy()
    members.append((mu, sd, dmu, 2 * sd[:, None] * dsd))
  mus = np.stack([q[0] for q in members])
  mean = mus.mean(0)
  var = np.mean([q[1] ** 2 for q in members], 0) + ((mus - mean) ** 2).mean(0)
  dvar = np.mean([q[3] for q in members], 0) + 2.0 / 3 * np.einsum('em,emd->md', mus - mean, np.stack([q[2] for q in members]))
  sd = np.sqrt(var)
  out = dev.score_grad(xs, gp.Acquisition(1.0, False, 1.0), with_aux=True)
  dev.synchronize()
  assert np.min(np.abs(mean) / sd) > 1e3
  np.testing.assert_allclose(out['stddev'].cpu().numpy(), sd, rtol=1e-9)
  want = np.stack([q[2] for q in members]).mean(0) + dvar / (2 * sd[:, None])
  np.testing.assert_allclose(out['grad'].cpu().numpy(), want, rtol=1e-7, atol=GRAD_TOL * np.max(np.abs(want)))
  one_pass = np.sqrt(np.maximum(np.mean([q[1] ** 2 + q[0] ** 2 for q in members], 0) - mean ** 2, 0))
  assert np.max(np.abs(one_pass - sd) / sd) > 1e-7     # the regime does tell the two forms apart
  dev.close()


@pytest.mark.parametrize('variant', ['no_dkss', 'dvar_as_dsd'])
def test_deliberate_breaks_are_caught(variant):
  """The device agrees with the oracle where the broken formulas (no dkss for the linear kernel, d var used for
  d sd) miss it by far more than the gradient tolerance: test_score_grad_matches_oracle fails on either break."""
  x, y, preds, dev = _model(64, 5, 2, True, seed=3)
  xs = np.random.default_rng(1).uniform(size=(25, 5))
  acq = _acq('ucb', 0.0, None)
  got, want = _check(dev, preds, xs, acq)
  broken = lo.score_and_grad(preds, xs, acq, variant=variant)
  assert np.max(np.abs(broken['grad'] - got['grad'])) > 1e3 * GRAD_TOL * np.max(np.abs(want['grad']))
  dev.close()


@pytest.mark.parametrize('E,linear', [(1, False), (1, True), (3, False)])
def test_optimizer_on_device_matches_oracle_run(E, linear):
  """The same L-BFGS-B restarts from the same inits, on the device and on the oracle: the same winners; every reward
  equals the final value of the restart that returned it."""
  x, y, preds, dev = _model(40, 3, E, linear, seed=21)
  acq = gp.Acquisition(1.8, True, 0.45, acq_fn=lo.acquisitions(float(np.max(y)))['ei'])
  opt = vb.LBFGSBOptimizer(((0.0, 1.0),) * 3, random_restarts=8, maxiter=30)
  res = opt(dev, acq, count=3, seed=5)
  assert opt.rounds > 1
  host = opt.optimize_host(lambda p: (lambda r: (r['score'], r['grad']))(lo.score_and_grad(preds, p, acq)),
                           count=3, seed=5)
  np.testing.assert_allclose(res.features, host.features, atol=1e-6)
  np.testing.assert_allclose(res.rewards, host.rewards, rtol=1e-8, atol=1e-10)
  # the reward (vzgp_score at the winner) is the restart's own final value (vzgp_score_grad there)
  np.testing.assert_allclose(res.rewards, -opt.final_losses, rtol=TOL if E == 1 else 1e-9, atol=TOL)
  assert set(res.aux) == {'mean', 'stddev', 'linf_distance', 'radius', 'raw_acquisition'}
  dev.close()


def _flat_scaled_problem():
  p = vz.ProblemStatement()
  p.search_space.root.add_float_param('lineardouble', -1.0, 2.0)
  p.search_space.root.add_float_param('logdouble', 1e-4, 1e2, scale_type=vz.ScaleType.LOG)
  p.metric_information.append(vz.MetricInformation(name='obj', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  return p


def _complete(suggestions, f, start_id):
  out = []
  for i, s in enumerate(suggestions):
    t = s.to_trial(start_id + i)
    xv = np.array([t.parameters[k].value for k in sorted(t.parameters)])
    t.complete(vz.Measurement({'obj': float(f(xv))}))
    out.append(t)
  return out


@pytest.mark.parametrize('iters,batch,seeds,ensemble,padding', [(3, 1, 1, 2, None), (5, 1, 3, 1, 'POWERS_OF_2')])
def test_designer_on_flat_continuous_space(iters, batch, seeds, ensemble, padding):
  """gp_bandit_test.py:130-164, the two LBFGSB rows, with linear_coef = 0.1: suggestion counts, sample / predict, and
  the recorded acquisition equal to the device score at the suggested point."""
  p = _flat_scaled_problem()
  d = gp_bandit.VizierGPBandit.from_problem(p, seed=2, acquisition_optimizer_factory=vb.LBFGSBOptimizerFactory(),
                                            ensemble_size=ensemble, linear_coef=0.1, num_seed_trials=seeds,
                                            padding_schedule=padding)
  f = lambda v: -np.sum((v - 0.3) ** 2)
  tid = 1
  for _ in range(seeds):
    trials = _complete(d.suggest(1), f, tid); tid += 1
    d.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  for _ in range(iters):
    sugg = d.suggest(batch)
    assert len(sugg) == batch
    info = sugg[0].metadata.ns('devinfo')
    md = json.loads(info['acquisition_optimization'])
    for k in ('acquisition', 'mean', 'stddev', 'raw_acquisition', 'linf_distance', 'radius'):
      assert k in md and np.isfinite(md[k])
    assert 'acquisition_optimization_warning' not in info
    assert 'time_spent' in sugg[0].metadata.ns('oss_gp_bandit').ns('devinfo')
    xs, _ = d._converter.to_features([sugg[0].to_trial(0)])
    acq = d._acquisition(len(d._trials), d._trials_to_data(d._trials)[2], features=None)
    sc = d._dev.score(xs, acq)
    d._dev.synchronize()
    np.testing.assert_allclose(md['acquisition'], sc['score'].cpu().numpy()[0], rtol=1e-9, atol=1e-9)
    trials = _complete(sugg, f, tid); tid += len(trials)
    d.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  assert len(d.suggest(3)) == 3
  pts = [vz.Trial(parameters={'lineardouble': v, 'logdouble': 0.1}) for v in (-1.0, 0.5, 2.0)]
  s = d.sample(pts, num_samples=5)
  assert s.shape == (5, 3) and np.isfinite(s).all()
  pr = d.predict(pts)
  assert len(pr.mean) == 3 and np.isfinite(pr.mean).all() and np.isfinite(pr.stddev).all()


def test_minimisation_converges_faster_than_random():
  p = vz.ProblemStatement()
  for i in range(3):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='obj', goal=vz.ObjectiveMetricGoal.MINIMIZE))
  f = lambda v: np.sum((v - 0.7) ** 2)
  d = gp_bandit.VizierGPBandit.from_problem(p, seed=3, acquisition_optimizer_factory=vb.LBFGSBOptimizerFactory())
  best, tid = np.inf, 1
  for _ in range(15):
    trials = _complete(d.suggest(1), f, tid); tid += 1
    best = min(best, trials[0].final_measurement.metrics['obj'].value)
    d.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  rng = np.random.default_rng(0)
  assert best < 0.02 and best < min(f(rng.uniform(size=3)) for _ in range(15))
