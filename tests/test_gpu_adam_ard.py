"""ARD with Adam (ard.OptaxTrain) on the device: the fused kernel `vzgp_ard_adam_small` (csrc/ard_adam.cu) against the
NumPy restatement (adam_oracle.py over oracle/gp_oracle.py), its loss against `DeviceGP.make_loss_fn`, the fused route
against the host-stepped one, and both designers end to end.

Tolerances.  The kernel and the oracle evaluate the same loss by different summation orders (~1e-13 relative), so
per-epoch losses and final parameters are held to 1e-9 relative; a parameter near its lower bound is held in absolute
terms to 1e-12 of its box width, since SoftClip computes it as high - (high - low - small) and rounds at the scale of
`high`.  The fused and host-stepped routes perform the same IEEE operations (ard.py mirrors ard_adam.cu) on losses that
agree to 1e-13, so they are held to 1e-12 over 200 epochs (measured on an H100: ~1e-14 on the losses, ~1e-13 on the
parameters).  The initial points keep the noise variance moderate (`_inits`): with K_y near singular the gradient's
round-off grows with its condition number and Adam's sign-like first steps amplify it, so two correct implementations
part after a few dozen epochs."""
import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

import adam_oracle as ao  # noqa: E402
import fit_fixtures as ff  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402
from vizier_b200 import ard, gp, vz  # noqa: E402
from vizier_b200.designers import gp_bandit, gp_ucb_pe  # noqa: E402

LR = 1e-2
ORACLE_EPOCHS = 50


def _data(n, dc, dk, seed):
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, dc))
  z = rng.integers(0, 4, size=(n, dk)).astype(np.int32) if dk else None
  y = np.sin(3.0 * x.sum(1)) - np.sum((x - 0.4) ** 2, 1) + 0.05 * rng.normal(size=n)
  if dk:
    y = y + 0.3 * np.cos(z.sum(1))
  return x, y, z


def _inits(rng, dc, dk, r):
  """Log-uniform initial points with a moderate noise variance: K_y stays well conditioned, so two correct
  implementations follow the same trajectory (with a noise variance near 1e-10 the gradient's round-off grows with the
  condition number and Adam's sign-like first steps amplify it)."""
  th = ard.log_uniform_init(rng, dc, dk, r)
  th[:, dk + dc] = rng.uniform(0.01, 0.1, size=r)
  return th


def _rel(got, want, lo, hi):
  """max |got - want| / (|want| + 1e-12 (hi - lo)) over the parameters (NaN where both are NaN counts as equal)."""
  got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
  both_nan = np.isnan(got) & np.isnan(want)
  err = np.abs(got - want) / (np.abs(want) + 1e-12 * (hi - lo))
  err = np.where(both_nan, 0.0, err)
  return float(np.max(np.where(np.isnan(err), np.inf, err)))


def _rel_trace(got, want):
  both_nan = np.isnan(got) & np.isnan(want)
  scale = np.nanmax(np.abs(want)) if np.any(np.isfinite(want)) else 1.0
  err = np.where(both_nan, 0.0, np.abs(got - want) / np.maximum(np.abs(want), 1e-9 * scale))
  return float(np.max(np.where(np.isnan(err), np.inf, err)))


def _run_fused(dev, x, y, z, th0, lo, hi, epochs, n_valid):
  return dev.ard_adam_small(x, y, th0, lo, hi, learning_rate=LR, b1=0.9, b2=0.999, eps=1e-8, eps_root=0.0,
                            epochs=epochs, z=z, n_valid=n_valid)


def _oracle_fn(x, y, z, n_valid):
  row_valid = np.arange(x.shape[0]) < n_valid
  return lambda th: go.loss_and_grad(th, x, y, z, row_valid=row_valid)


def _check_against_oracle(x, y, z, n_valid, th0, lo, hi, restarts=None, epochs=ORACLE_EPOCHS):
  dev = gp.DeviceGP(0)
  theta, final, status, trace = _run_fused(dev, x, y, z, th0, lo, hi, epochs, n_valid)
  r = th0.shape[0]
  assert theta.shape == th0.shape and final.shape == (r,) and trace.shape == (epochs, r)
  np.testing.assert_array_equal(final, trace[-1])
  idx = range(r) if restarts is None else restarts
  fn = _oracle_fn(x, y, z, n_valid)
  want_th, want_final, want_trace = ao.adam_train(th0[list(idx)], lo, hi, fn, learning_rate=LR, epochs=epochs)
  e_trace = _rel_trace(trace[:, list(idx)], want_trace)
  e_theta = _rel(theta[list(idx)], want_th, lo, hi)
  print(f'kernel vs oracle: loss trace {e_trace:.3e}, final parameters {e_theta:.3e}')
  assert e_trace < 1e-9 and e_theta < 1e-9, (e_trace, e_theta)
  return theta, final, status, trace


@pytest.mark.parametrize('n,n_valid', [(1, 1), (2, 1), (17, 14), (63, 60), (64, 61), (64, 64)])
def test_fused_matches_oracle_across_study_sizes(n, n_valid):
  dc, dk = 3, 2
  x, y, z = _data(n, dc, dk, seed=n)
  lo, hi = gp.param_bounds(dc, dk)
  th0 = _inits(np.random.default_rng(n + 1), dc, dk, 4)
  _check_against_oracle(x, y, z, n_valid, th0, lo, hi)


@pytest.mark.parametrize('dc,dk', [(1, 0), (5, 3), (20, 33), (64, 0), (64, 33), (1, 64)])
def test_fused_matches_oracle_across_feature_counts(dc, dk):
  n = 40
  x, y, z = _data(n, dc, dk, seed=dc + 7 * dk)
  lo, hi = gp.param_bounds(dc, dk)
  th0 = _inits(np.random.default_rng(dc * dk + 2), dc, dk, 3)
  _check_against_oracle(x, y, z, n - 2, th0, lo, hi)


@pytest.mark.parametrize('r', [1, 4, 132, 133])
def test_fused_matches_oracle_across_restart_counts(r):
  """Restarts past the 132 SMs run in a later wave; each CTA's restart is independent, so the oracle replays the first,
  the SM-boundary and the last restarts."""
  dc, dk, n = 4, 1, 20
  x, y, z = _data(n, dc, dk, seed=r)
  lo, hi = gp.param_bounds(dc, dk)
  th0 = _inits(np.random.default_rng(r), dc, dk, r)
  picks = sorted({0, min(r - 1, 131), r - 1})
  theta, final, _, _ = _check_against_oracle(x, y, z, n, th0, lo, hi, restarts=picks)
  assert np.all(np.isfinite(final)) and np.all(np.isfinite(theta))


def test_fused_takes_the_jitter_retry_like_the_oracle():
  """Every trial three times, the fixture's hyper-parameters and a noise variance of 1e-30: K_y is singular to rounding,
  so the first factorisation fails and the first jitter succeeds, on the device and in LAPACK alike (fit_fixtures.py).
  SoftClip resolves 1e-30 only in a box like [1e-40, 1e-20], where it is the difference of two numbers near 1e-20: the
  last bits of exp / log1p then move the noise variance by ~1e-6 relative between implementations, and the
  regulariser carries that into the loss at ~1e-7.  So one evaluation is compared, at 1e-6."""
  n, dc, dk = 30, 2, 1
  x, y, z = ff.tripled(n, dc, dk, seed=5)
  lo, hi = gp.param_bounds(dc, dk)
  lo[dk + dc], hi[dk + dc] = 1e-40, 1e-20
  th0 = np.stack([ff.params(dc, dk, 1e-30, sf2=0.8 * s).to_vector() for s in (1.0, 1.1, 0.9)])
  _, final, status, trace = _run_fused(gp.DeviceGP(0), x, y, z, th0, lo, hi, 1, n)
  np.testing.assert_array_equal(status, 1)
  assert np.all(np.isfinite(final))
  fn = _oracle_fn(x, y, z, n)
  th_eval = ao.soft_clip(ao.soft_clip_inverse(th0, lo, hi), lo, hi)
  for i in range(3):
    assert go.retrying_cholesky(go.kernel_matrix(ff.params(dc, dk, th_eval[i, dk + dc]), x, z))[2] == 1
  want = np.array([fn(t)[0] for t in th_eval])
  np.testing.assert_allclose(trace[0], want, rtol=1e-6)


def test_fused_stops_restarts_whose_retries_are_exhausted():
  """A NaN feature makes every factorisation fail: each restart stops at its first evaluation with retries
  exhausted, a NaN loss for every epoch and the parameters it was evaluated at."""
  n, dc, dk = 12, 2, 0
  x, y, z = _data(n, dc, dk, seed=9)
  x[3, 1] = np.nan
  lo, hi = gp.param_bounds(dc, dk)
  th0 = ard.log_uniform_init(np.random.default_rng(9), dc, dk, 3)
  theta, final, status, trace = _run_fused(gp.DeviceGP(0), x, y, z, th0, lo, hi, 7, n)
  assert np.all(np.isnan(trace)) and np.all(np.isnan(final))
  np.testing.assert_array_equal(status, ff.MAX_RETRIES + 1)
  assert _rel(theta, ard.soft_clip(ard.soft_clip_inverse(th0, lo, hi), lo, hi)[0], lo, hi) < 1e-9
  opt = ard.OptaxTrain(ard.adam(LR), epochs=7)
  dev = gp.DeviceGP(0)
  xt = torch.from_numpy(x).cuda()
  yt = torch.from_numpy(y).cuda()
  _, losses = opt.fit(dev, xt, yt, None, th0, lo, hi, best_n=2)
  assert opt.last_metrics['route'] == 'fused' and np.all(np.isnan(losses))


@pytest.mark.parametrize('dc,dk', [(3, 2), (6, 40)])
def test_fused_loss_equals_make_loss_fn(dc, dk):
  n = 30
  x, y, z = _data(n, dc, dk, seed=3 + dk)
  lo, hi = gp.param_bounds(dc, dk)
  th0 = ard.log_uniform_init(np.random.default_rng(11), dc, dk, 6)
  dev = gp.DeviceGP(0)
  _, _, _, trace = _run_fused(dev, x, y, z, th0, lo, hi, 1, n - 1)
  fn = dev.make_loss_fn(x, y, z, n - 1)
  th_eval, _ = ard.soft_clip(ard.soft_clip_inverse(th0, lo, hi), lo, hi)
  want = np.array([fn(t)[0] for t in th_eval])
  np.testing.assert_allclose(trace[0], want, rtol=1e-13)


@pytest.mark.parametrize('dc,dk', [(3, 2), (5, 36)])
def test_fused_and_host_stepped_agree_over_200_epochs(dc, dk):
  n, r, epochs = 48, 4, 200
  x, y, z = _data(n, dc, dk, seed=21 + dk)
  lo, hi = gp.param_bounds(dc, dk)
  th0 = _inits(np.random.default_rng(22), dc, dk, r)
  dev = gp.DeviceGP(0)
  xt = torch.from_numpy(x).cuda()
  yt = torch.from_numpy(y).cuda()
  zt = torch.from_numpy(z).cuda() if dk else None
  fused = ard.OptaxTrain(ard.adam(5e-2), epochs=epochs)
  best_f, final_f = fused.fit(dev, xt, yt, zt, th0, lo, hi, best_n=r, n_valid=n - 3)
  assert fused.last_metrics['route'] == 'fused'
  host = ard.OptaxTrain(ard.adam(5e-2), epochs=epochs)
  best_h, final_h = host(th0, dev.make_loss_fn(xt, yt, zt, n - 3), list(zip(lo, hi)), best_n=r)
  assert host.last_metrics['route'] == 'host'
  e_trace = _rel_trace(fused.last_metrics['loss'], host.last_metrics['loss'])
  e_theta = _rel(np.array(best_f), np.array(best_h), lo, hi)
  print(f'fused vs host-stepped over {epochs} epochs: loss trace {e_trace:.3e}, final parameters {e_theta:.3e}')
  assert e_trace < 1e-12 and e_theta < 1e-12, (e_trace, e_theta)
  np.testing.assert_array_equal(np.argsort(final_f, kind='stable'), np.argsort(final_h, kind='stable'))
  assert np.all(final_f < fused.last_metrics['loss'][0])


def test_65_trials_take_the_host_stepped_route():
  n, dc, dk = 65, 3, 1
  x, y, z = _data(n, dc, dk, seed=65)
  lo, hi = gp.param_bounds(dc, dk)
  th0 = _inits(np.random.default_rng(65), dc, dk, 4)
  dev = gp.DeviceGP(0)
  opt = ard.OptaxTrain(ard.adam(5e-2), epochs=30)
  xt, yt, zt = (torch.from_numpy(a).cuda() for a in (x, y, z))
  best, final = opt.fit(dev, xt, yt, zt, th0, lo, hi, best_n=2)
  assert opt.last_metrics['route'] == 'host' and opt.last_metrics['loss'].shape == (30, 4)
  fn = _oracle_fn(x, y, z, n)
  want_th, want_final, want_trace = ao.adam_train(th0, lo, hi, fn, learning_rate=5e-2, epochs=30)
  assert _rel_trace(opt.last_metrics['loss'], want_trace) < 1e-9
  assert _rel(best[0], want_th[ao.best_n(want_final, 1)[0]], lo, hi) < 1e-9


# ---------------------------------------------------------------------------------------------------- designers
def _problem(n_metrics):
  p = vz.ProblemStatement()
  p.search_space.root.add_float_param('x0', -2.0, 2.0)
  p.search_space.root.add_float_param('x1', 0.0, 1.0)
  p.search_space.root.add_categorical_param('c', ['a', 'b', 'c'])
  for m in range(n_metrics):
    p.metric_information.append(vz.MetricInformation(name=f'm{m}', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  return p


def _completed(n, n_metrics, seed):
  rng = np.random.default_rng(seed)
  out = []
  for i in range(n):
    t = vz.Trial(parameters={'x0': float(rng.uniform(-2, 2)), 'x1': float(rng.uniform(0, 1)),
                             'c': str(rng.choice(['a', 'b', 'c']))})
    x0, x1 = t.parameters['x0'].value, t.parameters['x1'].value
    t.complete(vz.Measurement({f'm{m}': float(-(x0 - 0.3 * m) ** 2 + np.sin(3 * x1) + 0.05 * rng.normal())
                               for m in range(n_metrics)}))
    out.append(t)
  return out


def _check_suggestions(sugg, count):
  assert len(sugg) == count
  for s in sugg:
    assert -2.0 <= s.parameters['x0'].value <= 2.0 and 0.0 <= s.parameters['x1'].value <= 1.0
    assert s.parameters['c'].value in ('a', 'b', 'c')


def _check_improved(opt, route):
  m = opt.last_metrics
  assert m['route'] == route
  assert np.nanmin(m['final_loss']) < np.nanmin(m['loss'][0])


@pytest.mark.parametrize('n,kw,route', [
    (20, {}, 'fused'),
    (80, {}, 'host'),
    (20, {'ensemble_size': 2}, 'fused'),
    (80, {'ensemble_size': 2}, 'host'),
    (20, {'n_metrics': 2}, 'host'),
    (20, {'linear_coef': 0.1}, 'host'),
])
def test_gp_bandit_with_adam_ard(n, kw, route):
  kw = dict(kw)
  n_metrics = kw.pop('n_metrics', 1)
  opt = ard.OptaxTrain(ard.adam(5e-2), epochs=100)
  d = gp_bandit.VizierGPBandit(_problem(n_metrics), ard_optimizer=opt, rng=3, **kw)
  d.update(vz.CompletedTrials(_completed(n, n_metrics, seed=n)), vz.ActiveTrials())
  _check_suggestions(d.suggest(2), 2)
  _check_improved(opt, route)


@pytest.mark.parametrize('n_metrics,route', [(1, 'fused'), (2, 'host')])
def test_gp_ucb_pe_with_adam_ard(n_metrics, route):
  opt = ard.OptaxTrain(ard.adam(5e-2), epochs=100)
  d = gp_ucb_pe.VizierGPUCBPEBandit(_problem(n_metrics), ard_optimizer=opt, rng=4)
  d.update(vz.CompletedTrials(_completed(24, n_metrics, seed=24)), vz.ActiveTrials())
  _check_suggestions(d.suggest(3), 3)
  _check_improved(opt, route)
  assert opt.last_metrics['loss'].shape == (100, 5)   # 1 fixed + 4 random initial points


def test_gp_bandit_with_adam_ard_trains_every_level_of_a_prior_stack():
  opt = ard.OptaxTrain(ard.adam(5e-2), epochs=100)
  d = gp_bandit.VizierGPBandit(_problem(1), ard_optimizer=opt, rng=5)
  d.set_priors([vz.CompletedTrials(_completed(30, 1, seed=30))])
  _check_improved(opt, 'fused')                    # the prior level
  d.update(vz.CompletedTrials(_completed(10, 1, seed=10)), vz.ActiveTrials())
  _check_suggestions(d.suggest(2), 2)
  _check_improved(opt, 'fused')                    # the current study's level, on the residuals


@pytest.mark.parametrize('kw,route', [({'ensemble_size': 2}, 'fused'), ({'mixes_linear_kernel': True}, 'host')])
def test_gp_ucb_pe_ensemble_and_linear_kernel_with_adam_ard(kw, route):
  """The linear kernel's fixed initial point has its slope on the lower bound: it maps to a finite unconstrained
  coordinate and its restart trains like the others."""
  opt = ard.OptaxTrain(ard.adam(5e-2), epochs=100)
  d = gp_ucb_pe.VizierGPUCBPEBandit(_problem(1), ard_optimizer=opt, rng=6, **kw)
  d.update(vz.CompletedTrials(_completed(24, 1, seed=25)), vz.ActiveTrials())
  _check_suggestions(d.suggest(3), 3)
  _check_improved(opt, route)
  assert opt.last_metrics['loss'].shape == (100, 5) and np.all(np.isfinite(opt.last_metrics['loss']))


def test_wide_models_past_one_ctas_shared_memory_take_the_host_stepped_route():
  """The widest categorical model the fused kernel holds at Dc = 1 runs fused; one feature more needs more than the
  227 KiB a CTA may use, and `fit` takes the host-stepped route instead of failing the launch."""
  from vizier_b200 import _lib
  supported = _lib.load().vzgp_ard_adam_small_supported
  dc = 1
  dk = max(k for k in range(33, 1025) if supported(64, dc, k))
  dev = gp.DeviceGP(0)
  for k, route in ((dk, 'fused'), (dk + 1, 'host')):
    x, y, z = _data(12, dc, k, seed=k)
    lo, hi = gp.param_bounds(dc, k)
    th0 = _inits(np.random.default_rng(k), dc, k, 2)
    opt = ard.OptaxTrain(ard.adam(LR), epochs=5)
    xt, yt, zt = (torch.from_numpy(a).cuda() for a in (x, y, z))
    _, final = opt.fit(dev, xt, yt, zt, th0, lo, hi, best_n=1)
    assert opt.last_metrics['route'] == route and np.all(np.isfinite(final))
    want_th, want_final, want_trace = ao.adam_train(th0, lo, hi, _oracle_fn(x, y, z, 12), learning_rate=LR, epochs=5)
    assert _rel_trace(opt.last_metrics['loss'], want_trace) < 1e-9
