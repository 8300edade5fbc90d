"""k_score's fast instance (no trust-region distance) forms d^2 = |a_c|^2 + |b_c|^2 - 2 a_c.b_c on the DMMA pipe, from
features centred on the midpoint of the trials' range and scaled by 1/ls.  These tests run it through the public API
on the cluster route and hold it to the route tests' tolerances: against oracle/gp_oracle.py, against the trust-region
instance (which keeps the difference-first d^2) and, on an ill-conditioned model, against the long-double posterior."""
import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from oracle import gp_oracle as go  # noqa: E402
from oracle import hp_oracle as hp  # noqa: E402
import test_gpu_score_routes as routes  # noqa: E402

CLUSTER = routes.CLUSTER


def _gp():
  from vizier_b200 import gp
  return gp


@pytest.fixture(scope='module')
def dev():
  d = _gp().DeviceGP(0)
  d.set_int('score_i8', 0)
  d.set_int('small_tiles', -1)
  yield d
  d.close()


def _pool_size(dev):
  # more tiles than half the SMs: the cluster route without a column split
  return (dev.get_int('sm_count') // 2 + 40) * 64


def _score_both(dev, xs, zs=None):
  """The fast instance (mean and stddev, no distance) and the trust-region-distance instance on one pool."""
  gp = _gp()
  acq = gp.Acquisition(1.8, False, 1.0)
  m = xs.shape[0]
  xst = torch.from_numpy(xs).cuda()
  zst = torch.from_numpy(zs).cuda() if zs is not None else None
  out = {k: torch.empty(m, dtype=torch.float64, device=dev.device) for k in ('score', 'mean', 'stddev')}
  dev.score(xst, acq, zs=zst, out=out)
  dev.synchronize()
  assert dev.get_int('score_route') == CLUSTER
  fast = {k: out[k].cpu().numpy().copy() for k in ('score', 'mean', 'stddev')}
  aux = dev.score(xst, acq, zs=zst, with_aux=True)
  dev.synchronize()
  assert dev.get_int('score_route') == CLUSTER
  return fast, {k: aux[k].cpu().numpy().copy() for k in ('score', 'mean', 'stddev')}


def _check(fast, aux, pred, xs, zs=None):
  mu, sd = go.predict(pred, xs, zs)
  want = {'score': go.ucb(mu, sd, 1.8), 'mean': mu, 'stddev': sd}
  for k in ('score', 'mean', 'stddev'):
    assert np.all(np.isfinite(fast[k])), k
    np.testing.assert_allclose(fast[k], want[k], atol=routes.TOL, rtol=0, err_msg=k)
  np.testing.assert_allclose(fast['score'], aux['score'], atol=routes._variant_tol(pred), rtol=0)


def _fit(dev, x, y, ls2, z=None, lk=None, sf2=1.0, sn2=1e-3):
  gp = _gp()
  assert dev.fit(x, y, gp.GPHyperParams(sf2, ls2, sn2, lk), z=z) == 0
  return go.precompute_predictive(go.GPParams(sf2, ls2, sn2, lk), x, y, z)


def test_features_far_from_the_origin(dev):
  """Trials in [1e3, 1e3 + 1]^5: uncentred, |a|^2 / ls^2 ~ 1e7 would cost ~1e-9 of d^2 to cancellation."""
  rng = np.random.default_rng(3)
  n, d = 300, 5
  x = 1e3 + rng.uniform(size=(n, d))
  y = -np.sum((x - 1e3 - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  m = _pool_size(dev)
  xs = 1e3 + rng.uniform(-0.5, 1.5, size=(m, d))
  near = rng.permutation(m)[:m // 3]
  xs[near] = x[rng.integers(0, n, near.size)] + rng.uniform(-0.04, 0.04, size=(near.size, d))
  pred = _fit(dev, x, y, 0.5 * (1 + np.arange(d) / d))
  fast, aux = _score_both(dev, xs)
  _check(fast, aux, pred, xs)


@pytest.mark.parametrize('offset', [0.0, 1e3])
def test_candidates_equal_to_trials(dev, offset):
  """Every trial scored as a candidate: d^2 of the pair is 0 up to rounding; below zero the Matern takes it as 0."""
  rng = np.random.default_rng(5)
  n, d = 250, 7
  x = offset + rng.uniform(size=(n, d))
  y = -np.sum((x - offset - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  m = _pool_size(dev)
  xs = x[np.arange(m) % n].copy()
  pred = _fit(dev, x, y, 0.5 * (1 + np.arange(d) / d))
  fast, aux = _score_both(dev, xs)
  _check(fast, aux, pred, xs)
  np.testing.assert_allclose(fast['stddev'], aux['stddev'], atol=routes.TOL, rtol=0)


@pytest.mark.skipif(not hp.has_extended_precision(), reason='np.longdouble is fp64 on this platform')
def test_ill_conditioned_vs_long_double(dev):
  """sn2 = 1e-8, ls2 = 0.05 and duplicated trials (cond(K_y) ~ 1e10): the fast instance's mean is as accurate as
  fp64 LAPACK against a long-double reference, its stddev within the route tests' bounds."""
  gp = _gp()
  n, d = 300, 6
  rng = np.random.default_rng(77)
  x = rng.uniform(size=(n, d))
  x[1::10] = x[0::10]
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  ls2 = np.full(d, 0.05)
  po = go.GPParams(1.0, ls2, 1e-8)
  m = _pool_size(dev)
  xs = rng.uniform(size=(m, d))
  near = rng.permutation(m)[:m // 4]
  xs[near] = x[rng.integers(0, n, near.size)] + rng.uniform(-0.02, 0.02, size=(near.size, d))
  mu_h, sd_h = hp.predict(hp.precompute_predictive(po, x, y), xs)
  mu_f, sd_f = go.predict(go.precompute_predictive(po, x, y), xs)
  assert dev.fit(x, y, gp.GPHyperParams(1.0, ls2, 1e-8)) == 0
  fast, _ = _score_both(dev, xs)

  def errs(v, ref):
    e = np.abs((np.asarray(v, np.longdouble) - ref).astype(np.float64))
    return float(e.max()), float(np.sqrt(np.mean(e * e)))

  gm, gr = errs(fast['mean'], mu_h)
  fm, fr = errs(mu_f, mu_h)
  assert gm <= routes.HARD_FACTOR * fm + routes.HARD_FLOOR, (gm, fm)
  assert gr <= routes.HARD_FACTOR * fr + routes.HARD_FLOOR, (gr, fr)
  sm, sr = errs(fast['stddev'], sd_h)
  assert sm <= routes.HARD_SD_MAX and sr <= routes.HARD_SD_RMS, (sm, sr)


@pytest.mark.parametrize('dc,dk', [(1, 0), (7, 0), (8, 0), (9, 3), (45, 0), (46, 0), (61, 0), (62, 3), (64, 0)])
def test_feature_counts(dev, dc, dk):
  """dc around the k-step of 8 (dimensions past dc are zero on both operands) and at the phase-1 staging plan's
  switches (45 / 46 and 61 / 62); with categorical features added to d^2 after the DMMAs at two of them."""
  rng = np.random.default_rng(100 + dc)
  n = 200
  x = rng.uniform(size=(n, dc))
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  z = rng.integers(0, 4, size=(n, dk)).astype(np.int32) if dk else None
  m = _pool_size(dev)
  xs = rng.uniform(-0.5, 1.5, size=(m, dc))
  near = rng.permutation(m)[:m // 3]
  src = rng.integers(0, n, near.size)
  xs[near] = x[src] + rng.uniform(-0.04, 0.04, size=(near.size, dc))
  xs[:3] = x[:3]
  zs = None
  if dk:
    zs = rng.integers(0, 4, size=(m, dk)).astype(np.int32)
    zs[near] = z[src]
    zs[:3] = z[:3]
  # length scales that grow with dc keep K* away from zero at every dc
  ls2 = 0.5 * (1 + np.arange(dc) / dc) * max(1.0, dc / 8)
  pred = _fit(dev, x, y, ls2, z=z, lk=routes.LK3[:dk] if dk else None)
  fast, aux = _score_both(dev, xs, zs)
  _check(fast, aux, pred, xs, zs)


def test_non_finite_candidate_is_not_a_winner(dev):
  """A NaN feature makes that candidate's d^2, and so its score, NaN, as in the difference-first form; top-1 skips it."""
  gp = _gp()
  rng = np.random.default_rng(11)
  n, d = 200, 5
  x = rng.uniform(size=(n, d))
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  m = _pool_size(dev)
  xs = rng.uniform(size=(m, d))
  pred = _fit(dev, x, y, 0.5 * (1 + np.arange(d) / d))
  mu, sd = go.predict(pred, xs)
  want = go.ucb(mu, sd, 1.8)
  best = int(np.argmax(want))
  xs[best, 2] = np.nan
  out = {k: torch.empty(m, dtype=torch.float64, device=dev.device) for k in ('score', 'mean', 'stddev')}
  dev.score(torch.from_numpy(xs).cuda(), gp.Acquisition(1.8, False, 1.0), out=out)
  dev.synchronize()
  assert dev.get_int('score_route') == CLUSTER
  got = out['score'].cpu().numpy()
  assert np.isnan(got[best])
  rest = np.arange(m) != best
  np.testing.assert_allclose(got[rest], want[rest], atol=routes.TOL, rtol=0)
  idx, _ = dev.topk(out['score'], 1)
  assert int(idx[0]) == int(np.argmax(np.where(rest, want, -np.inf)))
