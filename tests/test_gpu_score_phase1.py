"""k_score's phase 1 builds K* with the branch-free Matern of matern_fast.cuh; the small route keeps the libm
Matern.  These tests pin the fast Matern through the public API and check that scores do not move."""
import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from oracle import hp_oracle as hp  # noqa: E402

SMALL, CLUSTER = 0, 2   # vzgp_score_route (include/vzgp.h)


def _gp():
  from vizier_b200 import gp
  return gp


@pytest.fixture(scope='module')
def dev():
  d = _gp().DeviceGP(0)
  d.set_int('score_i8', 0)
  yield d
  d.close()


def _route_tiles(dev):
  # more tiles than half the SMs: the cluster route without a column split
  return dev.get_int('sm_count') // 2 + 40


@pytest.mark.skipif(not hp.has_extended_precision(), reason='np.longdouble is fp64 on this platform')
@pytest.mark.parametrize('sf2', [1.0, 2.7])
@pytest.mark.parametrize('aux', [False, True])
def test_fast_matern_mean_within_4_ulp(dev, sf2, aux):
  """One trial at the origin, candidates on one axis: mu = k(d2) alpha with d2 = x^2 swept densely over
  [0, 2e5], d2 = 0 exactly and s = sqrt(5 d2) just below and above 708.  With one trial the 64-column step
  straddles n_valid.  aux=True runs the trust-region-distance instance of k_score."""
  gp = _gp()
  x = np.zeros((1, 1))
  assert dev.fit(x, np.array([0.7]), gp.GPHyperParams(sf2, np.ones(1), 1e-3)) == 0
  alpha = float(dev.alpha().cpu().numpy()[0])
  m = _route_tiles(dev) * 64
  edge = np.array([0.0, 708.0 - 1e-9, 708.0 - 1e-12, 708.0, 708.0 + 1e-12, 708.0 + 1e-9]) ** 2 / 5.0
  d2_want = np.concatenate([edge, np.linspace(0.0, 2e5, m - edge.size)])
  xs = np.sqrt(d2_want)[:, None]
  d2 = xs[:, 0] * xs[:, 0]                    # what the kernel forms: (x - 0)^2, rounded once
  out = {k: torch.empty(m, dtype=torch.float64, device=dev.device) for k in ('score', 'mean', 'stddev')}
  if aux:
    out['linf_distance'] = torch.empty(m, dtype=torch.float64, device=dev.device)
  dev.set_int('small_tiles', 0)
  try:
    dev.score(torch.from_numpy(xs).cuda(), gp.Acquisition(1.8, False, 1.0), out=out)
    dev.synchronize()
    assert dev.get_int('score_route') == CLUSTER
  finally:
    dev.set_int('small_tiles', -1)
  mu = out['mean'].cpu().numpy()
  s = np.sqrt(5.0 * d2)                       # IEEE sqrt, as the fast sequence rounds
  S = s.astype(np.longdouble)
  k_ref = np.longdouble(sf2) * (1 + S + S * S / 3) * np.exp(-S)
  want = k_ref * np.longdouble(alpha)
  # 4 ulp of k, scaled by alpha, plus the rounding of the product k * alpha
  tol = 4 * np.spacing(np.abs(k_ref.astype(np.float64))) * abs(alpha) + 0.5 * np.spacing(np.abs(mu))
  above = s > 708.0
  assert above.sum() >= 2 and (~above).sum() > 1000
  err = np.abs((mu.astype(np.longdouble) - want)).astype(np.float64)
  bad = np.flatnonzero(~above & (err > tol))
  assert bad.size == 0, (bad[:5], d2[bad[:5]], err[bad[:5]], tol[bad[:5]])
  np.testing.assert_array_equal(mu[above], 0.0)
  assert mu[0] == np.float64(sf2) * np.float64(alpha)   # d2 = 0: k = sf2 exactly


def _scores_two_routes(dev, xs, acq):
  res = {}
  for route, small_tiles in ((CLUSTER, 0), (SMALL, 1 << 30)):
    dev.set_int('small_tiles', small_tiles)
    try:
      c0 = dev.clamped_count()
      out = dev.score(torch.from_numpy(xs).cuda(), acq, with_aux=True)
      dev.synchronize()
      assert dev.get_int('score_route') == route
      res[route] = ({k: out[k].cpu().numpy() for k in ('score', 'mean', 'stddev')}, dev.clamped_count() - c0)
    finally:
      dev.set_int('small_tiles', -1)
  return res[CLUSTER], res[SMALL]


def test_c2_pool_fast_matern_matches_libm_route(dev):
  """The C2 pool (N=1000, D=20, M=100k) scored by k_score and by the small route (libm Matern).  The accuracy of
  the cluster route on an ill-conditioned model is checked against long double in test_gpu_score_routes."""
  gp = _gp()
  rng = np.random.default_rng(0)
  n, d, m = 1000, 20, 100_000
  x = rng.uniform(size=(n, d))
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  assert dev.fit(x, y, gp.GPHyperParams(1.0, 0.5 * (1 + np.arange(d) / d), 1e-3)) == 0
  xs = rng.uniform(size=(m, d))
  (fast, c_fast), (ref, c_ref) = _scores_two_routes(dev, xs, gp.Acquisition(1.8, False, 0.0))
  diff = float(np.max(np.abs(fast['score'] - ref['score'])))
  print(f'C2 max |score(k_score) - score(small route)| = {diff:.3e}')
  assert diff <= 1e-12
  assert c_fast == c_ref
  assert int(np.argmax(fast['score'])) == int(np.argmax(ref['score']))

