"""The wgmma integer-split scoring kernel (score_i8.cu) against the oracle and against the DMMA kernel.

`vzgp_set_int(h, "score_i8", 1)` routes pools of at least one 64-candidate tile per SM through `k_score_i8`
(exact int8 digit products with int32 accumulation in registers, recombined in fp64); everything else about the
call is unchanged, so the same oracle checks apply with the same tolerances.
"""
import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from oracle import gp_oracle as go  # noqa: E402

TOL = 1e-10


@pytest.fixture()
def dev():
  from vizier_b200 import gp
  d = gp.DeviceGP(0)
  yield d
  d.close()


def _gp():
  from vizier_b200 import gp
  return gp


def _problem(n, d, seed=0, dk=0):
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, d))
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  z = rng.integers(0, 4, size=(n, dk)).astype(np.int32) if dk else None
  return x, y, z


def _params(d, dk=0, sf2=1.0, sn2=1e-3, ls=None):
  ls2 = 0.5 * (1 + np.arange(d) / d) if ls is None else np.full(d, ls)
  lk = np.linspace(0.6, 1.4, dk) if dk else None
  return go.GPParams(sf2, ls2, sn2, lk), _gp().GPHyperParams(sf2, ls2, sn2, lk)


def _pool(dev, m, d, seed):
  return dev.random_pool(m, d, seed=seed)


def _i8_tiles(dev):
  """64-candidate tiles of a pool the integer-split kernel takes: at least one per SM (148 on a 132-SM H100)."""
  return dev.get_int('sm_count') + 16


@pytest.mark.parametrize('n,d,sf2', [(1000, 20, 1.0), (520, 7, 2.7), (192, 3, 0.31), (1030, 12, 1.0), (300, 40, 1.0),
                                     (2000, 50, 0.9999999), (300, 64, 1.0)])
def test_i8_scores_match_oracle_and_dmma(dev, n, d, sf2):
  """np = 1024 / 576 (a half k chunk) / 192 / 1088; sf2 off a power of two; Dc = 40 and 50: one phase-1 trial
  buffer; Dc = 64: the phase-1 staging no longer fits next to the operand ring (nbuf = 1, phases back to back); C4's
  N = 2000 with sf2 just below a power of two (the balanced top digit needs the extra scale bit)."""
  m = _i8_tiles(dev) * 64 + 37     # one tile more than SMs + 16: some CTAs reuse their digit buffers
  x, y, _ = _problem(n, d, n)
  po, pg = _params(d, sf2=sf2)
  dev.fit(x, y, pg)
  xs = _pool(dev, m, d, seed=5)
  acq = _gp().Acquisition(1.8, True, go.trust_radius(n, d, 0))
  dev.set_int('score_i8', 0)
  ref = dev.score(xs, acq, with_aux=True)
  assert dev.get_int('score_route') == 2
  dev.set_int('score_i8', 1)
  out = dev.score(xs, acq, with_aux=True)
  assert dev.get_int('score_route') == 3 and dev.get_int('score_grid') == dev.get_int('sm_count')
  dev.synchronize()
  pred = go.precompute_predictive(po, x, y)
  sel = np.r_[0:256, m - 300:m]
  want, aux = go.score_with_aux(pred, xs.cpu().numpy()[sel])
  np.testing.assert_allclose(out['stddev'].cpu().numpy()[sel], aux['stddev'], atol=TOL, rtol=0)
  np.testing.assert_allclose(out['mean'].cpu().numpy()[sel], aux['mean'], atol=TOL, rtol=0)
  np.testing.assert_allclose(out['score'].cpu().numpy()[sel], want, atol=TOL, rtol=0)
  # the two device kernels on the whole pool: the mean differs by its summation order only, sigma agrees far below TOL
  np.testing.assert_allclose(out['mean'].cpu().numpy(), ref['mean'].cpu().numpy(), atol=1e-11, rtol=0)
  np.testing.assert_array_equal(out['linf_distance'].cpu().numpy(), ref['linf_distance'].cpu().numpy())
  np.testing.assert_allclose(out['stddev'].cpu().numpy(), ref['stddev'].cpu().numpy(), atol=1e-11, rtol=0)
  # throughput variant (no aux, pre-scaled features)
  fast = dev.score(xs, acq)
  dev.synchronize()
  np.testing.assert_allclose(fast['score'].cpu().numpy()[sel], want, atol=TOL, rtol=0)


def test_i8_ill_conditioned_and_categorical(dev):
  """sn2 = 1e-8 (Linv entries ~1e4, cancellation in W) and mixed continuous / categorical features."""
  n, d, m = 600, 6, _i8_tiles(dev) * 64
  x, y, _ = _problem(n, d, 3)
  po, pg = _params(d, sn2=1e-8, ls=0.05)
  dev.fit(x, y, pg)
  xs = _pool(dev, m, d, seed=9)
  acq = _gp().Acquisition(1.8, False, 0.0)
  dev.set_int('score_i8', 1)
  out = dev.score(xs, acq, with_aux=True)
  dev.set_int('score_i8', 0)
  ref = dev.score(xs, acq, with_aux=True)
  dev.synchronize()
  pred = go.precompute_predictive(po, x, y)
  sel = np.arange(512)
  _, sd_w = go.predict(pred, xs.cpu().numpy()[sel])
  np.testing.assert_allclose(out['stddev'].cpu().numpy()[sel], sd_w, atol=1e-7, rtol=0)
  # against the DMMA kernel the integer split must not be worse than fp64 accumulation itself
  np.testing.assert_allclose(out['stddev'].cpu().numpy(), ref['stddev'].cpu().numpy(), atol=1e-7, rtol=0)

  n, d, dk = 300, 5, 2
  x, y, z = _problem(n, d, 4, dk=dk)
  po, pg = _params(d, dk=dk)
  dev.fit(x, y, pg, z=z)
  rng = np.random.default_rng(1)
  xs = torch.from_numpy(rng.uniform(size=(m, d))).cuda()
  zs = torch.from_numpy(rng.integers(0, 4, size=(m, dk)).astype(np.int32)).cuda()
  acq = _gp().Acquisition(1.8, True, go.trust_radius(n, d + dk, 0))
  dev.set_int('score_i8', 1)
  out = dev.score(xs, acq, zs=zs, with_aux=True)
  dev.synchronize()
  pred = go.precompute_predictive(po, x, y, z=z)
  want, aux = go.score_with_aux(pred, xs.cpu().numpy()[:300], zs=zs.cpu().numpy()[:300])
  np.testing.assert_allclose(out['score'].cpu().numpy()[:300], want, atol=TOL, rtol=0)
  np.testing.assert_allclose(out['stddev'].cpu().numpy()[:300], aux['stddev'], atol=TOL, rtol=0)


def test_i8_refit_invalidates_digit_planes(dev):
  """A second fit on the same handle (new Linv) must re-slice; a pool too small for the path falls back."""
  n, d, m = 256, 4, _i8_tiles(dev) * 64
  acq = _gp().Acquisition(1.8, False, 0.0)
  dev.set_int('score_i8', 1)
  for seed in (1, 2):
    x, y, _ = _problem(n, d, seed)
    po, pg = _params(d, sn2=1e-2 * seed)
    dev.fit(x, y, pg)
    xs = _pool(dev, m, d, seed=seed)
    out = dev.score(xs, acq, with_aux=True)
    small = dev.score(xs[:1000], acq, with_aux=True)   # 16 tiles: DMMA / small-pool kernels
    dev.synchronize()
    pred = go.precompute_predictive(po, x, y)
    _, aux = go.score_with_aux(pred, xs.cpu().numpy()[:500])
    np.testing.assert_allclose(out['stddev'].cpu().numpy()[:500], aux['stddev'], atol=TOL, rtol=0)
    np.testing.assert_allclose(small['stddev'].cpu().numpy()[:500], aux['stddev'], atol=TOL, rtol=0)


def test_i8_two_handles_on_two_streams_concurrently():
  """Two models scoring large pools at the same time from two host threads (separate handles and streams): the
  kernels take turns on the SMs (one CTA per SM: shared memory and registers); results equal the serial ones."""
  import threading
  gp = _gp()
  devs, pools, want = [], [], []
  for k in range(2):
    n, d = 400 + 300 * k, 6 + 4 * k
    x, y, _ = _problem(n, d, 40 + k)
    _, pg = _params(d, sf2=1.0 + k)
    dv = gp.DeviceGP(0)
    dv.set_int('score_i8', 1)
    dv.fit(x, y, pg)
    xs = dv.random_pool(_i8_tiles(dv) * 64 * 3, d, seed=k)
    ref = dv.score(xs, gp.Acquisition(1.8, False, 0.0), with_aux=True)
    dv.synchronize()
    devs.append(dv); pools.append(xs); want.append(ref['stddev'].clone())
  got = [None, None]

  def run(k):
    for _ in range(5):
      out = devs[k].score(pools[k], gp.Acquisition(1.8, False, 0.0), with_aux=True)
    devs[k].synchronize()
    got[k] = out['stddev']

  ts = [threading.Thread(target=run, args=(k,)) for k in range(2)]
  [t.start() for t in ts]; [t.join() for t in ts]
  for k in range(2):
    assert devs[k].get_int('score_i8_launches') >= 6
    np.testing.assert_array_equal(got[k].cpu().numpy(), want[k].cpu().numpy())
    devs[k].close()
