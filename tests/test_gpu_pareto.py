"""Pareto dominance, Pareto rank and the cumulative hypervolume on the device (vizier_b200.multimetric, pareto.cu)
against oracle/pareto_oracle.py.

Dominance and rank are comparisons, so they must equal the oracle exactly, on integer data dense in ties and duplicate
rows, with NaN and +-inf coordinates, at every row count around the kernels' CTA (256 points) and slab (4096 / kM
rows, kM = M rounded up to a power of two) boundaries.  The hypervolume matches the oracle to rtol 1e-12 and repeats
bit for bit."""
import json
import os

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from oracle import pareto_oracle as po  # noqa: E402

G = json.load(open(os.path.join(os.path.dirname(__file__), 'golden', 'pareto_known_answers.json')))
SIZES = [0, 1, 31, 32, 33, 255, 256, 257, 4097]
METRICS = [1, 2, 3, 8, 64]


def _mm():
  from vizier_b200 import multimetric
  return multimetric


def _dense(rng, n, m):
  """Integer-valued rows in {0, 1, 2}: ties everywhere, a quarter of the rows raised copies of others (dominators at
  any M), an eighth exact duplicates, and NaN / +inf / -inf coordinates in up to 60 rows."""
  x = rng.integers(0, 3, size=(n, m)).astype(np.float64)
  k = n // 4
  x[rng.integers(0, n, size=k)] = x[rng.integers(0, n, size=k)] + rng.integers(0, 2, size=(k, m))
  k = n // 8
  x[rng.integers(0, n, size=k)] = x[rng.integers(0, n, size=k)]
  for t, i in enumerate(rng.choice(n, size=min(n, 60), replace=False)):
    x[i, rng.integers(0, m)] = (np.nan, np.inf, -np.inf)[t % 3]
  return x


@pytest.mark.parametrize('m', METRICS)
@pytest.mark.parametrize('strict', [True, False])
def test_optimal_against_equals_oracle(m, strict):
  mm = _mm()
  rng = np.random.default_rng(100 + m)
  pts, against = _dense(rng, max(SIZES), m), _dense(rng, max(SIZES), m)
  against[:40] = pts[:40]   # shared rows: equal pairs across the two sets
  # the first dominating row of `against` for each point: against[:b2] dominates point i iff first[i] < b2
  d = po.domination_matrix(pts, against, strict)
  first = np.where(d.any(axis=1), d.argmax(axis=1), len(against))
  for b1 in SIZES:
    for b2 in SIZES:
      got = mm.is_pareto_optimal_against(pts[:b1], against[:b2], strict=strict)
      assert got.dtype == bool and got.shape == (b1,)
      np.testing.assert_array_equal(got, first[:b1] >= b2, err_msg=f'B1={b1} B2={b2}')
  np.testing.assert_array_equal(mm.is_pareto_optimal_against(pts[:257], against[:4097], strict=strict),
                                po.is_pareto_optimal_against(pts[:257], against[:4097], strict))


@pytest.mark.parametrize('m', METRICS)
def test_frontier_and_rank_equal_oracle(m):
  mm = _mm()
  pts = _dense(np.random.default_rng(200 + m), max(SIZES), m)
  d = po.domination_matrix(pts, pts, strict=True)
  for b in SIZES:
    rank = mm.pareto_rank(pts[:b])
    assert rank.dtype == np.int32 and rank.shape == (b,)
    np.testing.assert_array_equal(rank, d[:b, :b].sum(axis=1), err_msg=f'B={b}')
    np.testing.assert_array_equal(mm.is_frontier(pts[:b]), ~d[:b, :b].any(axis=1), err_msg=f'B={b}')
  np.testing.assert_array_equal(mm.pareto_rank(pts[:300]), po.pareto_rank(pts[:300]))
  np.testing.assert_array_equal(mm.get_frontier(pts[:300]), pts[:300][po.is_frontier(pts[:300])])


def test_known_answers():
  mm = _mm()
  g = G['pareto_rank']
  np.testing.assert_array_equal(mm.pareto_rank(np.array(g['ys'])), g['rank'])
  g = G['is_pareto_optimal']
  np.testing.assert_array_equal(mm.is_frontier(np.array(g['points'])), g['optimal'])
  np.testing.assert_array_equal(mm.is_frontier(np.vstack([g['points'], g['added']])), g['optimal_with_added'])
  g = G['is_pareto_optimal_against']
  for strict, key in ((True, 'strict'), (False, 'non_strict')):
    np.testing.assert_array_equal(mm.is_pareto_optimal_against(np.array(g['points']), np.array(g['against']),
                                                                strict=strict), g[key])
  g = G['update_pareto_optimal']
  np.testing.assert_array_equal(mm.DeviceParetoOptimalAlgorithm().update_pareto_optimal(
      np.array(g['current'], float), np.array(g['incremental'], float)), g['indices'])


def test_random_frontier_is_a_staircase():
  mm = _mm()
  ys = np.random.default_rng(7).random((20000, 2))
  on = mm.is_frontier(ys, num_shards=5)
  np.testing.assert_array_equal(on, po.is_frontier(ys))
  frontier = mm.get_frontier(ys, num_shards=5)
  assert frontier.shape[0] == np.sum(on)
  sid = frontier[:, 0].argsort()
  np.testing.assert_array_equal(frontier[sid, 1].argsort(), np.arange(len(frontier) - 1, -1, -1))
  np.testing.assert_array_equal(mm.pareto_rank(ys), po.pareto_rank(ys))


def test_tensors_in_tensors_out():
  mm = _mm()
  pts = _dense(np.random.default_rng(3), 1000, 3)
  t = torch.from_numpy(pts).cuda()
  got = mm.is_frontier(t)
  assert isinstance(got, torch.Tensor) and got.dtype == torch.bool and got.device == t.device
  np.testing.assert_array_equal(got.cpu().numpy(), po.is_frontier(pts))
  rank = mm.pareto_rank(t)
  assert rank.dtype == torch.int32
  np.testing.assert_array_equal(rank.cpu().numpy(), po.pareto_rank(pts))
  np.testing.assert_array_equal(mm.get_frontier(t).cpu().numpy(), pts[po.is_frontier(pts)])
  vec = np.abs(np.random.default_rng(4).normal(size=(300, 3)))
  hv = mm.cum_hypervolume_origin(t.abs(), torch.from_numpy(vec).cuda())
  assert isinstance(hv, torch.Tensor) and hv.dtype == torch.float64
  np.testing.assert_allclose(hv.cpu().numpy(), po.cum_hypervolume_origin(np.abs(pts), vec), rtol=1e-12)


def test_device_errors():
  from vizier_b200 import _lib
  from vizier_b200 import gp
  dev = gp.DeviceGP(0)
  p = torch.zeros((4, 65), dtype=torch.float64, device='cuda')
  out = torch.zeros(4, dtype=torch.int32, device='cuda')
  st = dev._lib.vzgp_pareto_rank(dev._h, p.data_ptr(), 4, 65, out.data_ptr())
  assert st == _lib.VZGP_ERR_ARG
  st = dev._lib.vzgp_pareto_optimal_against(dev._h, p.data_ptr(), 4, p.data_ptr(), -1, 2, 1, out.data_ptr())
  assert st == _lib.VZGP_ERR_ARG
  st = dev._lib.vzgp_cum_hypervolume_origin(dev._h, p.data_ptr(), 4, 0, p.data_ptr(), 4, out.data_ptr())
  assert st == _lib.VZGP_ERR_ARG
  # row counts past 2^30, and partial sums past the 256 MiB scratch even at the widest CTAs, are refused
  big = (1 << 30) + 1
  assert dev._lib.vzgp_pareto_rank(dev._h, p.data_ptr(), big, 2, out.data_ptr()) == _lib.VZGP_ERR_ARG
  assert dev._lib.vzgp_pareto_optimal_against(dev._h, p.data_ptr(), 4, p.data_ptr(), big, 2, 1,
                                              out.data_ptr()) == _lib.VZGP_ERR_ARG
  assert dev._lib.vzgp_cum_hypervolume_origin(dev._h, p.data_ptr(), 4, 2, p.data_ptr(), big,
                                              out.data_ptr()) == _lib.VZGP_ERR_ARG
  assert dev._lib.vzgp_cum_hypervolume_origin(dev._h, p.data_ptr(), (1 << 25) + 1, 2, p.data_ptr(), 4,
                                              out.data_ptr()) == _lib.VZGP_ERR_ARG
  # empty inputs do nothing
  assert dev._lib.vzgp_pareto_rank(dev._h, None, 0, 2, None) == 0
  assert dev._lib.vzgp_cum_hypervolume_origin(dev._h, None, 0, 2, None, 0, None) == 0
  dev.close()


def _directions(rng, v, m):
  u = np.abs(rng.normal(size=(v, m)))
  return u / np.linalg.norm(u, axis=1)[:, None]


@pytest.mark.parametrize('n,v,m', [(1, 1, 1), (255, 257, 2), (257, 31, 3), (4097, 1000, 8), (1000, 300, 64),
                                   (10000, 10000, 2), (10000, 10000, 3)])
def test_cum_hypervolume_equals_oracle(n, v, m):
  mm = _mm()
  rng = np.random.default_rng(n + v + m)
  pts = rng.uniform(0.0, 2.0, size=(n, m))
  vec = _directions(rng, v, m)
  want = po.cum_hypervolume_origin(pts, vec)
  got = mm.cum_hypervolume_origin(pts, vec)
  np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
  assert np.array_equal(mm.jax_cum_hypervolume_origin(pts, vec), got)   # bit for bit on a second call


def test_cum_hypervolume_wide_ctas_and_growing_scratch():
  """N = 2 x 10^5 with V = 2000 would need 400 MB of partial sums at four CTAs per SM, so the launcher gives each CTA
  more vectors; calls of growing N on one handle replace its scratch between them."""
  mm = _mm()
  rng = np.random.default_rng(21)
  vec = _directions(rng, 2000, 2)
  for n in (1000, 20_000, 200_000):
    pts = rng.uniform(0.0, 2.0, size=(n, 2))
    np.testing.assert_allclose(mm.cum_hypervolume_origin(pts, vec), po.cum_hypervolume_origin(pts, vec), rtol=1e-12,
                               atol=0, err_msg=f'N={n}')


def test_concurrent_calls_from_threads():
  """Threads share the module's handle: calls of different sizes at the same time each get their own answer."""
  import threading
  mm = _mm()
  rng = np.random.default_rng(31)
  vec = _directions(rng, 3000, 3)
  cases = []
  for n in (3000, 9000, 500, 6000):
    pts = rng.uniform(0.0, 2.0, size=(n, 3))
    cases.append((pts, po.cum_hypervolume_origin(pts, vec), po.is_frontier(pts)))
  start = threading.Barrier(len(cases))
  errors = []

  def work(pts, want_hv, want_front):
    try:
      start.wait()
      for _ in range(5):
        np.testing.assert_allclose(mm.cum_hypervolume_origin(pts, vec), want_hv, rtol=1e-12, atol=0)
        np.testing.assert_array_equal(mm.is_frontier(pts), want_front)
        t = torch.from_numpy(pts).cuda()
        np.testing.assert_allclose(mm.cum_hypervolume_origin(t, torch.from_numpy(vec).cuda()).cpu().numpy(), want_hv,
                                   rtol=1e-12, atol=0)
    except Exception as e:  # pylint: disable=broad-except
      errors.append(f'N={len(pts)}: {e}')

  threads = [threading.Thread(target=work, args=c) for c in cases]
  for t in threads:
    t.start()
  for t in threads:
    t.join()
  assert not errors, errors


def test_cum_hypervolume_non_finite():
  mm = _mm()
  rng = np.random.default_rng(11)
  pts = rng.uniform(0.0, 2.0, size=(700, 3))
  vec = _directions(rng, 500, 3)
  vec[7, 1] = 0.0              # p / 0 = inf: that coordinate never sets the min
  pts[3, 0] = np.inf
  pts[400, 2] = np.nan         # NaN from row 400 on, as NumPy's min and maximum.accumulate propagate it
  want = po.cum_hypervolume_origin(pts, vec)
  got = mm.cum_hypervolume_origin(pts, vec)
  assert np.all(np.isnan(got[400:])) and np.all(np.isfinite(got[:3]))
  np.testing.assert_allclose(got, want, rtol=1e-12, atol=0, equal_nan=True)
  assert np.all(np.isnan(mm.cum_hypervolume_origin(pts[:5], vec[:0])))


def test_pareto_frontier_on_device():
  mm = _mm()
  g = G['two_point_hypervolume']
  np.random.seed(0)
  for c in g['cases']:
    pf = mm.ParetoFrontier(np.array([[c['x'], c['y']], [c['y'], c['x']]]), np.array(g['origin'], float))
    assert abs(float(pf.hypervolume()) - c['expected']) <= g['delta'], c
  np.random.seed(1)
  points = np.random.normal(size=(100, 4))
  np.random.seed(2)
  pf = mm.ParetoFrontier(points, np.zeros(4))
  cum = pf.hypervolume(is_cumulative=True)
  assert len(cum) == len(points) and np.all(np.diff(cum) >= 0)
  assert cum[-1] == pytest.approx(float(pf.hypervolume()), rel=1e-12)
  np.random.seed(2)
  ref = mm.ParetoFrontier(points, np.zeros(4), cum_hypervolume_base=po.cum_hypervolume_origin)
  np.testing.assert_allclose(cum, ref.hypervolume(is_cumulative=True), rtol=1e-12)
  d = G['dimension_mismatch']
  with pytest.raises(ValueError, match=d['message']):
    mm.ParetoFrontier(np.array(d['points'], float), np.array(d['origin_3d'], float))
  pf = mm.ParetoFrontier(np.array(d['points'], float), np.array(d['origin'], float))
  with pytest.raises(ValueError, match=d['message']):
    pf.hypervolume(additional_points=np.array(d['origin_3d'], float)[..., np.newaxis])


class _FastParetoOptimal:
  """The divide-and-conquer frontier of Kung, Luccio and Preparata (the reference's FastParetoOptimalAlgorithm), with
  a pluggable base algorithm below `recursive_threshold` rows."""

  def __init__(self, base, recursive_threshold=10000):
    self._base = base
    self._threshold = recursive_threshold

  def is_pareto_optimal_against(self, points, against, *, strict):
    if len(points) == 0:
      return np.zeros(0, dtype=bool)
    if len(against) == 0:
      return np.ones(len(points), dtype=bool)
    if len(against) < self._threshold or len(points) < self._threshold:
      return np.array(self._base.is_pareto_optimal_against(points, against, strict=strict), dtype=bool)
    if against.shape[1] <= 1:
      top = np.max(against)
      return (points >= top).squeeze() if strict else (points > top).squeeze()
    order = points[:, 0].argsort()
    srt = points[order]
    split = round(len(points) / 2)
    value = srt[split][0]
    while srt[split][0] == value:
      split += 1
      if split == len(srt):
        return np.array(self._base.is_pareto_optimal_against(points, against, strict=strict), dtype=bool)
    dom = against[against[:, 0].argsort()]
    dsplit = np.searchsorted(dom[:, 0], value, side='right')
    upper = self.is_pareto_optimal_against(srt[split:], dom[dsplit:], strict=strict)
    lower = self.is_pareto_optimal_against(srt[:split], dom[:dsplit], strict=strict)
    cross = self.is_pareto_optimal_against(srt[:split, 1:], dom[dsplit:, 1:], strict=False)
    out = np.zeros(len(points), dtype=bool)
    out[order[:split]] = lower & cross
    out[order[split:]] = upper
    return out

  def is_pareto_optimal(self, points):
    if len(points) <= self._threshold:
      return np.array(self._base.is_pareto_optimal(points), dtype=bool)
    order = points[:, 0].argsort()
    srt = points[order]
    split = round(len(points) / 2)
    lower, upper = srt[:split], srt[split:]
    hi = self.is_pareto_optimal(upper)
    lo = self.is_pareto_optimal(lower) & self.is_pareto_optimal_against(lower, upper, strict=True)
    out = np.zeros(len(points), dtype=bool)
    out[order[:split]] = lo
    out[order[split:]] = hi
    return out


@pytest.mark.parametrize('threshold', [10000, 300])
def test_device_algorithm_as_base_of_divide_and_conquer(threshold):
  mm = _mm()
  base = mm.DeviceParetoOptimalAlgorithm()
  fast = _FastParetoOptimal(base, recursive_threshold=threshold)
  rng = np.random.default_rng(threshold)
  for m in (2, 3, 5):
    pts = rng.normal(size=(2000, m))
    pts = np.vstack([pts, pts[:500]])   # equal rows
    np.testing.assert_array_equal(fast.is_pareto_optimal(pts), po.is_frontier(pts))
    np.testing.assert_array_equal(base.is_pareto_optimal(pts), po.is_frontier(pts))
    against = rng.normal(size=(3000, m))
    for strict in (True, False):
      np.testing.assert_array_equal(fast.is_pareto_optimal_against(pts, against, strict=strict),
                                    po.is_pareto_optimal_against(pts, against, strict))
  sphere = _directions(rng, 1000, 3)
  assert np.all(fast.is_pareto_optimal(sphere))
