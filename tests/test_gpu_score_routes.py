"""Every candidate-scoring route against the oracle, at the tile, block, cluster and masking edges.

`launch_score` (csrc/score.cu) sends a pool down one of several routes, chosen from the tile count
ntiles = ceil(M / 64), the column blocks nblocks = ceil(np / 128) of the padded trial count np and the SM count:

  small    ntiles <= small_tiles (8)                  k_cross_small, k_var_small, k_small_finalize
  split    2 * ntiles <= SMs and nblocks >= 3         k_score, nsplit = ceil(nblocks / 2) CTAs per tile, k_score_finalize
  cluster  every other pool                           k_score in 2-CTA clusters (TMA multicast of Linv)
  i8       "score_i8" on, ntiles >= SMs, np >= 128    k_score_i8

The sizes below are planned from the SM count and the measured number of co-resident clusters, never hard-coded,
and every case first asserts the route, nsplit and grid the handle recorded (vzgp_get_int "score_route",
"score_nsplit", "score_grid").  Every candidate is then compared with oracle/gp_oracle.py: score, mean and
stddev within 1e-10, the L-inf trust-region distance bit for bit.  The ill-conditioned case is measured against
the long-double posterior of oracle/hp_oracle.py instead.
"""
import dataclasses
import os
from typing import Callable, Optional

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from oracle import gp_oracle as go  # noqa: E402
from oracle import hp_oracle as hp  # noqa: E402

TOL = 1e-10
SMALL, SPLIT, CLUSTER, I8 = 0, 1, 2, 3     # vzgp_score_route (include/vzgp.h)
ROUTES = {'small': SMALL, 'split': SPLIT, 'cluster': CLUSTER, 'i8': I8}
DEFAULT_SMALL_TILES = int(os.environ.get('VZGP_SMALL_TILES', '8'))


def _gp():
  from vizier_b200 import gp
  return gp


@dataclasses.dataclass
class Geometry:
  sm: int      # multiprocessors
  slots: int   # co-resident 2-CTA clusters of k_score


@pytest.fixture(scope='module')
def dev():
  d = _gp().DeviceGP(0)
  yield d
  d.close()


@pytest.fixture(scope='module')
def geom(dev):
  """SM count from the handle; cluster slots from the grid of a cluster-route launch too large to fit at once."""
  gp = _gp()
  sm = dev.get_int('sm_count')
  rng = np.random.default_rng(0)
  x = rng.uniform(size=(64, 2))
  dev.fit(x, np.sin(x.sum(1)), gp.GPHyperParams(1.0, np.full(2, 0.5), 1e-3))
  dev.set_int('score_i8', 0)
  dev.set_int('small_tiles', -1)
  tiles = 4 * sm
  dev.score(dev.random_pool(tiles * 64, 2, seed=1), gp.Acquisition(1.8, False, 1.0))
  dev.synchronize()
  assert dev.get_int('score_route') == CLUSTER and dev.get_int('score_nsplit') == 1
  grid = dev.get_int('score_grid')
  assert grid % 2 == 0 and 0 < grid <= sm
  return Geometry(sm, grid // 2)


def _plan(g: Geometry, tiles: int, n: int, dc: int, small_tiles: int = -1, i8: bool = False):
  """(route, nsplit, grid) launch_score must take; the same rules, restated."""
  np_ = -(-n // 64) * 64
  nblocks = -(-np_ // 128)
  if tiles <= (DEFAULT_SMALL_TILES if small_tiles < 0 else small_tiles):
    return SMALL, 0, 0
  if i8 and tiles >= g.sm and 128 <= np_ <= 4096 and dc >= 1:
    return I8, 1, min(tiles, g.sm)
  nsplit = (nblocks + 1) // 2 if (2 * tiles <= g.sm and nblocks >= 2) else 1
  if nsplit > 1:
    return SPLIT, nsplit, min(tiles * nsplit, g.sm)
  return CLUSTER, 1, min(-(-tiles // 2), g.slots) * 2


def _recorded(d):
  return d.get_int('score_route'), d.get_int('score_nsplit'), d.get_int('score_grid')


@dataclasses.dataclass
class Case:
  route: str                        # the route the sizes are meant to select
  n: int
  d: int
  tiles: Callable[[Geometry], int]
  last: int = 64                    # candidates in the last tile
  dk: int = 0
  sf2: float = 1.0
  small_tiles: int = -1             # per-handle override (-1: the default)
  radius: Optional[float] = 0.3     # None: no trust region; > 0.5: trust region switched off by its radius
  mask_off: tuple = ()              # continuous dims left out of the trust-region distance
  nv: Optional[int] = None          # valid trials (n_valid)
  tr_rows: Optional[int] = None     # trusted rows
  strict: bool = False              # inside test dist < radius instead of <=
  dyadic: bool = False              # coordinates k / 64 and candidates exactly on the radius (implied by strict)
  seed: int = 0


def _t(k):
  return lambda g: k


HALF = lambda g: g.sm // 2            # noqa: E731  largest pool of the split route
HALF1 = lambda g: g.sm // 2 + 1       # noqa: E731  smallest pool past it
ROUND_M1 = lambda g: 2 * g.slots - 1  # noqa: E731  one cluster round, last CTA scores the padding tile
ROUND = lambda g: 2 * g.slots         # noqa: E731
ROUND_P1 = lambda g: 2 * g.slots + 1  # noqa: E731  a second round: one real tile + one padding tile
I8T = lambda g: g.sm + 1             # noqa: E731  cluster route with score_i8 off, k_score_i8 with it on
LK3 = np.array([0.3, 1.1, 4.0])

CASES = [
    # np / nblocks
    pytest.param(Case('cluster', 1, 3, _t(9)), id='N1'),
    pytest.param(Case('cluster', 37, 5, _t(9), last=17, radius=None), id='N37-np64'),
    pytest.param(Case('cluster', 128, 20, _t(12), last=1, radius=0.7, sf2=0.31), id='N128-D20'),
    pytest.param(Case('cluster', 129, 1, _t(9), radius=0.25), id='N129-D1'),
    pytest.param(Case('split', 300, 8, _t(9), last=63, dk=3, mask_off=(2, 5)), id='N300-split-dk3'),
    pytest.param(Case('split', 500, 6, _t(10), sf2=2.7), id='N500-split-even'),
    pytest.param(Case('split', 520, 7, _t(9), radius=None), id='N520-split-nsplit3'),
    pytest.param(Case('split', 1030, 12, _t(9), last=5, mask_off=(0,)), id='N1030-split-nsplit5'),
    pytest.param(Case('cluster', 500, 6, HALF1, radius=0.7), id='N500-cluster'),
    pytest.param(Case('cluster', 1030, 4, HALF1, last=33), id='N1030-cluster'),
    # tile counts
    pytest.param(Case('cluster', 100, 4, _t(1), last=37, small_tiles=0), id='T1-cluster-padding-peer'),
    pytest.param(Case('split', 300, 4, _t(1), small_tiles=0, dk=3), id='T1-split'),
    pytest.param(Case('cluster', 200, 5, _t(8), last=1, small_tiles=0, sf2=2.7), id='T8-cluster'),
    pytest.param(Case('split', 520, 5, _t(8), small_tiles=0, radius=None), id='T8-split'),
    pytest.param(Case('cluster', 200, 5, _t(9), mask_off=(1,)), id='T9-padding-cta'),
    pytest.param(Case('split', 300, 8, HALF, last=1), id='Thalf-split'),
    pytest.param(Case('cluster', 300, 8, HALF1, last=63, dk=3), id='Thalf1-cluster-dk3'),
    pytest.param(Case('cluster', 150, 6, ROUND_M1, radius=None), id='T2slots-1'),
    pytest.param(Case('cluster', 150, 6, ROUND, sf2=0.31, mask_off=(3,)), id='T2slots'),
    pytest.param(Case('cluster', 150, 6, ROUND_P1, last=1, dk=3), id='T2slots+1-dk3'),
    # features
    pytest.param(Case('split', 300, 64, _t(9), last=40), id='D64-split'),
    pytest.param(Case('cluster', 200, 64, HALF1, radius=None), id='D64-cluster'),
    pytest.param(Case('small', 200, 64, _t(3)), id='D64-small'),
    # n_valid < n: candidates sit next to the masked rows
    pytest.param(Case('small', 300, 5, _t(4), nv=263, dk=3), id='nvalid-small'),
    pytest.param(Case('split', 300, 5, _t(9), nv=263), id='nvalid-split'),
    pytest.param(Case('cluster', 300, 5, HALF1, nv=263, dk=3), id='nvalid-cluster'),
    pytest.param(Case('cluster', 300, 5, I8T, nv=263, radius=None), id='nvalid-cluster-i8'),
    # tr_rows < n_valid: candidates sit next to the untrusted rows
    pytest.param(Case('small', 300, 5, _t(5), nv=280, tr_rows=200), id='trrows-small'),
    pytest.param(Case('split', 300, 5, _t(9), nv=280, tr_rows=200, dk=3), id='trrows-split'),
    pytest.param(Case('cluster', 300, 5, HALF1, nv=280, tr_rows=200, mask_off=(4,)), id='trrows-cluster'),
    pytest.param(Case('cluster', 300, 5, I8T, last=20, nv=280, tr_rows=200, dk=3), id='trrows-cluster-i8'),
    # strict trust region with candidates exactly on the radius
    pytest.param(Case('small', 300, 4, _t(6), radius=0.0625, strict=True), id='strict-small'),
    pytest.param(Case('split', 300, 4, _t(9), radius=0.0625, strict=True, tr_rows=250, mask_off=(1,)), id='strict-split'),
    pytest.param(Case('cluster', 300, 4, HALF1, radius=0.0625, strict=True, dk=3), id='strict-cluster'),
    pytest.param(Case('cluster', 300, 4, I8T, radius=0.0625, strict=True, nv=290, tr_rows=260), id='strict-cluster-i8'),
    pytest.param(Case('cluster', 300, 4, HALF1, radius=0.0625, dyadic=True), id='ties-nonstrict-cluster'),
]


def _problem(c: Case, m: int):
  """Trials, labels and a pool of m candidates.  A third of the pool sits next to particular trials: masked rows
  (n_valid), untrusted rows (tr_rows) or any row.  On dyadic coordinates (multiples of 1/64, so |a - b| is exact)
  another sixth lies exactly on the radius of a trusted trial in one trust-region dimension."""
  rng = np.random.default_rng(1000 + c.seed + c.n + 7 * c.d)
  n, d = c.n, c.d
  nv = c.nv or n
  dyadic = c.strict or c.dyadic
  x = rng.uniform(size=(n, d))
  if dyadic:
    x = np.round(x * 64) / 64
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  z = rng.integers(0, 4, size=(n, c.dk)).astype(np.int32) if c.dk else None
  xs = rng.uniform(-0.5, 1.5, size=(m, d))      # reaching outside the trials' box: both sides of any radius
  if dyadic:
    xs = np.round(xs * 64) / 64
  zs = rng.integers(0, 4, size=(m, c.dk)).astype(np.int32) if c.dk else None
  perm = rng.permutation(m)
  near, edge = perm[:max(1, m // 3)], perm[max(1, m // 3):max(1, m // 2)]
  if c.tr_rows:
    lo, hi = c.tr_rows, nv
  elif c.nv:
    lo, hi = nv, n
  else:
    lo, hi = 0, n
  src = rng.integers(lo, hi, near.size)
  if dyadic:
    xs[near] = x[src] + rng.integers(-3, 4, size=(near.size, d)) / 64
    # on the radius of a trusted trial in one trust-region dimension, within it in the others
    on = [k for k in range(d) if k not in c.mask_off]
    src_e = rng.integers(0, c.tr_rows or nv, edge.size)
    step = rng.integers(-3, 4, size=(edge.size, d)) / 64
    step[np.arange(edge.size), rng.choice(on, edge.size)] = rng.choice([-1.0, 1.0], edge.size) * c.radius
    xs[edge] = x[src_e] + step
    if zs is not None:
      zs[edge] = z[src_e]
  else:
    xs[near] = x[src] + rng.uniform(-0.04, 0.04, size=(near.size, d))
  if zs is not None:
    zs[near] = z[src]
  k = min(3, m)
  xs[:k] = x[lo:lo + k]            # exact copies: distance 0, sigma ~ sqrt(2 sn2)
  if zs is not None:
    zs[:k] = z[lo:lo + k]
  return x, y, z, xs, zs


def _oracle(c: Case, x, y, z, xs, zs):
  nv = c.nv or c.n
  lk = LK3[:c.dk] if c.dk else None
  ls2 = 0.5 * (1 + np.arange(c.d) / c.d)
  po = go.GPParams(c.sf2, ls2, 1e-3, lk)
  pg = _gp().GPHyperParams(c.sf2, ls2, 1e-3, lk)
  pred = go.precompute_predictive(po, x, y, z, row_valid=np.arange(c.n) < nv)
  mu, sd = go.predict(pred, xs, zs)
  mask = np.array([k not in c.mask_off for k in range(c.d)])
  dist = go.min_linf_distance(xs, x[:(c.tr_rows or nv)], mask)
  score = go.ucb(mu, sd, 1.8)
  if c.radius is not None:
    inside = ((dist < c.radius) if c.strict else (dist <= c.radius)) | (c.radius > 0.5)
    score = np.where(inside, score, -1e4 - dist)
  return pg, mask, {'score': score, 'mean': mu, 'stddev': sd, 'linf_distance': dist}


def _score(d, xs, zs, acq, aux=True):
  out = d.score(xs, acq, zs=zs, with_aux=aux)
  d.synchronize()
  keys = ('score', 'mean', 'stddev', 'linf_distance') if aux else ('score',)
  return {k: out[k].cpu().numpy().copy() for k in keys}, _recorded(d)


def _check_oracle(got, want):
  for k in ('score', 'mean', 'stddev'):
    if k in got:
      np.testing.assert_allclose(got[k], want[k], atol=TOL, rtol=0, err_msg=k)
  if 'linf_distance' in got:
    np.testing.assert_array_equal(got['linf_distance'], want['linf_distance'])


@pytest.mark.parametrize('c', CASES)
def test_score_route_matches_oracle(dev, geom, c):
  gp = _gp()
  tiles = c.tiles(geom)
  m = (tiles - 1) * 64 + c.last
  plan = _plan(geom, tiles, c.n, c.d, c.small_tiles)
  assert plan[0] == ROUTES[c.route], f'{tiles} tiles of N={c.n} take route {plan[0]} on this GPU'
  x, y, z, xs, zs = _problem(c, m)
  pg, mask, want = _oracle(c, x, y, z, xs, zs)
  if c.radius is not None and c.radius <= 0.5:
    assert (want['score'] < -1e3).any() and (want['score'] > -1e3).any()   # both sides of the region
  if c.strict or c.dyadic:
    ties = int(np.sum(want['linf_distance'] == c.radius))
    assert ties >= 10, ties                                                 # the boundary itself is exercised
  dev.set_int('score_i8', 0)
  dev.set_int('small_tiles', c.small_tiles)
  try:
    dev.fit(x, y, pg, z=z, n_valid=c.nv or c.n)
    xst = torch.from_numpy(xs).cuda()
    zst = torch.from_numpy(zs).cuda() if zs is not None else None
    acq = gp.Acquisition(1.8, c.radius is not None, 1.0 if c.radius is None else c.radius, mask,
                         tr_rows=c.tr_rows or 0, tr_strict=c.strict)
    got, rec = _score(dev, xst, zst, acq)
    assert rec == plan, (rec, plan)
    _check_oracle(got, want)
    # without the aux outputs: k_score<false> (pre-scaled features) unless a radius <= 0.5 needs the distance
    fast, rec = _score(dev, xst, zst, acq, aux=False)
    assert rec == plan
    np.testing.assert_allclose(fast['score'], got['score'], atol=1e-12, rtol=0)
    _check_oracle(fast, want)
    again, rec = _score(dev, xst, zst, acq)
    assert rec == plan
    for k in got:
      np.testing.assert_array_equal(again[k], got[k], err_msg=k)
    if c.small_tiles == 0 and tiles <= DEFAULT_SMALL_TILES:
      # the same pool down the small-pool kernels
      dev.set_int('small_tiles', -1)
      small, rec = _score(dev, xst, zst, acq)
      assert rec == (SMALL, 0, 0)
      for k in ('score', 'mean', 'stddev'):
        np.testing.assert_allclose(small[k], got[k], atol=1e-12, rtol=0, err_msg=k)
      np.testing.assert_array_equal(small['linf_distance'], got['linf_distance'])
    i8_plan = _plan(geom, tiles, c.n, c.d, c.small_tiles, i8=True)
    if i8_plan[0] == I8:
      dev.set_int('score_i8', 1)
      for aux in (True, False):
        res, rec = _score(dev, xst, zst, acq, aux=aux)
        assert rec == i8_plan, (rec, i8_plan)
        _check_oracle(res, want)
  finally:
    dev.set_int('score_i8', 0)
    dev.set_int('small_tiles', -1)


def test_i8_cases_present(geom):
  """The cases meant to reach k_score_i8 do reach it on this GPU (their tile counts are >= the SM count)."""
  ids = [p.id for p in CASES if p.id.endswith('-i8')]
  assert len(ids) >= 3
  for p in CASES:
    if p.id.endswith('-i8'):
      c = p.values[0]
      assert _plan(geom, c.tiles(geom), c.n, c.d, c.small_tiles, i8=True)[0] == I8, p.id


def test_pe_score_on_cluster_route(dev, geom):
  """GP-UCB-PE (vzgp_score_pe) on a pool large enough for the cluster route: strict trust region over the first
  tr_rows trials of model B, candidates exactly on the radius."""
  gp = _gp()
  n, n_pending, d, r, rows = 200, 40, 4, 0.0625, 215
  tiles = geom.sm // 2 + 1
  m = (tiles - 1) * 64 + 9
  assert _plan(geom, tiles, n + n_pending, d)[0] == CLUSTER
  c = Case('cluster', n + n_pending, d, _t(tiles), last=9, radius=r, strict=True, mask_off=(2,), tr_rows=rows, seed=5)
  xb, yb, _, xs, _ = _problem(c, m)
  x, y = xb[:n], yb[:n]
  yb = np.concatenate([y, np.zeros(n_pending)])
  ls2 = 0.5 * (1 + np.arange(d) / d)
  po = go.GPParams(1.3, ls2, 1e-3)
  pg = gp.GPHyperParams(1.3, ls2, 1e-3)
  pred_a, pred_b = go.precompute_predictive(po, x, y), go.precompute_predictive(po, xb, yb)
  mask = np.array([True, True, False, True])
  thr = go.ucb_threshold(pred_a, pred_b, 1.8)
  want, aux = go.ucb_pe_score(pred_a, pred_b, xs, mode=0, threshold=thr, tr_dim_mask=mask, tr_rows=rows,
                              trust_radius_value=r)
  dist = go.min_linf_distance(xs, xb[:rows], mask)
  assert int(np.sum(dist == r)) >= 10 and (want < -1e3).any() and (want > -1e3).any()
  dev_b = gp.DeviceGP(0, stream=dev.stream)
  try:
    dev.set_int('score_i8', 0)
    dev.fit(x, y, pg)
    dev_b.fit(xb, yb, pg)
    pe = gp.UcbPeAcquisition(mode=0, threshold=thr, trust_radius=r, tr_dim_mask=mask, tr_rows=rows)
    out = dev.score_pe(dev_b, xs, pe)
    plan = _plan(geom, tiles, n, d)
    assert _recorded(dev) == plan and _recorded(dev_b) == _plan(geom, tiles, n + n_pending, d)
    np.testing.assert_allclose(out['mean'].cpu().numpy(), aux['mean'], atol=TOL, rtol=0)
    np.testing.assert_allclose(out['stddev'].cpu().numpy(), aux['stddev'], atol=TOL, rtol=0)
    np.testing.assert_allclose(out['stddev_from_all'].cpu().numpy(), aux['stddev_from_all'], atol=TOL, rtol=0)
    np.testing.assert_allclose(out['score'].cpu().numpy(), want, atol=TOL, rtol=0)
  finally:
    dev_b.close()


def test_ensemble_on_split_route(geom):
  """A uniform ensemble (vzgp_score_ensemble) whose members take the split route, against the oracle mixture."""
  gp = _gp()
  n, d, tiles, r = 300, 6, 9, 0.3
  m = (tiles - 1) * 64 + 50
  assert _plan(geom, tiles, n, d)[0] == SPLIT
  c = Case('split', n, d, _t(tiles), last=50, seed=9)
  x, y, _, xs, _ = _problem(c, m)
  rng = np.random.default_rng(91)
  plist_o, plist_g = [], []
  for _ in range(2):
    ls2 = np.exp(rng.uniform(np.log(0.1), np.log(2.0), d))
    sf2, sn2 = float(np.exp(rng.uniform(-1, 1))), float(np.exp(rng.uniform(-8, -3)))
    plist_o.append(go.GPParams(sf2, ls2, sn2))
    plist_g.append(gp.GPHyperParams(sf2, ls2, sn2))
  preds = [go.precompute_predictive(p, x, y) for p in plist_o]
  mu, sd = go.predict_ensemble(preds, xs)
  dist = go.min_linf_distance(xs, x, np.ones(d, bool))
  want = go.apply_trust_region(go.ucb(mu, sd, 1.8), dist, r)
  assert (want < -1e3).any() and (want > -1e3).any()
  ens = gp.EnsembleGP(0, 2)
  try:
    ens.fit(x, y, plist_g)
    out = ens.score(xs, gp.Acquisition(1.8, True, r), with_aux=True)
    ens.synchronize()
    for mem in ens.members:
      assert _recorded(mem) == _plan(geom, tiles, n, d)
    np.testing.assert_allclose(out['mean'].cpu().numpy(), mu, atol=TOL, rtol=0)
    np.testing.assert_allclose(out['stddev'].cpu().numpy(), sd, atol=TOL, rtol=0)
    np.testing.assert_allclose(out['score'].cpu().numpy(), want, atol=TOL, rtol=0)
    np.testing.assert_array_equal(out['linf_distance'].cpu().numpy(), dist)
  finally:
    for mem in ens.members:
      mem.close()


# Device error against the long-double posterior over the pool (max and RMS).  Mean: at most HARD_FACTOR times
# the fp64 oracle's own error plus a floor; measured on an H100 80GB HBM3 (400 W), every route's mean is 0.28-0.54
# times the oracle's error (one step of iterative refinement of alpha).  Stddev: the oracle's triangular solve is
# accurate to 7e-15 here, the device's W = K* Linv^T to 2.6e-10 (small, split) - 1.3e-9 (cluster, i8), RMS
# 1.6e-11 - 3.9e-11; the bounds are 4x those measurements, so a kernel 100x worse still fails.  The gap comes from
# the fit, not the scoring kernels: the device's Cholesky factor is 1.3e-10 from the long-double one (LAPACK's:
# 1.3e-12), and LAPACK's explicit inverse of the device's factor gives the same 2.6e-10 stddev error on the host.
HARD_FACTOR = 4.0
HARD_FLOOR = 1e-12
HARD_SD_MAX = 5e-9
HARD_SD_RMS = 2e-10


@pytest.mark.skipif(not hp.has_extended_precision(), reason='np.longdouble is fp64 on this platform')
def test_ill_conditioned_scoring_vs_long_double(dev, geom):
  """sn2 = 1e-8, ls2 = 0.05 and duplicated trials (cond(K_y) ~ 1e10) on the small, split, cluster and i8 routes:
  the device's mean is as accurate as fp64 LAPACK against a long-double reference, its stddev within the measured
  bounds above."""
  gp = _gp()
  n, d = 300, 6
  rng = np.random.default_rng(77)
  x = rng.uniform(size=(n, d))
  x[1::10] = x[0::10]                      # 30 duplicated trials
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  ls2 = np.full(d, 0.05)
  po = go.GPParams(1.0, ls2, 1e-8)
  pg = gp.GPHyperParams(1.0, ls2, 1e-8)
  tiles = {'small': 4, 'split': 9, 'cluster': geom.sm // 2 + 1, 'i8': geom.sm + 3}
  m = tiles['i8'] * 64
  xs = rng.uniform(size=(m, d))
  near = rng.permutation(m)[:m // 4]
  xs[near] = x[rng.integers(0, n, near.size)] + rng.uniform(-0.02, 0.02, size=(near.size, d))
  mu_h, sd_h = hp.predict(hp.precompute_predictive(po, x, y), xs)
  pred_f = go.precompute_predictive(po, x, y)
  assert pred_f.n_retries == 0
  mu_f, sd_f = go.predict(pred_f, xs)

  def errs(mu, sd, k):
    e = [np.abs((np.asarray(v[:k], np.longdouble) - ref[:k]).astype(np.float64)) for v, ref in ((mu, mu_h), (sd, sd_h))]
    return [(float(a.max()), float(np.sqrt(np.mean(a * a)))) for a in e]

  assert dev.fit(x, y, pg) == 0             # no jitter: the device factors the same K_y as the references
  acq = gp.Acquisition(1.8, False, 1.0)
  rows = []
  try:
    for route, t in tiles.items():
      k = t * 64
      dev.set_int('score_i8', 1 if route == 'i8' else 0)
      out = dev.score(torch.from_numpy(xs[:k]).cuda(), acq, with_aux=True)
      dev.synchronize()
      assert _recorded(dev)[0] == ROUTES[route]
      got = errs(out['mean'].cpu().numpy(), out['stddev'].cpu().numpy(), k)
      ref = errs(mu_f, sd_f, k)
      rows += [(route, name) + g + f for name, g, f in zip(('mean', 'stddev'), got, ref)]
  finally:
    dev.set_int('score_i8', 0)
  report = [f'{r:8s} {q:6s} device max {gm:.3e} rms {gr:.3e} | fp64 oracle max {fm:.3e} rms {fr:.3e} | '
            f'ratio max {gm / fm:.3g} rms {gr / fr:.3g}' for r, q, gm, gr, fm, fr in rows]
  print('\n' + '\n'.join(report))
  for line, (_, q, gm, gr, fm, fr) in zip(report, rows):
    if q == 'mean':
      assert gm <= HARD_FACTOR * fm + HARD_FLOOR, line
      assert gr <= HARD_FACTOR * fr + HARD_FLOOR, line
    else:
      assert gm <= HARD_SD_MAX and gr <= HARD_SD_RMS, line
