"""Candidates exactly on the trust-region radius, on every scoring route whose own tests have no such case: the uniform
ensemble, the transfer-learning stack, the general (`linear_coef`) route, GP-UCB-PE on the small route, multi-metric
GP-UCB-PE in both modes, set-PE and q-acquisition sets.

Coordinates are multiples of 1/64 and the radius is 4/64, so every L-inf distance is exact and a sixth of the pool
lies exactly on the radius of a trusted trial.  Each route scores the pool twice, with the trust region and without
it, and the difference must be the route's rule restated on the host:
  pointwise, non-strict (acquisitions.py:160-166)  outside iff dist > radius:   score = -1e4 - dist
  pointwise, strict (gp_ucb_pe.py:221-242)         outside iff dist >= radius:  score = -1e4 - dist
  set (gp_ucb_pe.py:245-269)                       score += sum over the set's points with dist > radius of -1e4 - dist
"""
import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from oracle import gp_oracle as go  # noqa: E402

R = 4 / 64
D = 4
MASK = np.array([True, True, False, True])
SMALL, GENERAL = 0, 4   # vzgp_score_route


def _gp():
  from vizier_b200 import gp
  return gp


def _params(linear=False, sf2=1.0):
  gp = _gp()
  ls2 = 0.5 * (1 + np.arange(D) / D)
  if linear:
    return gp.GPHyperParams(sf2, ls2, 1e-3, None, 1.0, 0.9, 0.3, -0.4)
  return gp.GPHyperParams(sf2, ls2, 1e-3)


def _trials(rng, n, n_metrics=1):
  x = np.round(rng.uniform(size=(n, D)) * 64) / 64
  y = np.stack([-np.sum((x - 0.3 + 0.1 * k) ** 2, axis=1) + 0.05 * rng.normal(size=n) for k in range(n_metrics)], 1)
  return x, (y[:, 0] if n_metrics == 1 else y)


def _pool(rng, x, rows, m):
  """m dyadic candidates: a third next to trials, a sixth exactly on the radius of one of the first `rows` trials in
  one trust-region dimension (within it in the others), the rest anywhere."""
  xs = np.round(rng.uniform(-0.25, 1.25, size=(m, D)) * 64) / 64
  perm = rng.permutation(m)
  near, edge = perm[:m // 3], perm[m // 3:m // 2]
  xs[near] = x[rng.integers(0, len(x), near.size)] + rng.integers(-6, 7, size=(near.size, D)) / 64
  step = rng.integers(-3, 4, size=(edge.size, D)) / 64
  on = np.flatnonzero(MASK)
  step[np.arange(edge.size), rng.choice(on, edge.size)] = rng.choice([-1.0, 1.0], edge.size) * R
  xs[edge] = x[rng.integers(0, rows, edge.size)] + step
  return xs


def _dist(xs, x, rows):
  dist = go.min_linf_distance(xs, x[:rows], MASK)
  assert int(np.sum(dist == R)) >= 10                       # the boundary itself is exercised
  return dist


def _np(t):
  return t.cpu().numpy().copy()


def _check_pointwise(on, off, dist, strict):
  inside = (dist < R) if strict else (dist <= R)
  assert inside.any() and (~inside).any()
  np.testing.assert_array_equal(on[~inside], -1e4 - dist[~inside])
  np.testing.assert_allclose(on[inside], off[inside], atol=1e-10, rtol=0)


def _check_set(on, off, dist, q):
  term = np.where(dist > R, -1e4 - dist, 0.0).reshape(-1, q).sum(axis=1)
  assert (term < 0).any() and (term == 0).any()
  np.testing.assert_allclose(on, off + term, atol=1e-9, rtol=0)


@pytest.mark.parametrize('strict', [False, True], ids=['nonstrict', 'strict'])
def test_ensemble(strict):
  gp = _gp()
  rng = np.random.default_rng(11)
  n, rows = 150, 140
  x, y = _trials(rng, n)
  xs = _pool(rng, x, rows, 700)
  ens = gp.EnsembleGP(0, 2)
  try:
    ens.fit(x, y, [_params(sf2=1.0), _params(sf2=1.7)])
    out = {}
    for use in (True, False):
      acq = gp.Acquisition(1.8, use, R, MASK, tr_rows=rows, tr_strict=strict)
      res = ens.score(xs, acq, with_aux=True)
      ens.synchronize()
      out[use] = _np(res['score'])
    np.testing.assert_array_equal(_np(res['linf_distance']), _dist(xs, x, rows))
    _check_pointwise(out[True], out[False], _dist(xs, x, rows), strict)
  finally:
    for mem in ens.members:
      mem.close()


@pytest.mark.parametrize('strict', [False, True], ids=['nonstrict', 'strict'])
def test_stack(strict):
  gp = _gp()
  rng = np.random.default_rng(12)
  x0, y0 = _trials(rng, 90)
  x, y = _trials(rng, 120)
  rows = 110
  xs = _pool(rng, x, rows, 700)
  stack = gp.StackedGP(0)
  try:
    for xl, yl in ((x0, y0), (x, y)):
      level = stack.new_level()
      level.fit(xl, yl - stack.mean(xl), _params())
      stack.push(level, len(xl))
    out = {}
    for use in (True, False):
      res = stack.score(xs, gp.Acquisition(1.8, use, R, MASK, tr_rows=rows, tr_strict=strict), with_aux=True)
      stack.synchronize()
      out[use] = _np(res['score'])
    dist = _dist(xs, x, rows)                               # the top level's trials
    np.testing.assert_array_equal(_np(res['linf_distance']), dist)
    _check_pointwise(out[True], out[False], dist, strict)
  finally:
    stack.close()


@pytest.mark.parametrize('strict', [False, True], ids=['nonstrict', 'strict'])
def test_general_route(strict):
  gp = _gp()
  rng = np.random.default_rng(13)
  n, rows = 130, 120
  x, y = _trials(rng, n)
  xs = _pool(rng, x, rows, 600)
  dev = gp.DeviceGP(0)
  try:
    dev.fit(x, y, _params(linear=True))
    out = {}
    for use in (True, False):
      res = dev.score(xs, gp.Acquisition(1.8, use, R, MASK, tr_rows=rows, tr_strict=strict), with_aux=True)
      dev.synchronize()
      assert dev.get_int('score_route') == GENERAL
      out[use] = _np(res['score'])
    dist = _dist(xs, x, rows)
    np.testing.assert_array_equal(_np(res['linf_distance']), dist)
    _check_pointwise(out[True], out[False], dist, strict)
  finally:
    dev.close()


def _pe_models(rng, n, n_pending, n_metrics=1):
  gp = _gp()
  x, y = _trials(rng, n, n_metrics)
  xb = np.concatenate([x, np.round(rng.uniform(size=(n_pending, D)) * 64) / 64])
  dev_a = gp.DeviceGP(0)
  dev_b = gp.DeviceGP(0, stream=dev_a.stream)
  assert dev_a.fit(x, y, _params()) == 0
  assert dev_b.fit(xb, np.zeros(n + n_pending), _params()) == 0
  return x, y, xb, dev_a, dev_b


@pytest.mark.parametrize('mode', [0, 1])
def test_ucb_pe_small_route(mode):
  gp = _gp()
  rng = np.random.default_rng(14 + mode)
  n, n_pending = 100, 12
  rows = n + n_pending - 4
  x, y, xb, dev_a, dev_b = _pe_models(rng, n, n_pending)
  xs = _pool(rng, xb, rows, 300)
  try:
    out = {}
    for use in (True, False):
      pe = gp.UcbPeAcquisition(mode=mode, threshold=float(np.median(y)), use_trust_region=use, trust_radius=R,
                               tr_dim_mask=MASK, tr_rows=rows)
      out[use] = _np(dev_a.score_pe(dev_b, xs, pe)['score'])
      assert dev_a.get_int('score_route') == SMALL and dev_b.get_int('score_route') == SMALL
    _check_pointwise(out[True], out[False], _dist(xs, xb, rows), strict=True)
  finally:
    dev_b.close(); dev_a.close()


@pytest.mark.parametrize('mode', [0, 1])
def test_ucb_pe_multi(mode):
  gp = _gp()
  rng = np.random.default_rng(16 + mode)
  n, n_pending, nm = 100, 12, 2
  rows = n + n_pending - 4
  x, y, xb, dev_a, dev_b = _pe_models(rng, n, n_pending, nm)
  xs = _pool(rng, xb, rows, 300)
  w = np.abs(rng.normal(size=(64, nm)))
  w /= np.linalg.norm(w, axis=1, keepdims=True)
  ref = go.hv_reference_point(y)
  sc = gp.ScalarizedUcbAcquisition(w, ref, go.hv_max_scalarized(y, w, ref), 1.8) if mode == 0 else None
  try:
    out = {}
    for use in (True, False):
      pe = gp.UcbPeMultiAcquisition(n_metrics=nm, mode=mode, thresholds=np.median(y, axis=0), scalarization=sc,
                                    use_trust_region=use, trust_radius=R, tr_dim_mask=MASK, tr_rows=rows)
      out[use] = _np(dev_a.score_pe_multi(dev_b, xs, pe)['score'])
    _check_pointwise(out[True], out[False], _dist(xs, xb, rows), strict=True)
  finally:
    dev_b.close(); dev_a.close()


def test_set_pe():
  gp = _gp()
  rng = np.random.default_rng(18)
  n, n_pending, q = 100, 12, 3
  rows = n + n_pending - 4
  x, y, xb, dev_a, dev_b = _pe_models(rng, n, n_pending)
  xs = _pool(rng, xb, rows, 120 * q)
  try:
    out = {}
    for use in (True, False):
      pe = gp.UcbPeAcquisition(mode=1, threshold=float(np.median(y)), use_trust_region=use, trust_radius=R,
                               tr_dim_mask=MASK, tr_rows=rows)
      res = dev_a.score_set_pe(dev_b, xs, q, pe)
      dev_a.synchronize()
      out[use] = _np(res['score'])
    _check_set(out[True], out[False], _dist(xs, xb, rows), q)
  finally:
    dev_b.close(); dev_a.close()


def test_qsets():
  gp = _gp()
  from vizier_b200 import _lib
  rng = np.random.default_rng(19)
  n, rows, q = 120, 110, 3
  x, y = _trials(rng, n)
  xs = _pool(rng, x, rows, 150 * q)
  dev = gp.DeviceGP(0)
  try:
    dev.fit(x, y, _params())
    out = {}
    for use in (True, False):
      qa = gp.QAcquisition(_lib.QACQ_QUCB, num_samples=64, use_trust_region=use, trust_radius=R, tr_dim_mask=MASK,
                           tr_rows=rows)
      res = dev.score_qsets(xs, q, qa, seed=5, with_aux=True)
      dev.synchronize()
      out[use] = _np(res['score'])
    dist = _dist(xs, x, rows)
    np.testing.assert_array_equal(_np(res['linf_distance']), dist)
    _check_set(out[True], out[False], dist, q)
  finally:
    dev.close()
