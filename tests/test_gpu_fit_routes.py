"""Every fit and NLL + gradient route against the oracle, with the Cholesky jitter retry forced on each of them.

vzgp_nll_grad_multi (csrc/c_abi.cu) takes one of these routes; vzgp_get_int "nll_route" records which:

  0 small   N <= 64, one metric, no linear_coef   k_nll_grad_small, retry loop inside the kernel
  1 graph   otherwise, no pivot flagged           replayed CUDA graph: panel kernels (N <= 64) or k_chol_dataflow
  2 eager   a pivot flagged in the graph,         fit_common's host retry loop, k_lauum planes
            linear_coef, VZGP_NLL_GRAPH=0
  3 batch   vzgp_nll_grad_batch (ARD restarts)    one graph for all restarts; a flagged restart falls back to 2

and "factor_route" the factorisation of the last fit / evaluation: 0 panel kernels, 1 k_chol_dataflow.  Every case
asserts both before it compares numbers.

The jitter fixtures (tests/fit_fixtures.py) repeat every trial three times: at sn2 = 1e-30 the first factorisation
fails and the first jitter (1e-4) succeeds with a wide margin; a negative sn2 (fit only) walks further up the
ladder.  Tolerances: the NLL 1e-9 relative on the loss without the regulariser, the gradient 1e-8 of max |g|; the
fit's Cholesky 1e-11, alpha 1e-8 of max |alpha|, scores 1e-10.
"""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

import fit_fixtures as ff  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402

SMALL, GRAPH, EAGER, BATCH = 0, 1, 2, 3     # vzgp_nll_route (include/vzgp.h)
PANEL, DATAFLOW = 0, 1                      # vzgp_factor_route
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))
LIN_COEF = 0.7


def _gp():
  from vizier_b200 import gp
  return gp


@pytest.fixture(scope='module')
def dev():
  d = _gp().DeviceGP(0)
  yield d
  d.close()


def _hyper(po, linear=False):
  gp = _gp()
  if linear:
    lp = po.linear
    return gp.GPHyperParams(po.signal_variance, po.continuous_length_scale_squared, po.observation_noise_variance,
                            po.categorical_length_scale_squared, linear_coef=lp.coef,
                            linear_slope_amplitude=lp.slope_amplitude, linear_shift=lp.shift,
                            mean_constant=lp.mean_constant)
  return gp.GPHyperParams(po.signal_variance, po.continuous_length_scale_squared, po.observation_noise_variance,
                          po.categorical_length_scale_squared)


def _with(po, sn2=None, linear=False):
  import dataclasses
  po = dataclasses.replace(po, observation_noise_variance=po.observation_noise_variance if sn2 is None else sn2)
  if linear:
    po = dataclasses.replace(po, linear=go.LinearParams(LIN_COEF, 0.9, 0.2, -0.3))
  return po


def _cuda(a, dtype=torch.float64):
  return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to('cuda', dtype)


def _routes(d):
  return d.get_int('nll_route'), d.get_int('factor_route')


def _oracle_nll(po, x, y, z, nv):
  lin = po.linear.coef if po.linear is not None else None
  return go.loss_and_grad(po.to_vector(), x, y, z, np.arange(x.shape[0]) < nv, linear_coef=lin)


def _assert_nll(loss, grad, want_l, want_g, po, skip_noise):
  """Loss without the regulariser within 1e-9 relative; gradient within 1e-8 of max |g| (the noise component
  excluded where its regulariser derivative swallows the data part)."""
  reg = go.regularizer(po)
  data, want_data = loss - reg, want_l - reg
  assert abs(data - want_data) < 1e-9 * max(1.0, abs(want_data)), (data, want_data)
  keep = np.ones(len(want_g), bool)
  if skip_noise:
    keep[-2] = False
  scale = max(1.0, float(np.max(np.abs(want_g[keep]))))
  np.testing.assert_allclose(grad[keep], want_g[keep], atol=1e-8 * scale, rtol=0)


def _oracle_retries(po, x, z, nv):
  return go.retrying_cholesky(go.kernel_matrix(po, x, z, np.arange(x.shape[0]) < nv))[2]


# ---------------------------------------------------------------------------------------------------------------
# vzgp_cholesky_retry: the panel ladder on spectra placed between two ladder steps
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [65, 200, 448])
def test_cholesky_retry_ladder(dev, n):
  for want in sorted(ff.LADDER_LAMBDA):
    a = ff.spd_with_lambda_min(n, ff.LADDER_LAMBDA[want], seed=n + want)
    l, shift, retries = dev.cholesky_retry(a)
    assert _routes(dev)[1] == PANEL
    assert retries == want, (want, retries)
    l = l.cpu().numpy()
    if want > ff.MAX_RETRIES:
      assert np.isnan(l).any()
      continue
    assert shift == ff.LADDER[want]
    ref = np.linalg.cholesky(a + shift * np.eye(n))
    np.testing.assert_allclose(l, ref, atol=1e-11 * max(1.0, np.max(np.abs(ref))), rtol=0)
    assert np.all(np.triu(l, 1) == 0)


# ---------------------------------------------------------------------------------------------------------------
# vzgp_fit: the retry ladder through the panel (N <= 64) and the dataflow kernel (N > 64)
# ---------------------------------------------------------------------------------------------------------------
FIT_CASES = [(64, 3, 0, 64), (64, 20, 2, 44), (65, 4, 0, 65), (65, 4, 0, 45), (129, 6, 2, 129), (129, 6, 2, 100),
             (700, 8, 0, 700), (700, 8, 0, 680), (4097, 6, 2, 4000)]


def _check_fit(d, x, y, z, po, nv, want_retries, route):
  gp = _gp()
  n = x.shape[0]
  valid = np.arange(n) < nv
  pred = go.precompute_predictive(po, x, y, z, row_valid=valid)
  assert pred.n_retries == want_retries
  retries = d.fit(x, y, _hyper(po), z=z, n_valid=nv)
  assert d.get_int('factor_route') == route
  assert retries == want_retries
  shift = ff.LADDER[retries]
  ky = go.kernel_matrix(po, x, z, row_valid=valid) + shift * np.eye(n)
  l = d.cholesky().cpu().numpy()
  # the factor itself: backward error at round-off, forward error within eps * cond(K_y + shift I) (a jittered
  # K_y with duplicated trials has cond ~ 1e5-1e6, so two factorisations may differ by ~1e-11 in L)
  assert np.max(np.abs(l @ l.T - ky)) <= 1e-12
  ev = np.linalg.eigvalsh(ky)
  tol_l = max(1e-11, 1e-15 * ev[-1] / ev[0])
  np.testing.assert_allclose(l, pred.chol, atol=tol_l * max(1.0, np.max(np.abs(pred.chol))), rtol=0)
  alpha = d.alpha().cpu().numpy()
  np.testing.assert_allclose(alpha, pred.alpha, atol=1e-8 * np.max(np.abs(pred.alpha)), rtol=0)
  assert np.max(np.abs(ky @ alpha - np.where(valid, y, 0.0))) <= 1e-11
  rng = np.random.default_rng(n)
  xs = rng.uniform(size=(500, x.shape[1]))
  zs = rng.integers(0, 3, size=(500, z.shape[1])).astype(np.int32) if z is not None else None
  mu_w, sd_w = go.predict(pred, xs, zs)
  out = d.score(xs, gp.Acquisition(1.8, False, 1.0), zs=zs, with_aux=True)
  d.synchronize()
  np.testing.assert_allclose(out['mean'].cpu().numpy(), mu_w, atol=1e-10, rtol=0)
  np.testing.assert_allclose(out['stddev'].cpu().numpy(), sd_w, atol=1e-10, rtol=0)
  np.testing.assert_allclose(out['score'].cpu().numpy(), go.ucb(mu_w, sd_w, 1.8), atol=1e-10, rtol=0)


@pytest.mark.parametrize('n,dc,dk,nv', FIT_CASES)
def test_fit_retry_ladder(dev, n, dc, dk, nv):
  route = DATAFLOW if n > 64 else PANEL
  for sn2, want in [(1e-30, 1)] + [(s, r) for s, r in sorted(ff.NEGATIVE_SN2.items(), reverse=True) if r <= 5]:
    x, y, z, po = ff.case_inputs('tripled', n, dc, dk, 1, sn2)
    _check_fit(dev, x, y, z, po, nv, want, route)


@pytest.mark.parametrize('n,dc,dk,nv', [(64, 3, 0, 64), (129, 6, 2, 100), (700, 8, 0, 700)])
def test_fit_ladder_exhausted_then_recovers(n, dc, dk, nv):
  d = _gp().DeviceGP(0)
  try:
    x, y, z, po = ff.case_inputs('tripled', n, dc, dk, 1, -3.0)
    with pytest.warns(RuntimeWarning):
      retries = d.fit(x, y, _hyper(po), z=z, n_valid=nv)
    assert d.get_int('factor_route') == (DATAFLOW if n > 64 else PANEL)
    assert retries == ff.MAX_RETRIES + 1 and d.cholesky_failed
    rng = np.random.default_rng(1)
    xs = rng.uniform(size=(500, dc))
    zs = rng.integers(0, 3, size=(500, dk)).astype(np.int32) if dk else None
    out = d.score(xs, _gp().Acquisition(1.8, False, 1.0), zs=zs)
    d.synchronize()
    assert np.isnan(out['score'].cpu().numpy()).all()
    # the same handle, a good fit: exact again
    x, y, z, po = ff.case_inputs('tripled', n, dc, dk, 1, 1e-30)
    _check_fit(d, x, y, z, po, nv, 1, DATAFLOW if n > 64 else PANEL)
    assert not d.cholesky_failed
  finally:
    d.close()


# ---------------------------------------------------------------------------------------------------------------
# NLL + gradient with one retry, on every route; then the same closure at well-conditioned parameters
# ---------------------------------------------------------------------------------------------------------------
# (n, dc, dk, n_valid, n_metrics, linear, route of the jittered evaluation, route of the good one, factor route)
NLL_RETRY_CASES = [
    (12, 3, 0, 8, 1, False, SMALL, SMALL, PANEL),
    (60, 3, 0, 40, 1, False, SMALL, SMALL, PANEL),
    (64, 20, 2, 44, 2, False, EAGER, GRAPH, PANEL),
    (60, 3, 0, 40, 8, False, EAGER, GRAPH, PANEL),
    (65, 4, 0, 45, 1, False, EAGER, GRAPH, DATAFLOW),
    (129, 6, 2, 109, 1, False, EAGER, GRAPH, DATAFLOW),
    (129, 6, 2, 109, 3, False, EAGER, GRAPH, DATAFLOW),
    (700, 8, 0, 680, 1, False, EAGER, GRAPH, DATAFLOW),
    (200, 0, 2, 180, 1, False, EAGER, GRAPH, DATAFLOW),
    (60, 3, 0, 40, 1, True, EAGER, EAGER, PANEL),
    (129, 6, 2, 109, 1, True, EAGER, EAGER, DATAFLOW),
]


@pytest.mark.parametrize('n,dc,dk,nv,m,lin,route_bad,route_good,froute', NLL_RETRY_CASES)
def test_nll_retry_every_route(dev, n, dc, dk, nv, m, lin, route_bad, route_good, froute):
  gp = _gp()
  x, y, z, po = ff.case_inputs('tripled', n, dc, dk, m, 1e-30)
  po = _with(po, linear=lin)
  # the masked identity rows carry the jitter too: an n_valid-row log-det would be off by this much
  assert 0.5 * m * (n - nv) * math.log1p(ff.JITTER0) >= 10 * 1e-9 * abs(go.nll(po, x, y, z, np.arange(n) < nv))
  assert _oracle_retries(po, x, z, nv) == 1
  want_l, want_g = _oracle_nll(po, x, y, z, nv)
  xt, yt, zt = _cuda(x), _cuda(y), _cuda(z, torch.int32)
  loss, grad, retries = dev.loss_and_grad(xt, yt, _hyper(po, lin), z=zt, n_valid=nv)
  assert _routes(dev) == (route_bad, froute)
  assert retries == 1
  # at sn2 = 1e-30 the noise regulariser's derivative (~1e30) swallows the data part of the noise component
  _assert_nll(loss, grad, want_l, want_g, po, skip_noise=True)
  # the closure the ARD driver uses: the jittered point, then a well-conditioned one on the same closure
  f = dev.make_loss_fn(xt, yt, zt, n_valid=nv, linear_coef=LIN_COEF if lin else None)
  l1, g1 = f(_hyper(po, lin).to_vector())
  assert _routes(dev) == (route_bad, froute)
  _assert_nll(l1, g1, want_l, want_g, po, skip_noise=True)
  good = _with(po, sn2=1e-2)
  want_l, want_g = _oracle_nll(good, x, y, z, nv)
  l2, g2 = f(_hyper(good, lin).to_vector())
  assert _routes(dev) == (route_good, froute)
  _assert_nll(l2, g2, want_l, want_g, good, skip_noise=False)
  fresh = gp.DeviceGP(0)
  try:
    l3, g3 = fresh.make_loss_fn(xt, yt, zt, n_valid=nv, linear_coef=LIN_COEF if lin else None)(
        _hyper(good, lin).to_vector())
    assert _routes(fresh) == (route_good, froute)
  finally:
    fresh.close()
  assert l2 == l3
  np.testing.assert_array_equal(g2, g3)


def test_graph_capture_after_linear_model():
  """The graph's label-padding node captures the handle's prior mean: a linear_coef evaluation (mean coef * m) on
  the same handles before a plain model's graph or batch capture must not shift that model's labels."""
  gp = _gp()
  x, y, z, po = ff.case_inputs('well', 129, 4, 1, 1, 2e-3)
  lin = _with(po, linear=True)
  xt, yt, zt = _cuda(x), _cuda(y), _cuda(z, torch.int32)
  devs = [gp.DeviceGP(0) for _ in range(2)]
  try:
    want_l, want_g = _oracle_nll(po, x, y, z, 129)
    for d in devs:
      d.loss_and_grad(xt, yt, _hyper(lin, True), z=zt)
      assert d.get_int('nll_route') == EAGER
    l1, g1 = devs[0].make_loss_fn(xt, yt, zt)(po.to_vector())
    assert _routes(devs[0]) == (GRAPH, DATAFLOW)
    _assert_nll(l1, g1, want_l, want_g, po, skip_noise=False)
    for d in devs:
      d.loss_and_grad(xt, yt, _hyper(lin, True), z=zt)
    losses, grads = gp.DeviceGP.make_batch_loss_fn(devs, xt, yt, zt)([0, 1], [po.to_vector()] * 2)
    for r in range(2):
      assert devs[r].get_int('nll_route') == BATCH
      _assert_nll(losses[r], grads[r], want_l, want_g, po, skip_noise=False)
  finally:
    for d in devs:
      d.close()


# ---------------------------------------------------------------------------------------------------------------
# Edges without retries: categorical-only and 64-feature models, 8 metrics
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n,dc,dk,nv,m', [(40, 0, 1, 40, 1), (64, 0, 4, 64, 1), (129, 0, 4, 65, 1), (129, 0, 1, 129, 2),
                                          (129, 64, 0, 129, 1), (64, 64, 0, 64, 1), (129, 5, 0, 120, 8),
                                          (40, 5, 0, 40, 8), (128, 4, 2, 64, 8)])
def test_nll_edges(dev, n, dc, dk, nv, m):
  x, y, z, po = ff.case_inputs('well', n, dc, dk, m, 2e-3)
  want_l, want_g = _oracle_nll(po, x, y, z, nv)
  loss, grad, retries = dev.loss_and_grad(_cuda(x), _cuda(y), _hyper(po), z=_cuda(z, torch.int32), n_valid=nv)
  assert _routes(dev) == ((SMALL, PANEL) if n <= 64 and m == 1 else (GRAPH, DATAFLOW if n > 64 else PANEL))
  assert retries == 0
  _assert_nll(loss, grad, want_l, want_g, po, skip_noise=False)


@pytest.mark.parametrize('n,dc,dk,nv', [(40, 0, 4, 40), (129, 0, 4, 100), (129, 64, 0, 129), (63, 64, 2, 63)])
def test_fit_edges(dev, n, dc, dk, nv):
  x, y, z, po = ff.case_inputs('well', n, dc, dk, 1, 2e-3)
  _check_fit(dev, x, y, z, po, nv, 0, DATAFLOW if n > 64 else PANEL)


# ---------------------------------------------------------------------------------------------------------------
# Batched ARD: one restart needs the jitter and falls back, the others stay on the batch graph
# ---------------------------------------------------------------------------------------------------------------
def _restart_params(po, r):
  """Restart r of a batch: r == 0 is the sn2 = 1e-30 point, the others are well conditioned."""
  import dataclasses
  if r == 0:
    return po
  return dataclasses.replace(po, observation_noise_variance=[1e-2, 3e-3, 5e-2, 2e-2][(r - 1) % 4],
                             signal_variance=0.6 + 0.2 * r,
                             continuous_length_scale_squared=po.continuous_length_scale_squared * (1.0 + 0.15 * r))


@pytest.mark.parametrize('n,dc,dk,nv,restarts', [(129, 6, 2, 109, 4), (700, 8, 0, 680, 4), (700, 8, 0, 700, 5),
                                                 (4097, 8, 0, 4097, 4)])
def test_batched_ard_fallback(n, dc, dk, nv, restarts):
  from vizier_b200 import ard
  gp = _gp()
  x, y, z, po = ff.case_inputs('tripled', n, dc, dk, 1, 1e-30)
  xt, yt, zt = _cuda(x), _cuda(y), _cuda(z, torch.int32)
  devs = [gp.DeviceGP(0) for _ in range(restarts)]
  single = gp.DeviceGP(0)
  share = ard._cta_share(restarts) if restarts == 5 else 0
  oracle = {}     # the two rounds share restarts; the host NLL costs seconds at N = 4097
  try:
    for d in devs + [single]:
      d.set_int('dataflow_ctas', share)
    fb = gp.DeviceGP.make_batch_loss_fn(devs, xt, yt, zt, n_valid=nv)
    fs = single.make_loss_fn(xt, yt, zt, n_valid=nv)
    for rnd, bad in ((0, True), (1, False)):
      ps = [_restart_params(po, r) if bad else _restart_params(po, r + 1) for r in range(restarts)]
      losses, grads = fb(list(range(restarts)), [p.to_vector() for p in ps])
      for r, p in enumerate(ps):
        jittered = p.observation_noise_variance < 1e-20
        key = p.to_vector().tobytes()
        if key not in oracle:
          oracle[key] = _oracle_nll(p, x, y, z, nv)
        want_l, want_g = oracle[key]
        assert devs[r].get_int('nll_route') == (EAGER if jittered else BATCH), (rnd, r)
        assert devs[r].get_int('factor_route') == DATAFLOW
        assert fb.status[r] == (1 if jittered else 0), (rnd, r)
        _assert_nll(losses[r], grads[r], want_l, want_g, p, skip_noise=jittered)
        if not jittered:
          l1, g1 = fs(p.to_vector())
          assert single.get_int('nll_route') == GRAPH
          assert losses[r] == l1
          np.testing.assert_array_equal(grads[r], g1)
  finally:
    for d in devs + [single]:
      d.close()


# ---------------------------------------------------------------------------------------------------------------
# The README's A/B switches, read once per process: each in a child process
# ---------------------------------------------------------------------------------------------------------------
_CHILD = r'''
import json, sys
import numpy as np
import torch
import fit_fixtures as ff
from vizier_b200 import gp
d = gp.DeviceGP(0)
out = []
for kind, fixture, n, dc, dk, nv, m, sn2 in json.loads(sys.argv[1]):
  x, y, z, po = ff.case_inputs(fixture, n, dc, dk, m, sn2)
  hp = gp.GPHyperParams(po.signal_variance, po.continuous_length_scale_squared, po.observation_noise_variance,
                        po.categorical_length_scale_squared)
  if kind == 'fit':
    r = d.fit(x, y, hp, z=z, n_valid=nv)
    out.append(dict(retries=r, factor_route=d.get_int('factor_route'), alpha=d.alpha().cpu().numpy().tolist()))
  else:
    zt = None if z is None else torch.from_numpy(z).cuda()
    loss, grad, r = d.loss_and_grad(torch.from_numpy(x).cuda(), torch.from_numpy(np.ascontiguousarray(y)).cuda(), hp,
                                    z=zt, n_valid=nv)
    out.append(dict(retries=r, nll_route=d.get_int('nll_route'), factor_route=d.get_int('factor_route'), loss=loss,
                    grad=grad.tolist()))
d.close()
print('RESULT ' + json.dumps(out))
'''

# (switch, [(kind, fixture, n, dc, dk, n_valid, n_metrics, sn2, retries, nll route, factor route)])
SWITCH_CASES = {
    'VZGP_DATAFLOW': [('fit', 'tripled', 129, 6, 2, 100, 1, 1e-30, 1, None, PANEL),
                      ('fit', 'well', 200, 5, 0, 200, 1, 2e-3, 0, None, PANEL),
                      ('nll', 'tripled', 129, 6, 2, 109, 1, 1e-30, 1, EAGER, PANEL),
                      ('nll', 'well', 200, 5, 0, 190, 1, 2e-3, 0, GRAPH, PANEL),
                      # nb = 65: the panel route's k_lauum planes inside the NLL graph
                      ('nll', 'well', 4097, 6, 0, 4000, 1, 2e-3, 0, GRAPH, PANEL)],
    'VZGP_NLL_GRAPH': [('nll', 'well', 129, 6, 2, 129, 1, 2e-3, 0, EAGER, DATAFLOW),
                       ('nll', 'well', 60, 3, 0, 60, 2, 2e-3, 0, EAGER, PANEL),
                       ('nll', 'tripled', 129, 6, 2, 109, 1, 1e-30, 1, EAGER, DATAFLOW)],
    'VZGP_NLL_SMALL': [('nll', 'well', 40, 3, 0, 40, 1, 2e-3, 0, GRAPH, PANEL),
                       ('nll', 'tripled', 60, 3, 0, 40, 1, 1e-30, 1, EAGER, PANEL),
                       ('fit', 'tripled', 60, 3, 0, 40, 1, 1e-30, 1, None, PANEL)],
}


@pytest.mark.parametrize('switch', sorted(SWITCH_CASES))
def test_environment_switches(switch):
  cases = SWITCH_CASES[switch]
  env = dict(os.environ)
  env[switch] = '0'
  env['PYTHONPATH'] = os.pathsep.join([ROOT, TESTS] + ([env['PYTHONPATH']] if env.get('PYTHONPATH') else []))
  arg = json.dumps([list(c[:8]) for c in cases])
  proc = subprocess.run([sys.executable, '-c', _CHILD, arg], cwd=ROOT, env=env, capture_output=True, text=True,
                        timeout=600)
  assert proc.returncode == 0, proc.stderr[-4000:]
  line = [ln for ln in proc.stdout.splitlines() if ln.startswith('RESULT ')][-1]
  got = json.loads(line[len('RESULT '):])
  for c, g in zip(cases, got):
    kind, fixture, n, dc, dk, nv, m, sn2, want_r, nll_route, froute = c
    assert g['retries'] == want_r and g['factor_route'] == froute, (c, g)
    x, y, z, po = ff.case_inputs(fixture, n, dc, dk, m, sn2)
    if kind == 'fit':
      pred = go.precompute_predictive(po, x, y, z, row_valid=np.arange(n) < nv)
      assert pred.n_retries == want_r
      np.testing.assert_allclose(g['alpha'], pred.alpha, atol=1e-8 * np.max(np.abs(pred.alpha)), rtol=0)
    else:
      assert g['nll_route'] == nll_route, (c, g)
      want_l, want_g = _oracle_nll(po, x, y, z, nv)
      _assert_nll(g['loss'], np.asarray(g['grad']), want_l, want_g, po, skip_noise=sn2 < 1e-20)
