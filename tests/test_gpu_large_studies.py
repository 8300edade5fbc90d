"""Studies past C4's 2048 trials where no other test has a home: both sides of the dataflow factorisation's
nb = 256 limit through vzgp_fit, the panel kernels at nb = 65 and 128 through their stage-wise entry points, and a
check that every comparison used at these sizes catches a 1e-9 relative error in one tile, partial or candidate.

k_chol_dataflow (csrc/dataflow.cu) plans nb = np / 64 <= 256 blocks; a study of N > 16384 trials is factored by the
panel kernels (potrf_blocked, trtri_doubling).  Every case first asserts the route it is meant to take (vzgp_get_int
"factor_route", "score_route") and then compares against oracle/gp_oracle.py or LAPACK with the tolerances of the
neighbouring tests: L 1e-11, L^-1 and K^-1 1e-10 of their largest entry, alpha 1e-8 of max |alpha|, scores, means and
stddevs 1e-10.  At N >= 16384 the factor is checked by its backward error ||L L^T - K_y||_max / ||K_y||_max, formed
on the device by torch (cuBLAS, none of this project's kernels), against 2 N eps.

Device memory of a case: a fitted handle holds 5 np^2 doubles (L, L^-1, L^-T, K_y, workspace), the factor_inverse /
NLL planes of K^-1 another 4 np^2, the k_score scratch grid * 64 * np; the tensors a case keeps on the device come on
top.  A case that would not fit in the free memory is skipped with the bytes it needs."""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.linalg as sla

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

import fit_fixtures as ff  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402
from test_gpu_dataflow import _check as check_factor_inverse, _lapack, _spd  # noqa: E402
from test_gpu_score_routes import _check_oracle  # noqa: E402

PANEL, DATAFLOW = 0, 1                  # vzgp_get_int "factor_route"
SPLIT, CLUSTER = 1, 2                   # vzgp_get_int "score_route"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = np.finfo(np.float64).eps
RESIDUAL_FACTOR = 2.0                   # backward error bound: RESIDUAL_FACTOR * N * eps
PERTURB = 1e-9                          # relative error the sensitivity test plants


def _gp():
  from vizier_b200 import gp
  return gp


def _np(n):
  return -(-n // 64) * 64


@pytest.fixture(scope='module')
def device_room():
  """need(case bytes) -> skips unless the free device memory holds them now; returns the free bytes before."""
  sm = torch.cuda.get_device_properties(0).multi_processor_count

  def need(nbytes):
    ff.require_device_bytes(nbytes)
    return torch.cuda.mem_get_info(0)[0]

  need.sm = sm
  return need


def _report(label, free0):
  torch.cuda.synchronize()
  print(f'{label}: {(free0 - torch.cuda.mem_get_info(0)[0]) / 2**30:.2f} GiB of device memory in use')


def _release():
  torch.cuda.synchronize()
  torch.cuda.empty_cache()


def _assert_residual(l, k, n):
  """||L L^T - K_y||_max / ||K_y||_max <= RESIDUAL_FACTOR * N * eps, on the device (L, K_y torch tensors)."""
  r = l @ l.T
  r.sub_(k)
  rel = float(r.abs_().max() / k.abs().max())
  del r
  assert rel <= RESIDUAL_FACTOR * n * EPS, (rel, RESIDUAL_FACTOR * n * EPS)
  return rel


# ---------------------------------------------------------------------------------------------------------------
# vzgp_fit on both sides of the dataflow limit: nb = 256 (the last size k_chol_dataflow plans) and nb = 257
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n,route', [(16384, DATAFLOW), (16385, PANEL)], ids=['N16384-dataflow', 'N16385-panel'])
def test_fit_across_dataflow_limit(device_room, n, route):
  gp = _gp()
  np_ = _np(n)
  free0 = device_room(8 * (5 * np_ * np_ + device_room.sm * 64 * np_ + 3 * n * n))
  d = 4
  rng = np.random.default_rng(n)
  x = rng.uniform(size=(n, d))
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  ls2 = 0.5 * (1 + np.arange(d) / d)
  po, pg = go.GPParams(1.0, ls2, 1e-2), gp.GPHyperParams(1.0, ls2, 1e-2)
  # precompute_predictive's steps, keeping K_y for the residual check (it costs seconds to rebuild at this size)
  ky = go.kernel_matrix(po, x)
  l_host, _, retries = go.retrying_cholesky(ky)
  assert retries == 0
  alpha = sla.solve_triangular(l_host.T, sla.solve_triangular(l_host, y, lower=True), lower=False)
  pred = go.Predictive(po, x, None, l_host, alpha, np.ones(n, bool))
  del l_host
  dev = gp.DeviceGP(0)
  try:
    assert dev.fit(x, y, pg) == 0
    assert dev.get_int('factor_route') == route
    np.testing.assert_allclose(dev.alpha().cpu().numpy(), alpha, atol=1e-8 * np.max(np.abs(alpha)), rtol=0)
    # one cluster-route pool: the first 256 candidates and the last tile against the oracle
    dev.set_int('score_i8', 0)
    tiles = device_room.sm // 2 + 1
    m = (tiles - 1) * 64 + 17
    xs = rng.uniform(-0.2, 1.2, size=(m, d))
    xs[:3] = x[:3]
    radius = go.trust_radius(n, d, 0)
    out = dev.score(xs, gp.Acquisition(1.8, True, radius), with_aux=True)
    dev.synchronize()
    assert (dev.get_int('score_route'), dev.get_int('score_nsplit')) == (CLUSTER, 1)
    pick = np.r_[0:256, (tiles - 1) * 64:m]
    want, aux = go.score_with_aux(pred, xs[pick])
    got = {k: out[k].cpu().numpy()[pick] for k in ('score', 'mean', 'stddev', 'linf_distance')}
    _check_oracle(got, {'score': want, **aux})
    # the factor by its backward error
    kt = torch.from_numpy(ky).cuda()
    del ky
    lt = dev.cholesky()
    print(f'N={n}: ||L L^T - K_y|| / ||K_y|| = {_assert_residual(lt, kt, n):.3e}')
    _report(f'N={n} fit', free0)
    del kt, lt, out
  finally:
    dev.close()
    _release()


# ---------------------------------------------------------------------------------------------------------------
# The panel kernels at nb = 65 and 128: potrf_blocked and trtri_doubling (non-power-of-two right parts of the
# recursive doubling) through vzgp_cholesky_retry / vzgp_tri_inverse, which never take the dataflow kernel
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [4097, 8192])
def test_panel_kernels_match_lapack(device_room, n):
  np_ = _np(n)
  free0 = device_room(8 * (5 * np_ * np_ + 3 * n * n))
  dev = _gp().DeviceGP(0)
  a = _spd(n, seed=n + 1)
  want_l, want_linv, _ = _lapack(a)
  try:
    l, shift, retries = dev.cholesky_retry(a)
    assert dev.get_int('factor_route') == PANEL
    assert (shift, retries) == (0.0, 0)
    np.testing.assert_allclose(l.cpu().numpy(), want_l, atol=1e-11 * max(1.0, np.max(np.abs(want_l))), rtol=0)
    del l
    linv = dev.tri_inverse(want_l).cpu().numpy()
    assert np.all(np.triu(linv, 1) == 0)
    np.testing.assert_allclose(linv, want_linv, atol=1e-10 * np.max(np.abs(want_linv)), rtol=0)
    _report(f'N={n} panel kernels', free0)
  finally:
    dev.close()
    _release()


_CHILD = r'''
import sys
import numpy as np
from vizier_b200 import gp
d = gp.DeviceGP(0)
outs, bad = d.factor_inverse(np.load(sys.argv[1]))
d.synchronize()
np.save(sys.argv[2], np.stack([o.cpu().numpy() for o in outs]))
print('RESULT', bad, d.get_int('factor_route'))
d.close()
'''


def test_factor_inverse_panel_route_at_nb65(device_room, tmp_path):
  """vzgp_factor_inverse with VZGP_DATAFLOW=0 (read once per process, so in a child): potrf_blocked,
  trtri_doubling, k_lauum in its partial planes and k_sum_planes at N = 4097, against LAPACK."""
  n = 4097
  np_ = _np(n)
  device_room(8 * (9 * np_ * np_ + 4 * n * n))
  a = _spd(n, seed=7)
  np.save(tmp_path / 'a.npy', a)
  env = dict(os.environ)
  env['VZGP_DATAFLOW'] = '0'
  env['PYTHONPATH'] = os.pathsep.join([ROOT] + ([env['PYTHONPATH']] if env.get('PYTHONPATH') else []))
  proc = subprocess.run([sys.executable, '-c', _CHILD, str(tmp_path / 'a.npy'), str(tmp_path / 'out.npy')], cwd=ROOT,
                        env=env, capture_output=True, text=True, timeout=600)
  assert proc.returncode == 0, proc.stderr[-4000:]
  line = [ln for ln in proc.stdout.splitlines() if ln.startswith('RESULT ')][-1]
  bad, route = map(int, line.split()[1:])
  assert route == PANEL and bad == 0
  outs = np.load(tmp_path / 'out.npy')
  check_factor_inverse([torch.from_numpy(o) for o in outs], _lapack(a))


# ---------------------------------------------------------------------------------------------------------------
# Sensitivity: each comparison above fails when one tile, one k_score partial or one candidate is off by 1e-9
# ---------------------------------------------------------------------------------------------------------------
def _perturb_tile(a, rel=PERTURB):
  """A copy of a with the 64 x 64 tile holding its largest |entry| scaled by 1 + rel (a lower-triangular tile
  stays lower triangular)."""
  a = a.copy()
  i, j = np.unravel_index(np.argmax(np.abs(a)), a.shape)
  r, c = slice(i // 64 * 64, i // 64 * 64 + 64), slice(j // 64 * 64, j // 64 * 64 + 64)
  a[r, c] *= 1.0 + rel
  return a


@pytest.fixture(scope='module')
def sensitivity_data(device_room):
  """Device results at N = 4097 and the references they pass against: factor_inverse (dataflow) with LAPACK, and
  a split-route pool (17 CTAs per tile) of the fitted model with the oracle."""
  gp = _gp()
  n, d = 4097, 5
  np_ = _np(n)
  device_room(8 * (9 * np_ * np_ + device_room.sm * 64 * np_ + 6 * n * n))
  a = _spd(n, seed=11)
  rng = np.random.default_rng(12)
  x = rng.uniform(size=(n, d))
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  ls2 = 0.5 * (1 + np.arange(d) / d)
  po = go.GPParams(1.0, ls2, 1e-3)
  xs = rng.uniform(size=(9 * 64, d))
  xs[:3] = x[:3]              # candidates on trials 0-2: block 0 of L^-1 k* explains most of their variance
  xs[-1] = 3.0                # far from every trial: stddev ~ 1, so a 1e-9 relative error exceeds the 1e-10 tolerance
  dev = gp.DeviceGP(0)
  try:
    outs, bad = dev.factor_inverse(a)
    dev.synchronize()
    assert bad == 0 and dev.get_int('factor_route') == DATAFLOW
    lt = outs[0]
    kt = torch.from_numpy(a).cuda()
    factor = [o.cpu().numpy() for o in outs]
    dev.fit(x, y, gp.GPHyperParams(1.0, ls2, 1e-3))
    dev.set_int('score_i8', 0)
    out = dev.score(xs, gp.Acquisition(1.8, False, 1.0), with_aux=True)
    dev.synchronize()
    assert (dev.get_int('score_route'), dev.get_int('score_nsplit')) == (SPLIT, 17)
    got = {k: out[k].cpu().numpy() for k in ('score', 'mean', 'stddev')}
    yield dict(n=n, a=a, factor=factor, lapack=_lapack(a), lt=lt, kt=kt, got=got, po=po, x=x, y=y, xs=xs)
    del lt, kt, outs, out
  finally:
    dev.close()
    _release()


def _split_partial(data):
  """Candidate tile 0's partial from split 0 of k_score: sum_r (L^-1 k*)_r^2 over the rows of column blocks 0 and
  nblocks - 1 (128 rows each; split s takes blocks s and nblocks - 1 - s)."""
  pred = go.precompute_predictive(data['po'], data['x'], data['y'])
  ks = go.kernel(data['po'], data['xs'][:64], data['x'])
  v = sla.solve_triangular(pred.chol, ks.T, lower=True)
  last = (_np(data['n']) + 127) // 128 - 1
  rows = np.r_[0:128, 128 * last:data['n']]
  return pred, np.sum(v[rows] ** 2, axis=0)


@pytest.mark.parametrize('what', ['L', 'Linv', 'Kinv', 'residual', 'nsplit-partial', 'stddev'])
def test_comparisons_catch_a_1e9_error(sensitivity_data, what):
  data = sensitivity_data
  if what in ('L', 'Linv', 'Kinv'):
    check_factor_inverse([torch.from_numpy(f) for f in data['factor']], data['lapack'])
    k = ['L', 'Linv', 'Kinv'].index(what)
    bad = list(data['factor'])
    bad[k] = _perturb_tile(np.tril(bad[k]))
    with pytest.raises(AssertionError):
      check_factor_inverse([torch.from_numpy(f) for f in bad], data['lapack'])
    return
  if what == 'residual':
    _assert_residual(data['lt'], data['kt'], data['n'])
    bad = torch.from_numpy(_perturb_tile(data['factor'][0])).cuda()
    with pytest.raises(AssertionError):
      _assert_residual(bad, data['kt'], data['n'])
    return
  pred, partial = _split_partial(data)
  mu, sd = go.predict(pred, data['xs'])
  want = {'score': go.ucb(mu, sd, 1.8), 'mean': mu, 'stddev': sd}
  _check_oracle(data['got'], want)
  bad = dict(data['got'])
  sd_bad = bad['stddev'].copy()
  if what == 'stddev':
    i = int(np.argmax(sd_bad))
    sd_bad[i] *= 1.0 + PERTURB
  else:
    # the first CTA's partial of tile 0 off by 1e-9 relative: var = sf2 + sn2 - sum of the partials
    sd_bad[:64] = np.sqrt(sd_bad[:64] ** 2 - PERTURB * partial)
  bad['stddev'] = sd_bad
  with pytest.raises(AssertionError):
    _check_oracle(bad, want)
