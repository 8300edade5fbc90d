"""The dataflow factorisation (csrc/dataflow.cu) through its stage-wise entry point: L, L^-1 and the lower
triangle of A^-1 against LAPACK (NumPy / SciPy) from two 64-blocks up to nb = 128 (np = 2048 is BASELINE C4's size:
1549 tile tasks on 2 * SMs - 8 worker CTAs, 256 on a 132-SM H100 - more tasks than slots; the task count grows as
nb^3, so nb = 33, 65 and 128 run ticket queues 4x, 30x and 250x longer), alone and with several factorisations
running concurrently on different handles / streams (partial residency of every kernel)."""
import threading

import numpy as np
import pytest
import scipy.linalg as sla

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

import fit_fixtures as ff  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402

DATAFLOW = 1      # vzgp_get_int "factor_route"


def _spd(n, d=6, seed=0, sn2=1e-2):
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, d))
  return go.kernel_matrix(go.GPParams(1.0, np.full(d, 0.6), sn2), x)


def _lapack(a):
  want_l = np.linalg.cholesky(a)
  want_linv = sla.solve_triangular(want_l, np.eye(a.shape[0]), lower=True)
  return want_l, want_linv, want_linv.T @ want_linv


def _check(outs, want):
  l, linv, kinv = [o.cpu().numpy() for o in outs]
  want_l, want_linv, want_kinv = want
  np.testing.assert_allclose(l, want_l, atol=1e-11, rtol=0)
  assert np.all(np.triu(l, 1) == 0) and np.all(np.triu(linv, 1) == 0)
  scale = np.max(np.abs(want_linv))
  np.testing.assert_allclose(linv, want_linv, atol=1e-10 * scale, rtol=0)
  np.testing.assert_allclose(np.tril(kinv), np.tril(want_kinv), atol=1e-10 * np.max(np.abs(want_kinv)), rtol=0)


def _factor_inverse_bytes(n, handles=1):
  """Device bytes of factor_inverse at N = n: per handle 5 np^2 (L, L^-1, L^-T, K_y, workspace) and 4 np^2 (K^-1
  planes) doubles, plus the input and three outputs of N^2."""
  np_ = -(-n // 64) * 64
  return handles * 8 * (9 * np_ * np_ + 4 * n * n)


@pytest.mark.parametrize('n', [65, 128, 200, 640, 1000, 1537, 2000, 2049, 4097, 8192])
def test_factor_inverse_matches_lapack(n):
  from vizier_b200 import gp
  ff.require_device_bytes(_factor_inverse_bytes(n))
  dev = gp.DeviceGP(0)
  a = _spd(n, seed=n)
  want = _lapack(a)
  try:
    for _ in range(2):     # second call: warm workspaces, same answer
      outs, bad = dev.factor_inverse(a)
      dev.synchronize()
      assert dev.get_int('factor_route') == DATAFLOW
      assert bad == 0
      _check(outs, want)
      del outs
  finally:
    dev.close()


def _assert_bad_pivot_flagged(n, row):
  from vizier_b200 import gp
  ff.require_device_bytes(_factor_inverse_bytes(n))
  dev = gp.DeviceGP(0)
  a = _spd(n, seed=3)
  a[row, row] = -5.0          # not positive definite from the 64-block holding `row` on
  try:
    outs, bad = dev.factor_inverse(a)      # a tile wait that timed out would raise here
    dev.synchronize()
    assert dev.get_int('factor_route') == DATAFLOW
    assert bad == 1
  finally:
    dev.close()


def test_bad_pivot_is_flagged_not_hung():
  _assert_bad_pivot_flagged(300, 200)    # breaks in the 4th of 5 64-blocks


def test_bad_pivot_in_the_last_of_128_blocks_is_flagged_not_hung():
  """N = 8192: every task before the last 64-block runs first, and the CTAs waiting on the flagged tiles must
  still drain a ticket queue 250x longer than C4's."""
  _assert_bad_pivot_flagged(8192, 8170)


def _assert_concurrent_bit_identical(n, share=None):
  """Four dataflow kernels at once (the ARD restarts): each gets only part of the GPU, tickets keep every
  one of them deadlock-free, results are bit-identical to the solo run.  share: the number of concurrent
  evaluations whose ARD worker share (ard._cta_share) each handle gets; None lets every handle take every slot."""
  from vizier_b200 import ard, gp
  ff.require_device_bytes(_factor_inverse_bytes(n, 4) + 8 * 8 * n * n)
  mats = [_spd(n, seed=40 + i) for i in range(4)]
  devs = [gp.DeviceGP(0) for _ in range(4)]
  if share:
    for d in devs:
      d.set_int('dataflow_ctas', ard._cta_share(share))
  solo = []
  for d, a in zip(devs, mats):
    outs, bad = d.factor_inverse(a)
    d.synchronize()
    assert bad == 0
    solo.append([o.cpu().numpy() for o in outs])
  res = [None] * 4

  def run(i):
    for _ in range(5):
      outs, bad = devs[i].factor_inverse(mats[i])
      devs[i].synchronize()
      assert bad == 0
    res[i] = [o.cpu().numpy() for o in outs]

  ths = [threading.Thread(target=run, args=(i,)) for i in range(4)]
  [t.start() for t in ths]
  [t.join() for t in ths]
  for d in devs:
    assert d.get_int('factor_route') == DATAFLOW
    d.close()
  for i in range(4):
    for got, want in zip(res[i], solo[i]):
      np.testing.assert_array_equal(got, want)
  _check([torch.from_numpy(x) for x in res[0]], _lapack(mats[0]))


def test_concurrent_factorisations_on_four_streams():
  _assert_concurrent_bit_identical(1000)


def test_concurrent_factorisations_with_the_ard_share_at_nb65():
  """N = 4097 (nb = 65), each handle with the worker slots the ARD driver gives each of four evaluations."""
  _assert_concurrent_bit_identical(4097, share=4)
