"""The dataflow factorisation (csrc/dataflow.cu) through its stage-wise entry point: L, L^-1 and the lower
triangle of A^-1 against LAPACK (NumPy / SciPy) from two 64-blocks up to BASELINE C4's size (np = 2048:
1549 tile tasks on 2 * SMs - 8 worker CTAs, 256 on a 132-SM H100 - more tasks than slots), alone and with several factorisations
running concurrently on different handles / streams (partial residency of every kernel)."""
import threading

import numpy as np
import pytest
import scipy.linalg as sla

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from oracle import gp_oracle as go  # noqa: E402


def _spd(n, d=6, seed=0, sn2=1e-2):
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, d))
  return go.kernel_matrix(go.GPParams(1.0, np.full(d, 0.6), sn2), x)


def _check(outs, a):
  n = a.shape[0]
  l, linv, kinv = [o.cpu().numpy() for o in outs]
  want_l = np.linalg.cholesky(a)
  want_linv = sla.solve_triangular(want_l, np.eye(n), lower=True)
  want_kinv = want_linv.T @ want_linv
  np.testing.assert_allclose(l, want_l, atol=1e-11, rtol=0)
  assert np.all(np.triu(l, 1) == 0) and np.all(np.triu(linv, 1) == 0)
  scale = np.max(np.abs(want_linv))
  np.testing.assert_allclose(linv, want_linv, atol=1e-10 * scale, rtol=0)
  np.testing.assert_allclose(np.tril(kinv), np.tril(want_kinv), atol=1e-10 * np.max(np.abs(want_kinv)), rtol=0)


@pytest.mark.parametrize('n', [65, 128, 200, 640, 1000, 1537, 2000])
def test_factor_inverse_matches_lapack(n):
  from vizier_b200 import gp
  dev = gp.DeviceGP(0)
  a = _spd(n, seed=n)
  for _ in range(2):     # second call: warm workspaces, same answer
    outs, bad = dev.factor_inverse(a)
    dev.synchronize()
    assert bad == 0
    _check(outs, a)
  dev.close()


def test_bad_pivot_is_flagged_not_hung():
  from vizier_b200 import gp
  dev = gp.DeviceGP(0)
  a = _spd(300, seed=3)
  a[200, 200] = -5.0          # not positive definite from the 4th 64-block on
  outs, bad = dev.factor_inverse(a)
  dev.synchronize()
  assert bad == 1
  dev.close()


def test_concurrent_factorisations_on_four_streams():
  """Four dataflow kernels at once (the ARD restarts): each gets only part of the GPU, tickets keep every
  one of them deadlock-free, results are bit-identical to the solo run."""
  from vizier_b200 import gp
  n = 1000
  mats = [_spd(n, seed=40 + i) for i in range(4)]
  devs = [gp.DeviceGP(0) for _ in range(4)]
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
  for i in range(4):
    for got, want in zip(res[i], solo[i]):
      np.testing.assert_array_equal(got, want)
  _check([torch.from_numpy(x) for x in res[0]], mats[0])
