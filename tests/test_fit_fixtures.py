"""The jitter fixtures of tests/fit_fixtures.py, checked on the CPU: the oracle's retry count and the eigenvalue
margin that makes the device and LAPACK agree on it (the GPU route tests rely on both)."""
import math

import numpy as np
import pytest

import fit_fixtures as ff
from oracle import gp_oracle as go


def _brackets(lam, k):
  """lambda_min = lam puts the ladder's first success at retry k with a factor of about 3 on both sides:
  |lam| >= 2.9 LADDER[k-1] (attempt k - 1 fails clearly) and LADDER[k] >= 2.9 |lam| (attempt k succeeds clearly)."""
  ok = True
  if k >= 1:
    ok = ok and -lam >= 2.9 * ff.LADDER[k - 1]
  if k <= ff.MAX_RETRIES:
    ok = ok and (lam > 0 if k == 0 else 2.9 * -lam <= ff.LADDER[k])
  return ok


ONE_RETRY = [(12, 3, 0, 12), (12, 3, 0, 8), (60, 3, 0, 40), (64, 20, 2, 64), (64, 3, 0, 44), (65, 4, 0, 65),
             (65, 4, 0, 45), (129, 6, 2, 129), (129, 6, 2, 109), (700, 8, 0, 700), (700, 8, 0, 680),
             (200, 0, 2, 200), (200, 0, 2, 180)]


@pytest.mark.parametrize('n,dc,dk,nv', ONE_RETRY)
def test_tripled_rows_at_sn2_1e30_retry_once(n, dc, dk, nv):
  x, y, z, po = ff.case_inputs('tripled', n, dc, dk, 1, 1e-30)
  ky = ff.oracle_ky(po, x, z, nv)
  _, shift, retries = go.retrying_cholesky(ky)
  assert (retries, shift) == (1, ff.JITTER0)
  lam = np.linalg.eigvalsh(ky)[0]
  lam_j = np.linalg.eigvalsh(ky + ff.JITTER0 * np.eye(n))[0]
  # singular to rounding (the unshifted factorisation has nothing to stand on) ...
  assert abs(lam) < 1e-12
  # ... and the first jitter leaves lambda_min within 1 % of 1e-4: far from any rounding decision
  assert 0.99e-4 < lam_j < 1.01e-4
  # labels are smooth, so the quadratic form stays O(N) under the jitter
  pred = go.precompute_predictive(po, x, y, z, row_valid=np.arange(n) < nv)
  assert 0.5 * float(np.dot(np.where(np.arange(n) < nv, y, 0.0), pred.alpha)) < 10.0 * n


@pytest.mark.parametrize('n,dc,dk,nv', [c for c in ONE_RETRY if c[3] < c[0]])
def test_masked_rows_shift_the_logdet_far_beyond_the_tolerance(n, dc, dk, nv):
  """With n_valid < N the masked identity rows carry the jitter too (log(1 + 1e-4) each): the offset the NLL tests
  rely on to tell an N-row log-det from an n_valid-row one must be >= 10x their 1e-9 relative tolerance."""
  x, y, z, po = ff.case_inputs('tripled', n, dc, dk, 1, 1e-30)
  data = go.nll(po, x, y, z, row_valid=np.arange(n) < nv)
  offset = 0.5 * (n - nv) * math.log1p(ff.JITTER0)
  assert offset >= 10 * 1e-9 * max(1.0, abs(data))


@pytest.mark.parametrize('sn2,want', sorted(ff.NEGATIVE_SN2.items()))
def test_negative_sn2_walks_the_ladder(sn2, want):
  x, _, z, po = ff.case_inputs('tripled', 129, 6, 2, 1, sn2)
  ky = ff.oracle_ky(po, x, z, 129)
  lam = np.linalg.eigvalsh(ky)[0]
  assert abs(lam - sn2) < 1e-12      # the duplicates pin lambda_min(K_y) to sn2
  l, shift, retries = go.retrying_cholesky(ky)
  assert _brackets(lam, want)
  if want <= ff.MAX_RETRIES:
    assert retries == want and shift == ff.LADDER[want]
    assert np.all(np.isfinite(l))
  else:   # exhausted: the oracle stops after MAX_RETRIES with NaN; the C ABI reports MAX_RETRIES + 1
    assert retries == ff.MAX_RETRIES and np.isnan(l).all()


@pytest.mark.parametrize('n', [65, 200, 448])
@pytest.mark.parametrize('want', sorted(ff.LADDER_LAMBDA))
def test_cholesky_retry_spectra(n, want):
  lam = ff.LADDER_LAMBDA[want]
  a = ff.spd_with_lambda_min(n, lam, seed=n + want)
  ev = np.linalg.eigvalsh(a)
  assert abs(ev[0] - lam) < 1e-13 and ev[1] > 0.49
  assert _brackets(lam, want)
  _, shift, retries = go.retrying_cholesky(a)
  assert retries == min(want, ff.MAX_RETRIES)
  if want <= ff.MAX_RETRIES:
    assert shift == ff.LADDER[want]
