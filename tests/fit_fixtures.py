"""Problems that force the Cholesky jitter retry with a clear margin, shared by the fit / NLL route tests.

Every trial appears three times (identical features and labels), so K(X, X) is exactly singular and
K_y = K + sn2 I has lambda_min = sn2 up to rounding:

  * sn2 = 1e-30: K_y is singular to rounding and the first factorisation fails; K_y + 1e-4 I has
    lambda_min ~ 1e-4, so the first jitter succeeds (one retry) on the device and in LAPACK alike.
  * sn2 < 0 (fit only: the C ABI just adds it to the diagonal, but the regulariser takes log sn2):
    lambda_min(K_y) = sn2 exactly, so the ladder 1e-4, 1e-3, ... stops at the first shift > -sn2.
    -3e-4 -> 2 retries, -3e-3 -> 3, -3e-2 -> 4, -0.3 -> 5; sn2 <= -2 exhausts it (6).

The labels are a smooth function of the features, so the quadratic form stays O(N) under the jitter.
tests/test_fit_fixtures.py pins the oracle's retry counts and the eigenvalue margins on the CPU.
"""
import numpy as np

from oracle import gp_oracle as go

JITTER0 = 1e-4
MAX_RETRIES = 5
# shift after k retries: 0, 1e-4, 1e-3, ...
LADDER = [0.0] + [JITTER0 * 10.0 ** k for k in range(MAX_RETRIES)]
# negative sn2 -> retries of the fit's ladder (6 = exhausted)
NEGATIVE_SN2 = {-3e-4: 2, -3e-3: 3, -3e-2: 4, -0.3: 5, -3.0: 6}


def tripled(n, dc, dk, seed=0):
  """(x [n, dc], y [n], z [n, dk] or None): trial t = i // 3 on row i, labels sin/cos of the features."""
  rng = np.random.default_rng(seed)
  t = -(-n // 3)
  xt = rng.uniform(size=(t, dc))
  zt = rng.integers(0, 3, size=(t, dk)).astype(np.int32) if dk else None
  yt = np.sin(3.0 * xt.sum(1)) if dc else np.zeros(t)
  if dk:
    yt = yt + 0.3 * np.cos(zt.sum(1))
  rows = np.arange(n) // 3
  return xt[rows].copy(), yt[rows].copy(), (zt[rows].copy() if dk else None)


def well_posed(n, dc, dk, seed=0):
  """Distinct trials with smooth labels and a little noise (no retry at the usual hyper-parameters)."""
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, dc))
  z = rng.integers(0, 3, size=(n, dk)).astype(np.int32) if dk else None
  y = (np.sin(3.0 * x.sum(1)) if dc else np.zeros(n)) + 0.05 * rng.normal(size=n)
  if dk:
    y = y + 0.3 * np.cos(z.sum(1))
  return x, y, z


def params(dc, dk, sn2, sf2=0.8):
  """(oracle GPParams, length-scale vectors): moderate length scales, so K has a large numerical rank."""
  ls_c = 0.3 * (1.0 + np.arange(dc) / max(dc, 1)) if dc else np.zeros(0)
  ls_k = np.linspace(0.6, 1.2, dk) if dk else None
  return go.GPParams(sf2, ls_c, sn2, ls_k)


def case_inputs(fixture, n, dc, dk, n_metrics, sn2):
  """(x, y, z, po) of one case: fixture 'tripled' or 'well'; y is [n] for one metric, else [n, n_metrics]
  (every metric a smooth function of the features, so duplicated trials keep identical labels)."""
  x, y, z = (tripled if fixture == 'tripled' else well_posed)(n, dc, dk, seed=n + dc + 7 * dk)
  if n_metrics > 1:
    y = np.stack([(1.0 + 0.25 * m) * y + 0.1 * m for m in range(n_metrics)], axis=1)
  return x, y, z, params(dc, dk, sn2)


def oracle_ky(po, x, z, n_valid):
  n = x.shape[0]
  return go.kernel_matrix(po, x, z, row_valid=np.arange(n) < n_valid)


def spd_with_lambda_min(n, lam_min, seed=0):
  """Q diag(lam) Q^T with lam_min = lam_min exactly in the spectrum and the rest in [0.5, 2]."""
  rng = np.random.default_rng(seed)
  q, _ = np.linalg.qr(rng.normal(size=(n, n)))
  lam = rng.uniform(0.5, 2.0, size=n)
  lam[0] = lam_min
  a = (q * lam) @ q.T
  return 0.5 * (a + a.T)


# lambda_min of vzgp_cholesky_retry fixtures -> retries: each sits a factor >= 3 inside its ladder interval
# (shift k-1 + lambda_min < 0 < shift k + lambda_min, with margins of at least 3x on both sides)
LADDER_LAMBDA = {0: 1e-2, 1: -3e-5, 2: -3e-4, 3: -3e-3, 4: -3e-2, 5: -0.3, 6: -3.0}
