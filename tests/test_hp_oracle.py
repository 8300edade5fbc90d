"""Pins the long-double posterior (oracle/hp_oracle.py) that the ill-conditioned scoring tests measure the
device and the fp64 oracle against: 50-digit mpmath on tiny problems, the fp64 oracle on a well-conditioned one."""
import mpmath as mp
import numpy as np
import pytest

from oracle import gp_oracle as go
from oracle import hp_oracle as hp

pytestmark = pytest.mark.skipif(not hp.has_extended_precision(), reason='np.longdouble is fp64 on this platform')


def _to_mp(v):
  """Exact mpmath value of a long double (its 64-bit mantissa fits in two doubles)."""
  hi = float(v)
  return mp.mpf(hi) + mp.mpf(float(np.longdouble(v) - np.longdouble(hi)))


def _mp_posterior(p, x, y, xs, z=None, zs=None):
  n, dc = x.shape
  ls2 = [mp.mpf(float(v)) for v in p.continuous_length_scale_squared]
  lk = [mp.mpf(float(v)) for v in p.categorical_length_scale_squared]

  def k(a, b, za, zb):
    d2 = sum((mp.mpf(float(a[i])) - mp.mpf(float(b[i]))) ** 2 / ls2[i] for i in range(dc))
    if za is not None:
      d2 += sum((1 if za[i] != zb[i] else 0) / lk[i] for i in range(len(za)))
    s = mp.sqrt(5 * d2)
    return mp.mpf(p.signal_variance) * (1 + s + s * s / 3) * mp.exp(-s)

  zi = (lambda zz, i: None if zz is None else zz[i])
  K = mp.matrix(n, n)
  for i in range(n):
    for j in range(n):
      K[i, j] = k(x[i], x[j], zi(z, i), zi(z, j)) + (mp.mpf(p.observation_noise_variance) if i == j else 0)
  alpha = mp.lu_solve(K, mp.matrix([mp.mpf(float(v)) for v in y]))
  mu, sd = [], []
  for m in range(xs.shape[0]):
    ks = mp.matrix([k(xs[m], x[i], zi(zs, m), zi(z, i)) for i in range(n)])
    sol = mp.lu_solve(K, ks)
    mu.append(sum(ks[i] * alpha[i] for i in range(n)))
    var = mp.mpf(p.signal_variance) - sum(ks[i] * sol[i] for i in range(n)) + mp.mpf(p.observation_noise_variance)
    sd.append(mp.sqrt(var))
  return mu, sd


@pytest.mark.parametrize('sn2,ls,dup', [(1e-3, None, False), (1e-8, 0.05, True)])
def test_hp_posterior_vs_mpmath(sn2, ls, dup):
  """At a well-conditioned and at an ill-conditioned tiny size (duplicated trials, sn2 = 1e-8) the long-double
  posterior is within a few long-double ulps times cond(K_y) of 50 digits, and far closer than fp64 LAPACK."""
  mp.mp.dps = 50
  n, d, dk = 12, 3, 1
  rng = np.random.default_rng(3)
  x = rng.uniform(size=(n, d))
  z = rng.integers(0, 3, size=(n, dk)).astype(np.int32)
  if dup:
    x[1], z[1] = x[0], z[0]
    x[5], z[5] = x[4], z[4]
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  xs = np.concatenate([rng.uniform(size=(4, d)), x[:2] + 1e-3])
  zs = np.concatenate([rng.integers(0, 3, size=(4, dk)), z[:2]]).astype(np.int32)
  ls2 = 0.5 * (1 + np.arange(d) / d) if ls is None else np.full(d, ls)
  p = go.GPParams(1.3, ls2, sn2, np.array([0.7]))
  mu_mp, sd_mp = _mp_posterior(p, x, y, xs, z, zs)
  hpp = hp.precompute_predictive(p, x, y, z)
  mu_h, sd_h = hp.predict(hpp, xs, zs)
  mu_f, sd_f = go.predict(go.precompute_predictive(p, x, y, z), xs, zs)
  err_h = max(float(abs(_to_mp(a) - b)) for a, b in zip(list(mu_h) + list(sd_h), mu_mp + sd_mp))
  err_f = max(float(abs(mp.mpf(float(a)) - b)) for a, b in zip(list(mu_f) + list(sd_f), mu_mp + sd_mp))
  scale = max(float(abs(v)) for v in mu_mp + sd_mp)
  cond = np.linalg.cond(go.kernel_matrix(p, x, z))
  assert err_h <= 64 * np.finfo(np.longdouble).eps * cond * scale, (err_h, cond)
  # the reference is what the GPU tests need it to be: much more accurate than fp64 LAPACK
  assert err_h <= max(err_f / 100, 1e-17), (err_h, err_f)


def test_hp_matches_fp64_oracle_when_well_conditioned():
  rng = np.random.default_rng(4)
  n, d, m = 150, 5, 300
  x = rng.uniform(size=(n, d))
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  xs = rng.uniform(size=(m, d))
  valid = np.arange(n) < 140
  p = go.GPParams(0.8, 0.5 * (1 + np.arange(d) / d), 1e-3)
  mu_h, sd_h = hp.predict(hp.precompute_predictive(p, x, y, row_valid=valid), xs)
  mu_f, sd_f = go.predict(go.precompute_predictive(p, x, y, row_valid=valid), xs)
  np.testing.assert_allclose(mu_h.astype(np.float64), mu_f, atol=1e-12, rtol=0)
  np.testing.assert_allclose(sd_h.astype(np.float64), sd_f, atol=1e-12, rtol=0)


def test_cholesky_ld_rejects_indefinite():
  with pytest.raises(ValueError):
    hp.cholesky_ld(np.array([[1.0, 2.0], [2.0, 1.0]]))
