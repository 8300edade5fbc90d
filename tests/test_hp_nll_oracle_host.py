"""Pins the long-double ARD loss and gradient (oracle/hp_oracle.loss_and_grad_ld) that test_gpu_nll_conditioning.py
measures the device and the fp64 oracle against: the fp64 oracle where K_y is well conditioned, 40-digit mpmath on
tiny ill-conditioned problems, and the bound of tests/nll_conditioning.py, which must reject an fp64 evaluation whose
factorisation carries 50 ulp of backward error."""
import math

import numpy as np
import pytest

import fit_fixtures as ff
import nll_conditioning as nc
from oracle import gp_oracle as go
from oracle import hp_oracle as hp

pytestmark = pytest.mark.skipif(not hp.has_extended_precision(), reason='np.longdouble is fp64 on this platform')


def _to_mp(mp, v):
  """Exact mpmath value of a long double (its 64-bit mantissa fits in two doubles)."""
  hi = float(v)
  return mp.mpf(hi) + mp.mpf(float(np.longdouble(v) - np.longdouble(hi)))


# (n, dc, dk, n_valid, n_metrics, linear)
WELL_CASES = [(40, 3, 0, 40, 1, False), (60, 4, 2, 60, 1, False), (129, 4, 2, 100, 1, False),
              (60, 3, 0, 50, 2, False), (60, 3, 1, 55, 1, True)]


@pytest.mark.parametrize('n,dc,dk,nv,m,lin', WELL_CASES)
def test_matches_fp64_oracle_when_well_conditioned(n, dc, dk, nv, m, lin):
  """sn2 = 2e-3: the long-double loss and every gradient component equal gp_oracle.loss_and_grad to 1e-12 relative
  (1e-12 absolute for components below 1, where the fp64 oracle's own cancellation error is ~1e-13)."""
  x, y, z, po = ff.case_inputs('well', n, dc, dk, m, 2e-3)
  if lin:
    po.linear = go.LinearParams(nc.LIN['coef'], nc.LIN['slope_amplitude'], nc.LIN['shift'], nc.LIN['mean_constant'])
  rv = np.arange(n) < nv
  coef = nc.linear_coef(lin)
  want_l, want_g = go.loss_and_grad(po.to_vector(), x, y, z, rv, linear_coef=coef)
  got = hp.loss_and_grad_ld(po.to_vector(), x, y, z, rv, linear_coef=coef)
  assert got.grad.shape == want_g.shape
  assert abs(float(got.loss) - want_l) <= 1e-12 * abs(want_l)
  np.testing.assert_allclose(got.grad.astype(np.float64), want_g, rtol=1e-12, atol=1e-12)
  np.testing.assert_allclose(got.alpha.astype(np.float64).reshape(n, -1),
                             go.precompute_predictive(po, x, y, z, rv).alpha.reshape(n, -1), rtol=0,
                             atol=1e-12 * float(np.max(np.abs(got.alpha))))
  # the scales bound what they measure: every component's data part is a sum of terms no larger in total
  assert np.all(np.abs(got.grad - got.grad_reg) <= got.grad_scale * (1 + 1e-15))
  assert abs(got.data) <= got.data_scale


def test_shift_is_the_jitter_of_a_retried_factorisation():
  """Every trial three times at sn2 = 1e-30: LAPACK needs one retry; with that shift the long-double gradient is the
  fp64 oracle's (the noise component apart, where the 1e30 regulariser derivative swallows the data part)."""
  x, y, z, po = ff.case_inputs('tripled', 30, 3, 1, 1, 1e-30)
  assert go.retrying_cholesky(go.kernel_matrix(po, x, z))[2] == 1
  want_l, want_g = go.loss_and_grad(po.to_vector(), x, y, z)
  got = hp.loss_and_grad_ld(po.to_vector(), x, y, z, shift=ff.JITTER0)
  reg = go.regularizer(po)
  assert abs((float(got.loss) - reg) - (want_l - reg)) <= 1e-12 * abs(want_l - reg)
  keep = np.arange(len(want_g)) != len(want_g) - 2
  np.testing.assert_allclose(got.grad.astype(np.float64)[keep], want_g[keep], rtol=1e-11, atol=0)


def _mp_loss_and_grad(mp, theta, x, y):
  """The loss and gradient of gp_oracle.loss_and_grad (plain Matern model, one metric) in mpmath."""
  n, dc = x.shape
  p = go.GPParams.from_vector(theta, dc, 0)
  ls2 = [mp.mpf(float(v)) for v in p.continuous_length_scale_squared]
  sf2, sn2 = mp.mpf(p.signal_variance), mp.mpf(p.observation_noise_variance)
  xs = [[mp.mpf(float(v)) for v in row] for row in x]
  K, E, sq = mp.matrix(n, n), mp.matrix(n, n), [mp.matrix(n, n) for _ in range(dc)]
  for i in range(n):
    for j in range(n):
      for d in range(dc):
        sq[d][i, j] = (xs[i][d] - xs[j][d]) ** 2
      s = mp.sqrt(5 * sum(sq[d][i, j] / ls2[d] for d in range(dc)))
      K[i, j] = sf2 * (1 + s + s * s / 3) * mp.exp(-s)
      E[i, j] = -mp.mpf(5) / 6 * sf2 * (1 + s) * mp.exp(-s)
  Ky = K + sn2 * mp.eye(n)
  L = mp.cholesky(Ky)
  yv = mp.matrix([mp.mpf(float(v)) for v in y])
  alpha = mp.cholesky_solve(Ky, yv)
  loss = (sum(yv[i] * alpha[i] for i in range(n)) / 2 + sum(mp.log(L[i, i]) for i in range(n))
          + n * mp.log(2 * mp.pi) / 2)

  def reg(v, c):
    return go.REG_WEIGHT * mp.log(v / c) ** 2, 2 * go.REG_WEIGHT * mp.log(v / c) / v

  G = mp.inverse(Ky) - alpha * alpha.T
  grad = []
  for d in range(dc):
    r, rg = reg(ls2[d], mp.mpf(go.REG_CENTER_LENGTH))
    loss += r
    grad.append(sum(G[i, j] * E[i, j] * (-sq[d][i, j] / ls2[d] ** 2) for i in range(n) for j in range(n)) / 2 + rg)
  r, rg = reg(sn2, mp.mpf(go.REG_CENTER_NOISE))
  loss += r
  grad.append(sum(G[i, i] for i in range(n)) / 2 + rg)
  r, rg = reg(sf2, mp.mpf(go.REG_CENTER_SIGNAL))
  loss += r
  grad.append(sum(G[i, j] * K[i, j] for i in range(n) for j in range(n)) / (2 * sf2) + rg)
  return loss, grad


@pytest.mark.parametrize('n,ls2,sn2', [(16, (100.0, 60.0), nc.SN2_CORNER[0]), (24, (30.0,), 1e-9)])
def test_closer_to_mpmath_than_fp64_by_100x(n, ls2, sn2):
  """cond(K_y) ~ 1e10-1e11 at a few dozen trials: in every component, and in the loss, the long-double result is at
  least 100 times closer to 40-digit mpmath than the fp64 oracle is."""
  mp = pytest.importorskip('mpmath').mp
  mp.dps = 40
  x, y, _ = nc.data(n, len(ls2), 0)
  theta = np.concatenate([ls2, [sn2, 2.0]])
  po = go.GPParams.from_vector(theta, len(ls2), 0)
  assert np.linalg.cond(go.kernel_matrix(po, x)) > 1e10
  want_l, want_g = _mp_loss_and_grad(mp, theta, x, y)
  got = hp.loss_and_grad_ld(theta, x, y)
  l64, g64 = go.loss_and_grad(theta, x, y)
  for k in range(len(want_g)):
    e_ld = abs(_to_mp(mp, got.grad[k]) - want_g[k])
    e_64 = abs(mp.mpf(float(g64[k])) - want_g[k])
    assert e_ld * 100 <= e_64, (k, float(e_ld), float(e_64))
  assert abs(_to_mp(mp, got.loss) - want_l) * 100 <= abs(mp.mpf(l64) - want_l)


def test_bound_rejects_a_factorisation_with_50_ulp_of_backward_error(monkeypatch):
  """N = 300 at eight points of the ill-conditioned corner.  The fp64 oracle run on the factor of K_y + E, E a
  symmetric random perturbation of 50 ulp of each entry (a backward error 50 times a single rounding of K_y), misses
  the bound the device routes are held to; the oracle itself meets it.  (A relative error of the same size in the
  entries of L is not such a defect: it moves K_y only along L's own columns, away from the small eigenvalues, and
  leaves the error within 1% even at 5e4 ulp.)"""
  n, dc = 300, 4
  x, y, _ = nc.data(n, dc, 0)
  thetas = nc.corner_points(dc, 0, 8)
  refs = [hp.loss_and_grad_ld(th, x, y) for th in thetas]

  def errors():
    out = [r.errors(*go.loss_and_grad(th, x, y)) for r, th in zip(refs, thetas)]
    return np.array([e for e, _ in out])[:, None], np.stack([g for _, g in out])

  loss64, grad64 = errors()
  assert nc.exercised(grad64)
  assert nc.within_bound(grad64, grad64) and nc.within_bound(loss64, loss64)
  rng = np.random.default_rng(5)

  def perturbed(a, jitter=1e-4, max_iters=5):
    u = rng.uniform(-1.0, 1.0, size=a.shape)
    u = np.triu(u) + np.triu(u, 1).T
    return np.linalg.cholesky(a + 50 * nc.EPS * np.abs(a) * u), 0.0, 0

  monkeypatch.setattr(go, 'retrying_cholesky', perturbed)
  loss_bad, grad_bad = errors()
  assert not nc.within_bound(grad_bad, grad64)
  assert not nc.within_bound(loss_bad, loss64)


def test_scales_of_the_linear_model_follow_its_terms():
  """The mean constant's gradient is -coef * sum alpha + mean: its scale is coef * sum |alpha|, and the regulariser
  parts of the linear components are their 0.5 x^2 and log-slope derivatives."""
  x, y, z, po = ff.case_inputs('well', 40, 3, 0, 1, 2e-3)
  po.linear = go.LinearParams(nc.LIN['coef'], nc.LIN['slope_amplitude'], nc.LIN['shift'], nc.LIN['mean_constant'])
  got = hp.loss_and_grad_ld(po.to_vector(), x, y, linear_coef=po.linear.coef)
  o = 3
  assert float(got.grad_scale[o + 2]) == pytest.approx(po.linear.coef * float(np.sum(np.abs(got.alpha))), rel=1e-15)
  assert float(got.grad_reg[o]) == po.linear.shift
  assert float(got.grad_reg[o + 2]) == po.linear.mean_constant
  slope = po.linear.slope_amplitude
  assert float(got.grad_reg[o + 1]) == pytest.approx(2 * go.REG_WEIGHT * math.log(slope / go.REG_CENTER_SIGNAL) / slope,
                                                      rel=1e-15)
