"""GPU parity: every C-ABI entry point against the oracle on the same seeded inputs.

Tolerances (fp64 path): 1e-10 absolute on well-conditioned hyper-parameters
(north-star bar).  The oracle is a restatement validated by mpmath/scipy, not a
live TFP run ("parity unpinned" at the TFP boundary, see oracle/gp_oracle.py).
Integer/index results (top-k indices, Philox draws, retry counts) are bit-exact.
"""
import numpy as np
import pytest
import scipy.linalg as sla

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from oracle import eagle_oracle as eo  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402

TOL = 1e-10


@pytest.fixture(scope='module')
def dev():
  if not torch.cuda.is_available():
    pytest.skip('no CUDA device')
  from vizier_b200 import gp
  d = gp.DeviceGP(0)
  yield d
  d.close()


def _gp():
  from vizier_b200 import gp
  return gp


def _problem(n, d, seed=0, dk=0):
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, d))
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  z = rng.integers(0, 4, size=(n, dk)).astype(np.int32) if dk else None
  return x, y, z


def _params(d, dk=0, sf2=1.0, sn2=1e-3, ls=None):
  ls2 = 0.5 * (1 + np.arange(d) / d) if ls is None else np.full(d, ls)
  lk = np.linspace(0.6, 1.4, dk) if dk else None
  return go.GPParams(sf2, ls2, sn2, lk), _gp().GPHyperParams(sf2, ls2, sn2, lk)


@pytest.mark.parametrize('n,d,dk', [(1, 1, 0), (50, 4, 0), (100, 5, 2), (200, 20, 0), (64, 3, 0)])
def test_kernel_matrix(dev, n, d, dk):
  x, _, z = _problem(n, d, 1, dk)
  po, pg = _params(d, dk)
  nv = max(1, n - 3)
  want = go.kernel_matrix(po, x, z, row_valid=np.arange(n) < nv)
  got = dev.kernel_matrix(x, pg, z=z, n_valid=nv, diag_add=po.observation_noise_variance).cpu().numpy()
  np.testing.assert_allclose(got, want, atol=1e-13, rtol=0)
  np.testing.assert_array_equal(got, got.T)


def test_cross_kernel(dev):
  x, _, z = _problem(130, 7, 2, 3)
  xs, _, zs = _problem(257, 7, 3, 3)
  po, pg = _params(7, 3)
  want = go.kernel(po, xs, x, zs, z)
  got = dev.cross_kernel(xs, x, pg, zs=zs, z=z).cpu().numpy()
  np.testing.assert_allclose(got, want, atol=1e-13, rtol=0)


@pytest.mark.parametrize('n', [1, 17, 64, 65, 200, 448])
def test_cholesky_and_inverse(dev, n):
  x, _, _ = _problem(n, 4, 4)
  po, _ = _params(4)
  a = go.kernel_matrix(po, x)
  l, shift, retries = dev.cholesky_retry(a)
  assert retries == 0 and shift == 0.0
  want = np.linalg.cholesky(a)
  np.testing.assert_allclose(l.cpu().numpy(), want, atol=1e-12, rtol=0)
  linv = dev.tri_inverse(want).cpu().numpy()
  np.testing.assert_allclose(linv, sla.solve_triangular(want, np.eye(n), lower=True), atol=1e-9, rtol=1e-9)
  assert np.all(np.triu(linv, 1) == 0)


def test_cholesky_retry_semantics(dev):
  # indefinite by 1e-6 -> one retry with shift 1e-4 (tuned_gp_models.py:272-280 semantics)
  a = np.array([[1.0, 1.0], [1.0, 1.0 - 1e-6]])
  l, shift, retries = dev.cholesky_retry(a)
  lo, so, ro = go.retrying_cholesky(a)
  assert retries == ro == 1 and shift == so == 1e-4
  np.testing.assert_allclose(l.cpu().numpy(), lo, atol=1e-14)
  a = np.array([[1.0, 1.9], [1.9, 1.0]])   # lambda_min = -0.9: first success at shift 1e-4 * 10^4
  l, shift, retries = dev.cholesky_retry(a)
  lo, so, ro = go.retrying_cholesky(a)
  assert retries == ro == 5 and shift == so == pytest.approx(1.0)
  np.testing.assert_allclose(l.cpu().numpy(), lo, atol=1e-14)
  # [[1,2],[2,1]] + 1.0*I is EXACTLY singular: a host potrf "succeeds" there only through the rounding
  # of 2/sqrt(2); the device pivot a - w*w/d is exactly 0 and is rejected (DESIGN.md, deviations).
  a = np.array([[1.0, 2.0], [2.0, 1.0]])
  l, shift, retries = dev.cholesky_retry(a)
  assert retries in (5, 6)
  a = np.array([[1.0, 5.0], [5.0, 1.0]])  # never succeeds within 5 retries
  l, shift, retries = dev.cholesky_retry(a)
  assert retries == 6 and np.isnan(l.cpu().numpy()).any()


@pytest.mark.parametrize('n,d,dk,nv', [(50, 4, 0, 50), (200, 6, 0, 200), (150, 5, 2, 140), (333, 20, 0, 333), (63, 3, 0, 63),
                                        (64, 4, 0, 64), (65, 4, 0, 65), (127, 5, 0, 64), (128, 5, 2, 65), (129, 6, 0, 1)])
def test_fit_factor_and_alpha(dev, n, d, dk, nv):
  x, y, z = _problem(n, d, 5, dk)
  po, pg = _params(d, dk)
  valid = np.arange(n) < nv
  pred = go.precompute_predictive(po, x, y, z, row_valid=valid)
  retries = dev.fit(x, y, pg, z=z, n_valid=nv)
  assert retries == 0
  np.testing.assert_allclose(dev.cholesky().cpu().numpy(), pred.chol, atol=1e-11, rtol=0)
  alpha = dev.alpha().cpu().numpy()
  np.testing.assert_allclose(alpha, pred.alpha, atol=1e-8 * np.max(np.abs(pred.alpha)), rtol=0)
  # residual of the solve is at round-off level (the property that matters for mu)
  ky = go.kernel_matrix(po, x, z, row_valid=valid)
  yv = np.where(valid, y, 0.0)
  assert np.max(np.abs(ky @ alpha - yv)) < 1e-11


@pytest.mark.parametrize('n,d,dk,m,tr', [(20, 3, 0, 100, True), (50, 4, 0, 513, True), (96, 5, 2, 300, True),
                                        (300, 20, 0, 1000, True), (300, 20, 0, 1000, False)])
def test_score_with_aux(dev, n, d, dk, m, tr):
  x, y, z = _problem(n, d, 6, dk)
  xs, _, zs = _problem(m, d, 7, dk)
  xs[:5] = x[:5]  # include observed points (sigma ~ sqrt(2*sn2), distance 0)
  if zs is not None:
    zs[:5] = z[:5]
  po, pg = _params(d, dk)
  pred = go.precompute_predictive(po, x, y, z)
  mask = np.ones(d, bool)
  if d > 2:
    mask[1] = False
  want, aux = go.score_with_aux(pred, xs, zs, tr_dim_mask=mask, categorical_dof=dk, use_trust_region=tr)
  radius = go.trust_radius(n, int(mask.sum()), dk)
  dev.fit(x, y, pg, z=z)
  acq = _gp().Acquisition(1.8, tr, radius, mask)
  out = dev.score(xs, acq, zs=zs, with_aux=True)
  dev.synchronize()
  mu_w, sd_w = go.predict(pred, xs, zs)
  np.testing.assert_allclose(out['mean'].cpu().numpy(), mu_w, atol=TOL, rtol=0)
  np.testing.assert_allclose(out['stddev'].cpu().numpy(), sd_w, atol=TOL, rtol=0)
  np.testing.assert_allclose(out['score'].cpu().numpy(), want, atol=TOL, rtol=0)
  dist = go.min_linf_distance(xs, x, mask)
  np.testing.assert_array_equal(out['linf_distance'].cpu().numpy(), dist)  # max/min of exact differences
  if tr and radius <= 0.5:
    assert np.any(want < -1e3)  # the trust region really was active in this case
  # score-only path (no aux outputs; features pre-divided by the length scale when the trust
  # region is inactive) agrees to round-off
  out2 = dev.score(xs, acq, zs=zs, with_aux=False)
  dev.synchronize()
  np.testing.assert_allclose(out2['score'].cpu().numpy(), out['score'].cpu().numpy(), atol=1e-12, rtol=0)


def test_score_hard_conditioning_scaled_tolerance(dev):
  # sn2=1e-8, ls2=0.05: cond(K_y) ~ 1e10; both sides lose digits ~ eps*cond(L)*|v|.
  n, d, m = 200, 6, 400
  x, y, _ = _problem(n, d, 8)
  xs, _, _ = _problem(m, d, 9)
  po, pg = _params(d, sn2=1e-8, ls=0.05)
  pred = go.precompute_predictive(po, x, y)
  dev.fit(x, y, pg)
  out = dev.score(xs, _gp().Acquisition(1.8, False, 1.0), with_aux=True)
  dev.synchronize()
  mu_w, sd_w = go.predict(pred, xs)
  np.testing.assert_allclose(out['mean'].cpu().numpy(), mu_w, atol=1e-7, rtol=0)
  np.testing.assert_allclose(out['stddev'].cpu().numpy(), sd_w, atol=1e-7, rtol=0)


@pytest.mark.parametrize('n,d,dk,nv', [(40, 3, 0, 40), (130, 6, 2, 120), (256, 20, 0, 256), (65, 4, 0, 64), (127, 5, 0, 127),
                                        (128, 5, 1, 65), (129, 6, 2, 1), (129, 3, 0, 129)])
def test_nll_grad(dev, n, d, dk, nv):
  x, y, z = _problem(n, d, 10, dk)
  po, pg = _params(d, dk, sf2=0.7, sn2=2e-3)
  valid = np.arange(n) < nv
  want_l, want_g = go.loss_and_grad(po.to_vector(), x, y, z, valid)
  xt = torch.from_numpy(x).cuda(); yt = torch.from_numpy(y).cuda()
  zt = torch.from_numpy(z).cuda() if z is not None else None
  loss, grad, retries = dev.loss_and_grad(xt, yt, pg, z=zt, n_valid=nv)
  assert retries == 0
  assert abs(loss - want_l) < 1e-9 * max(1.0, abs(want_l))
  np.testing.assert_allclose(grad, want_g, atol=1e-8 * max(1.0, np.max(np.abs(want_g))), rtol=0)


@pytest.mark.parametrize('n,d,dk,nv', [(1, 1, 0, 1), (7, 2, 1, 7), (50, 4, 0, 50), (64, 20, 3, 64), (64, 64, 0, 57), (33, 5, 2, 20),
                                        (63, 3, 0, 63), (64, 4, 1, 1)])
def test_nll_grad_small_fused_kernel(dev, n, d, dk, nv):
  """N <= 64 takes the single-launch kernel (k_nll_grad_small): same oracle, same tolerances, and the
  make_loss_fn closure the ARD driver uses returns the same numbers; the fitted model is untouched."""
  x, y, z = _problem(n, d, 17, dk)
  po, pg = _params(d, dk, sf2=0.7, sn2=2e-3)
  valid = np.arange(n) < nv
  want_l, want_g = go.loss_and_grad(po.to_vector(), x, y, z, valid)
  xt = torch.from_numpy(x).cuda(); yt = torch.from_numpy(y).cuda()
  zt = torch.from_numpy(z).cuda() if z is not None else None
  dev.fit(x[:nv], y[:nv], pg, z=None if z is None else z[:nv])
  alpha_before = dev.alpha().cpu().numpy()
  l0 = dev.launch_count
  loss, grad, retries = dev.loss_and_grad(xt, yt, pg, z=zt, n_valid=nv)
  assert dev.launch_count - l0 == 1
  assert retries == 0
  assert abs(loss - want_l) < 1e-9 * max(1.0, abs(want_l))
  np.testing.assert_allclose(grad, want_g, atol=1e-8 * max(1.0, np.max(np.abs(want_g))), rtol=0)
  f = dev.make_loss_fn(xt, yt, zt, n_valid=nv)
  l2, g2 = f(pg.to_vector())
  assert l2 == loss
  np.testing.assert_array_equal(g2, grad)
  np.testing.assert_array_equal(dev.alpha().cpu().numpy(), alpha_before)


def test_nll_grad_small_near_singular(dev):
  """Triplicated points at the noise floor (cond ~ 1e10): the in-kernel factorisation + retry loop
  reports the oracle's retry count and loss (tuned_gp_models.py:272-280)."""
  rng = np.random.default_rng(19)
  x = rng.uniform(size=(12, 3)); x[5] = x[2]; x[9] = x[2]
  y = rng.normal(size=12)
  po = go.GPParams(1.0, np.full(3, 0.5), 1e-10); pg = _gp().GPHyperParams(1.0, np.full(3, 0.5), 1e-10)
  ky = go.kernel_matrix(po, x)
  _, shift, want_retries = go.retrying_cholesky(ky)
  want_l, want_g = go.loss_and_grad(po.to_vector(), x, y)
  loss, grad, retries = dev.loss_and_grad(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), pg)
  assert retries == want_retries
  if np.isfinite(want_l):
    assert abs(loss - want_l) < 1e-6 * max(1.0, abs(want_l))


def test_nll_graph_survives_workspace_growth():
  """The replayed NLL graph points into the handle's workspaces: a later, larger fit reallocates them and
  the graph must be rebuilt, not replayed (same tensors, same shape -> same cache key)."""
  gp = _gp()
  d = gp.DeviceGP(0)
  x, y, _ = _problem(130, 5, 23)
  po, pg = _params(5, sf2=0.7, sn2=2e-3)
  want_l, want_g = go.loss_and_grad(po.to_vector(), x, y)
  xt = torch.from_numpy(x).cuda(); yt = torch.from_numpy(y).cuda()
  f = d.make_loss_fn(xt, yt)
  for _ in range(3):                      # capture + two replays
    l1, g1 = f(pg.to_vector())
  xb, yb, _ = _problem(700, 5, 24)
  d.fit(xb, yb, pg)                       # grows every N x N workspace
  l2, g2 = f(pg.to_vector())
  assert l1 == l2
  np.testing.assert_array_equal(g1, g2)
  assert abs(l2 - want_l) < 1e-9 * max(1.0, abs(want_l))
  np.testing.assert_allclose(g2, want_g, atol=1e-8 * max(1.0, np.max(np.abs(want_g))), rtol=0)
  # and new hyper-parameters through the same graph
  po2, pg2 = _params(5, sf2=1.3, sn2=5e-2)
  w2, wg2 = go.loss_and_grad(po2.to_vector(), x, y)
  l3, g3 = f(pg2.to_vector())
  assert abs(l3 - w2) < 1e-9 * max(1.0, abs(w2))
  np.testing.assert_allclose(g3, wg2, atol=1e-8 * max(1.0, np.max(np.abs(wg2))), rtol=0)


def test_topk_ties_nan_and_order(dev):
  rng = np.random.default_rng(11)
  s = rng.normal(size=5000)
  s[[10, 4000, 77]] = s.max() + 1.0  # three-way tie for the top
  s[5] = np.nan
  s[6] = -np.inf
  idx, val = dev.topk(torch.from_numpy(s).cuda(), 7)
  want = go.top_k(np.where(np.isnan(s), -np.inf, s), 7)
  np.testing.assert_array_equal(idx, want)
  np.testing.assert_array_equal(val, s[want])
  idx, _ = dev.topk(torch.from_numpy(np.array([3.0, 1.0])).cuda(), 2)
  np.testing.assert_array_equal(idx, [0, 1])


def test_random_pool_matches_philox_oracle(dev):
  got = dev.random_pool(1000, 7, seed=0x1234ABCD5678, index_base=5).cpu().numpy()
  want = eo.philox_uniform(0x1234ABCD5678, eo.STREAM_RANDOM_POOL, 0, 1005 * 7).reshape(1005, 7)[5:]
  np.testing.assert_array_equal(got, want)


def test_random_search_matches_oracle(dev):
  n, d, m = 120, 6, 5000
  x, y, _ = _problem(n, d, 12)
  po, pg = _params(d)
  pred = go.precompute_predictive(po, x, y)
  dev.fit(x, y, pg)
  radius = go.trust_radius(n, d, 0)
  bx, _, bs, bi = dev.random_search(m, _gp().Acquisition(1.8, True, radius), count=3, seed=99)
  wx, ws, wi = eo.run_random_optimizer(lambda q: go.score_with_aux(pred, q)[0], dim=d, num_candidates=m, count=3, seed=99)
  np.testing.assert_array_equal(bi, wi)
  np.testing.assert_array_equal(bx, wx)
  np.testing.assert_allclose(bs, ws, atol=TOL)


# The last two rows are BASELINE C3's shape (P = B = 1000 fireflies, N = 1000 trials, D = 20) and a
# batch-600 case: batches above 512 take the replayed CUDA-graph form of the loop (c_abi.cu,
# eagle_run_impl) with k_eagle_suggest / k_eagle_update at 1000 flies and the large-pool k_score.
@pytest.mark.parametrize('n,d,pool,batch,steps', [(30, 4, 25, 25, 6), (60, 5, 20, 5, 14), (130, 3, 50, 25, 7),
                                                  (1000, 20, 1000, 1000, 6), (700, 12, 1200, 600, 7)])
def test_eagle_run_matches_oracle(dev, n, d, pool, batch, steps):
  x, y, _ = _problem(n, d, 13)
  po, pg = _params(d)
  pred = go.precompute_predictive(po, x, y)
  dev.fit(x, y, pg)
  radius = go.trust_radius(n, d, 0)
  score_fn = lambda q: go.score_with_aux(pred, q)[0]
  cfg_o = eo.EagleConfig()
  wx, wr, st = eo.run_eagle_optimizer(score_fn, dim=d, pool_size=pool, batch_size=batch,
                                      max_evaluations=steps * batch, count=3, seed=7, cfg=cfg_o, prior_features=x)
  from vizier_b200 import _lib
  cfg = _lib.EagleConfig(cfg_o.visibility, cfg_o.gravity, cfg_o.negative_gravity, cfg_o.perturbation,
                         cfg_o.perturbation_lower_bound, cfg_o.penalize_factor, cfg_o.normalization_scale,
                         cfg_o.prior_trials_pool_pct, pool, batch, steps * batch)
  bx, _, br = dev.eagle_run(cfg, _gp().Acquisition(1.8, True, radius), count=3, seed=7, prior=x)
  np.testing.assert_allclose(br, wr, atol=1e-9)
  np.testing.assert_allclose(bx, wx, atol=1e-9)


@pytest.mark.parametrize('n,d,m,members,tr', [(90, 5, 700, 2, True), (40, 3, 64, 3, True), (300, 8, 5000, 2, False)])
def test_ensemble_score_matches_oracle(n, d, m, members, tr):
  """Uniform mixture of E GPs (stochastic_process_model.py:846-868) through vzgp_score_ensemble:
  mean = avg mu_e, var = avg(sd_e^2 + mu_e^2) - mean^2, UCB + trust region on top."""
  gp = _gp()
  x, y, _ = _problem(n, d, 71)
  xs, _, _ = _problem(m, d, 72)
  rng = np.random.default_rng(73)
  plist_o, plist_g = [], []
  for _ in range(members):
    ls2 = np.exp(rng.uniform(np.log(0.05), np.log(5.0), d))
    sf2, sn2 = float(np.exp(rng.uniform(-2, 1))), float(np.exp(rng.uniform(-8, -2)))
    plist_o.append(go.GPParams(sf2, ls2, sn2))
    plist_g.append(gp.GPHyperParams(sf2, ls2, sn2))
  preds = [go.precompute_predictive(p, x, y) for p in plist_o]
  ens = gp.EnsembleGP(0, members)
  ens.fit(x, y, plist_g)
  radius = 0.3 if tr else go.trust_radius(n, d, 0)
  acq = gp.Acquisition(1.8, True, radius)
  mu, sd = go.predict_ensemble(preds, xs)
  dist = go.min_linf_distance(xs, x, np.ones(d, bool), np.ones(n, bool))
  want = go.apply_trust_region(go.ucb(mu, sd, 1.8), dist, radius)
  out = ens.score(xs, acq, with_aux=True)
  ens.synchronize()
  np.testing.assert_allclose(out['mean'].cpu().numpy(), mu, atol=TOL, rtol=0)
  np.testing.assert_allclose(out['stddev'].cpu().numpy(), sd, atol=TOL, rtol=0)
  np.testing.assert_allclose(out['score'].cpu().numpy(), want, atol=TOL, rtol=0)
  out2 = ens.score(xs, acq)
  ens.synchronize()
  np.testing.assert_allclose(out2['score'].cpu().numpy(), want, atol=TOL, rtol=0)
  # one-member "ensemble" == the plain model
  single = gp.EnsembleGP(0, 1)
  single.fit(x, y, plist_g[:1])
  o1 = single.score(xs, acq)
  single.synchronize()
  w1 = go.apply_trust_region(go.ucb(*go.predict(preds[0], xs), 1.8), dist, radius)
  np.testing.assert_allclose(o1['score'].cpu().numpy(), w1, atol=TOL, rtol=0)


def test_ensemble_eagle_and_random_search_match_oracle():
  gp = _gp()
  n, d, pool, batch, steps = 50, 4, 25, 25, 6
  x, y, _ = _problem(n, d, 81)
  plist_o = [go.GPParams(1.0, np.full(d, 0.4), 1e-3), go.GPParams(0.5, np.linspace(0.2, 2.0, d), 1e-2)]
  plist_g = [gp.GPHyperParams(p.signal_variance, p.continuous_length_scale_squared, p.observation_noise_variance) for p in plist_o]
  preds = [go.precompute_predictive(p, x, y) for p in plist_o]
  ens = gp.EnsembleGP(0, 2)
  ens.fit(x, y, plist_g)
  radius = go.trust_radius(n, d, 0)

  def score_fn(q):
    mu, sd = go.predict_ensemble(preds, q)
    dist = go.min_linf_distance(q, x, np.ones(d, bool), np.ones(n, bool))
    return go.apply_trust_region(go.ucb(mu, sd, 1.8), dist, radius)

  cfg_o = eo.EagleConfig()
  wx, wr, _ = eo.run_eagle_optimizer(score_fn, dim=d, pool_size=pool, batch_size=batch,
                                     max_evaluations=steps * batch, count=3, seed=7, cfg=cfg_o, prior_features=x)
  from vizier_b200 import _lib
  cfg = _lib.EagleConfig(cfg_o.visibility, cfg_o.gravity, cfg_o.negative_gravity, cfg_o.perturbation,
                         cfg_o.perturbation_lower_bound, cfg_o.penalize_factor, cfg_o.normalization_scale,
                         cfg_o.prior_trials_pool_pct, pool, batch, steps * batch)
  acq = gp.Acquisition(1.8, True, radius)
  bx, _, br = ens.eagle_run(cfg, acq, count=3, seed=7, prior=x)
  np.testing.assert_allclose(br, wr, atol=1e-9)
  np.testing.assert_allclose(bx, wx, atol=1e-9)
  wx, ws, wi = eo.run_random_optimizer(score_fn, dim=d, num_candidates=2000, count=3, seed=99)
  rx, _, rs, ri = ens.random_search(2000, acq, 3, seed=99)
  np.testing.assert_array_equal(ri, wi)
  np.testing.assert_allclose(rx, wx, atol=0)
  np.testing.assert_allclose(rs, ws, atol=TOL)


def test_c2_full_size_properties(dev):
  """BASELINE C2 (N=1000, D=20, M=100k): spot parity on a sample + size-independent properties."""
  n, d, m = 1000, 20, 100_000
  x, y, _ = _problem(n, d, 0)
  po, pg = _params(d)
  dev.fit(x, y, pg)
  xs = dev.random_pool(m, d, seed=2024)
  acq = _gp().Acquisition(1.8, True, go.trust_radius(n, d, 0))
  out = dev.score(xs, acq, with_aux=True)
  dev.synchronize()
  sc = out['score'].cpu().numpy()
  assert np.all(np.isfinite(sc)) and dev.clamped_count() == 0
  # (1) sample parity against the oracle
  pred = go.precompute_predictive(po, x, y)
  sel = np.random.default_rng(1).choice(m, 512, replace=False)
  want, _ = go.score_with_aux(pred, xs[torch.from_numpy(sel).cuda()].cpu().numpy())
  np.testing.assert_allclose(sc[sel], want, atol=TOL, rtol=0)
  # (2) position independence: the same candidates scored alone (small-pool path: column blocks
  # split across CTAs, row sums reduced in a different fixed order) agree to round-off, and
  # repeated evaluation is bit-reproducible
  sub = xs[torch.from_numpy(sel).cuda()].contiguous()
  out2 = dev.score(sub, acq)
  dev.synchronize()
  np.testing.assert_allclose(out2['score'].cpu().numpy(), sc[sel], atol=1e-12, rtol=0)
  out3 = dev.score(xs, acq, with_aux=True)
  dev.synchronize()
  np.testing.assert_array_equal(out3['score'].cpu().numpy(), sc)
  out4, out5 = dev.score(xs, acq), None
  dev.synchronize()
  first = out4['score'].cpu().numpy().copy()
  out5 = dev.score(xs, acq)
  dev.synchronize()
  np.testing.assert_array_equal(out5['score'].cpu().numpy(), first)
  np.testing.assert_allclose(first, sc, atol=1e-12, rtol=0)  # scaled-feature path vs difference-first path
  # (3) posterior sanity: 0 <= var <= sf2 + sn2, and UCB identity
  sd = out['stddev'].cpu().numpy(); mu = out['mean'].cpu().numpy()
  assert sd.min() >= 0 and sd.max() <= np.sqrt(1.0 + 1e-3) + 1e-12
  np.testing.assert_allclose(sc, mu + 1.8 * sd, atol=1e-12)
  # (4) top-k agrees with a host sort
  idx, val = dev.topk(out['score'], 5)
  np.testing.assert_array_equal(idx, go.top_k(sc, 5))


def test_c2_full_pool_parity(dev):
  """BASELINE C2, every one of the 100k candidates against the oracle (~30 s of CPU)."""
  n, d, m = 1000, 20, 100_000
  x, y, _ = _problem(n, d, 0)
  po, pg = _params(d)
  dev.fit(x, y, pg)
  xs = dev.random_pool(m, d, seed=77)
  out = dev.score(xs, _gp().Acquisition(1.8, True, go.trust_radius(n, d, 0)), with_aux=True)
  dev.synchronize()
  pred = go.precompute_predictive(po, x, y)
  want, aux = go.score_with_aux(pred, xs.cpu().numpy())
  np.testing.assert_allclose(out['score'].cpu().numpy(), want, atol=TOL, rtol=0)
  np.testing.assert_allclose(out['mean'].cpu().numpy(), aux['mean'], atol=TOL, rtol=0)
  np.testing.assert_allclose(out['stddev'].cpu().numpy(), aux['stddev'], atol=TOL, rtol=0)
  np.testing.assert_array_equal(out['linf_distance'].cpu().numpy(), aux['linf_distance'])
  # the throughput variant (no aux, pre-scaled features) on the same pool
  fast = dev.score(xs, _gp().Acquisition(1.8, True, go.trust_radius(n, d, 0)))
  dev.synchronize()
  np.testing.assert_allclose(fast['score'].cpu().numpy(), want, atol=TOL, rtol=0)
  np.testing.assert_array_equal(dev.topk(fast['score'], 8)[0], go.top_k(want, 8))


def test_ard_fit_matches_oracle_driver(dev):
  """Same inits + same SciPy L-BFGS-B driver: CUDA loss/grad vs oracle loss/grad (SURVEY A.4:
  compare fits by final loss, trajectories are not bit-reproducible across gradient implementations)."""
  from vizier_b200 import ard
  n, d = 60, 4
  x, y, _ = _problem(n, d, 21)
  y = (y - y.mean()) / y.std()
  inits = ard.log_uniform_init(np.random.default_rng(5), d, 0, 4)
  want_theta, want_losses = go.ard_fit(x, y, init_thetas=inits)
  xt = torch.from_numpy(x).cuda(); yt = torch.from_numpy(y).cuda()
  lo, hi = _gp().param_bounds(d, 0)

  def f(theta):
    loss, grad, _ = dev.loss_and_grad(xt, yt, _gp().GPHyperParams.from_vector(theta, d, 0))
    return loss, grad

  best, losses = ard.ScipyLbfgsB()(inits, f, list(zip(lo, hi)), best_n=1)
  # Individual restarts may stop in different places (L-BFGS-B amplifies 1e-10 gradient
  # differences over 50 iterations); what the designer uses is the best loss.
  assert abs(losses.min() - want_losses.min()) < 1e-6
  assert np.all(losses > want_losses.min() - 1e-6)
  # and the returned optimum is a stationary point of the ORACLE loss too
  l_o, g_o = go.loss_and_grad(best[0], x, y)
  assert abs(l_o - losses.min()) < 1e-8


def test_batched_ard_equals_threaded_ard():
  """The lock-step ARD (one graph launch evaluates all restarts, vzgp_nll_grad_batch) and the round-1 form
  (one host thread and one graph per restart) run the same optimisations: identical final losses and
  hyper-parameters; with categorical features and masked rows too."""
  from vizier_b200 import ard
  gp = _gp()
  for n, d, dk, nv in ((150, 4, 0, 150), (260, 6, 2, 250)):
    x, y, z = _problem(n, d, 31, dk)
    res = {}
    for batched in (True, False):
      ard.BATCHED_ARD = batched
      try:
        dev = gp.DeviceGP(0)
        best, losses = ard.train_gp(dev, x, y, z, rng=np.random.default_rng(5), random_restarts=5, ensemble_size=2,
                                    n_valid=nv)
        res[batched] = (np.stack([b.to_vector() for b in best]), losses)
      finally:
        ard.BATCHED_ARD = True
    np.testing.assert_array_equal(res[True][1], res[False][1])
    np.testing.assert_array_equal(res[True][0], res[False][0])


def test_posterior_covariance(dev):
  n, d, m = 150, 5, 70
  x, y, _ = _problem(n, d, 22)
  xs, _, _ = _problem(m, d, 23)
  po, pg = _params(d)
  pred = go.precompute_predictive(po, x, y)
  dev.fit(x, y, pg)
  mean, cov = dev.posterior(xs)
  ks = go.kernel(po, xs, x)
  v = sla.solve_triangular(pred.chol, ks.T, lower=True)
  want_cov = go.kernel(po, xs, xs) - v.T @ v + po.observation_noise_variance * np.eye(m)
  np.testing.assert_allclose(cov.cpu().numpy(), want_cov, atol=TOL, rtol=0)
  np.testing.assert_allclose(mean.cpu().numpy(), ks @ pred.alpha, atol=TOL, rtol=0)


def test_score_topk_fused_call(dev):
  n, d, m = 120, 6, 3000
  x, y, _ = _problem(n, d, 31)
  xs, _, _ = _problem(m, d, 32)
  po, pg = _params(d)
  pred = go.precompute_predictive(po, x, y)
  dev.fit(x, y, pg)
  acq = _gp().Acquisition(1.8, True, go.trust_radius(n, d, 0))
  xt = torch.from_numpy(xs).cuda()
  buf = torch.empty(m, dtype=torch.float64, device='cuda')
  bx, bs, bi = dev.score_topk(xt, acq, 4, score_out=buf)
  want, _ = go.score_with_aux(pred, xs)
  order = go.top_k(want, 4)
  np.testing.assert_array_equal(bi, order)
  np.testing.assert_array_equal(bx, xs[order])
  np.testing.assert_allclose(bs, want[order], atol=TOL)
  np.testing.assert_allclose(buf.cpu().numpy(), want, atol=TOL)


def test_score_topk_pack_and_device_merge(dev):
  """The asynchronous shard step (pack rows [score, global index, x]) and the device merge agree with
  the oracle's top-k and with the host merge used by the gloo test (multi_gpu.merge_topk)."""
  from vizier_b200 import multi_gpu
  n, d, m, count = 120, 6, 3000, 4
  x, y, _ = _problem(n, d, 31)
  xs, _, _ = _problem(m, d, 32)
  po, pg = _params(d)
  pred = go.precompute_predictive(po, x, y)
  dev.fit(x, y, pg)
  acq = _gp().Acquisition(1.8, True, go.trust_radius(n, d, 0))
  xt = torch.from_numpy(xs).cuda()
  payload = torch.empty((count, d + 2), dtype=torch.float64, device='cuda')
  base = 7_000_000_000   # > 2^32: global indices of a large sharded pool
  dev.score_topk_pack(xt, acq, count, base, payload)
  dev.synchronize()
  want, _ = go.score_with_aux(pred, xs)
  order = go.top_k(want, count)
  p = payload.cpu().numpy()
  np.testing.assert_array_equal(p[:, 1].astype(np.int64), order + base)
  np.testing.assert_array_equal(p[:, 2:], xs[order])
  np.testing.assert_allclose(p[:, 0], want[order], atol=TOL)
  # merge of "gathered" rows from 3 pretend ranks, with ties, NaN and missing (-1) winners
  rng = np.random.default_rng(5)
  rows = np.zeros((3 * count, d + 2))
  rows[:, 0] = rng.normal(size=3 * count)
  rows[:, 1] = rng.permutation(3 * count) + 100
  rows[:, 2:] = rng.uniform(size=(3 * count, d))
  rows[5, 0] = rows[2, 0]                 # tie -> lower global index wins
  rows[7, 0] = np.nan                     # NaN ranks as -inf
  rows[9, :2] = [-np.inf, -1.0]           # rank with fewer than `count` candidates
  rt = torch.from_numpy(rows).cuda()
  out = torch.empty((count, d + 2), dtype=torch.float64, device='cuda')
  host = torch.empty((count, d + 2), dtype=torch.float64).pin_memory()
  dev.merge_topk(rt, count, out, host)
  dev.synchronize()
  valid = rows[:, 1] >= 0
  wi, wv, wx = multi_gpu.merge_topk(rows[valid, 1].astype(np.int64), rows[valid, 0], rows[valid, 2:], count)
  np.testing.assert_array_equal(host.numpy()[:, 1].astype(np.int64), wi)
  np.testing.assert_array_equal(host.numpy()[:, 2:], wx)
  np.testing.assert_array_equal(out.cpu().numpy(), host.numpy())
  # world-size-1 exchange object (what bench.py drives): pack -> merge -> pinned host
  ex = multi_gpu.TopkExchange(None, dev, d, count)
  ex.step(1, xt, acq, index_base=base)
  gi, gv, gx = ex.result(1)
  np.testing.assert_array_equal(gi, order + base)
  np.testing.assert_array_equal(gx, xs[order])


@pytest.mark.parametrize('n,d,m', [(1, 1, 1), (2, 3, 63), (64, 2, 65), (65, 7, 129), (127, 64, 40), (129, 33, 200)])
def test_score_edge_shapes(dev, n, d, m):
  """Ragged sizes around the 64-row tiles / 128-column blocks, D=1 and the D=64 maximum.  These pools have at
  most 4 tiles: by default they take the small-pool kernels; with "small_tiles" = 0 the same pool runs k_score."""
  x, y, _ = _problem(n, d, 41)
  xs, _, _ = _problem(m, d, 42)
  po, pg = _params(d)
  pred = go.precompute_predictive(po, x, y)
  dev.fit(x, y, pg)
  acq = _gp().Acquisition(1.8, True, go.trust_radius(n, d, 0))
  want, aux = go.score_with_aux(pred, xs)
  for small_tiles, small_route in ((-1, True), (0, False)):
    dev.set_int('small_tiles', small_tiles)
    try:
      out = dev.score(xs, acq, with_aux=True)
      route = dev.get_int('score_route')
      out2 = dev.score(xs, acq)
      dev.synchronize()
    finally:
      dev.set_int('small_tiles', -1)
    assert (route == 0) == small_route, route
    np.testing.assert_allclose(out['score'].cpu().numpy(), want, atol=TOL, rtol=0)
    np.testing.assert_allclose(out['stddev'].cpu().numpy(), aux['stddev'], atol=TOL, rtol=0)
    np.testing.assert_allclose(out2['score'].cpu().numpy(), want, atol=TOL, rtol=0)


@pytest.mark.parametrize('n,d,m,radius', [(1000, 20, 25, None), (1000, 20, 512, 0.25), (960, 8, 64, 0.1),
                                          (1500, 12, 130, None)])
def test_score_small_pool_path(dev, n, d, m, radius):
  """Acquisition-optimiser batch sizes (<= 8 tiles) take the trial-axis kernels (k_cross_small /
  k_var_small / k_small_finalize): same oracle, with and without an ACTIVE trust region, and the
  same bits run to run (fixed-order reductions)."""
  x, y, _ = _problem(n, d, 61)
  xs, _, _ = _problem(m, d, 62)
  rng = np.random.default_rng(63)
  near = np.arange(0, m, 2)   # every other candidate sits next to a trial (inside a small trust radius)
  xs[near] = np.clip(x[rng.integers(0, n, near.size)] + rng.uniform(-0.05, 0.05, (near.size, d)), 0.0, 1.0)
  po, pg = _params(d)
  pred = go.precompute_predictive(po, x, y)
  dev.fit(x, y, pg)
  r = go.trust_radius(n, d, 0) if radius is None else radius
  acq = _gp().Acquisition(1.8, True, r)
  mu, sd = go.predict(pred, xs)
  dist = go.min_linf_distance(xs, pred.x, np.ones(d, bool), pred.row_valid)
  want = go.apply_trust_region(go.ucb(mu, sd, 1.8), dist, r)
  aux = {'mean': mu, 'stddev': sd, 'linf_distance': dist}
  out = dev.score(xs, acq, with_aux=True)
  dev.synchronize()
  got = {k: out[k].cpu().numpy().copy() for k in ('score', 'mean', 'stddev', 'linf_distance')}
  np.testing.assert_allclose(got['score'], want, atol=TOL, rtol=0)
  np.testing.assert_allclose(got['mean'], aux['mean'], atol=TOL, rtol=0)
  np.testing.assert_allclose(got['stddev'], aux['stddev'], atol=TOL, rtol=0)
  np.testing.assert_allclose(got['linf_distance'], aux['linf_distance'], atol=1e-15, rtol=0)
  if radius is not None:
    assert (want < -1e3).any() and (want > -1e3).any()   # both sides of the trust region are exercised
  out2 = dev.score(xs, acq, with_aux=True)
  dev.synchronize()
  for k in got:
    np.testing.assert_array_equal(out2[k].cpu().numpy(), got[k])
  out3 = dev.score(xs, acq)
  dev.synchronize()
  np.testing.assert_allclose(out3['score'].cpu().numpy(), want, atol=TOL, rtol=0)


def test_c5_shape_sample_parity(dev):
  """BASELINE C5 per-GPU shape (N=2000, D=50): 20k candidates, 256-sample parity + fit residual."""
  n, d, m = 2000, 50, 20_000
  rng = np.random.default_rng(5)
  x = rng.uniform(size=(n, d)); y = rng.normal(size=n)
  ls2 = np.full(d, 2.0)
  po = go.GPParams(1.0, ls2, 1e-2); pg = _gp().GPHyperParams(1.0, ls2, 1e-2)
  assert dev.fit(x, y, pg) == 0
  xs = dev.random_pool(m, d, seed=77)
  acq = _gp().Acquisition(1.8, True, go.trust_radius(n, d, 0))
  out = dev.score(xs, acq)
  dev.synchronize()
  sc = out['score'].cpu().numpy()
  pred = go.precompute_predictive(po, x, y)
  sel = np.random.default_rng(2).choice(m, 256, replace=False)
  want, _ = go.score_with_aux(pred, xs[torch.from_numpy(sel).cuda()].cpu().numpy())
  np.testing.assert_allclose(sc[sel], want, atol=TOL, rtol=0)
  idx, _ = dev.topk(out['score'], 3)
  np.testing.assert_array_equal(idx, go.top_k(sc, 3))


def test_error_behaviour(dev):
  """Status codes and messages instead of exceptions/crashes (SURVEY 8b: C ABI never throws)."""
  from vizier_b200 import _lib, gp
  fresh = gp.DeviceGP(0)
  xs = torch.zeros((4, 3), dtype=torch.float64, device='cuda')
  with pytest.raises(_lib.VzgpError) as e:
    fresh.score(xs, gp.Acquisition())
  assert e.value.status == _lib.VZGP_ERR_STATE and 'before vzgp_fit' in str(e.value)
  with pytest.raises(_lib.VzgpError) as e:
    fresh.fit(np.zeros((3, 65)), np.zeros(3), gp.GPHyperParams(1.0, np.ones(65), 1e-3))
  assert e.value.status == _lib.VZGP_ERR_ARG and 'Dc out of range' in str(e.value)
  with pytest.raises(_lib.VzgpError):
    fresh.fit(np.zeros((3, 2)), np.zeros(3), gp.GPHyperParams(1.0, np.ones(2), 1e-3), n_valid=0)
  # a NaN in the labels does not crash: the factor is fine, alpha carries the NaN
  x, y, _ = _problem(10, 2, 3)
  fresh.fit(x, y, gp.GPHyperParams(1.0, np.ones(2), 1e-3))
  out = fresh.score(np.zeros((0, 2)), gp.Acquisition())  # empty pool is a no-op
  assert out['score'].numel() == 0
  idx, val = fresh.topk(torch.tensor([1.0, 2.0], dtype=torch.float64, device='cuda'), 4)  # count > M
  assert idx.tolist() == [1, 0, -1, -1]
  fresh.close()


@pytest.mark.parametrize('n,d,sizes,pool,batch,steps', [(40, 3, (2, 4), 20, 5, 16), (70, 0, (3, 5, 2), 25, 25, 6), (90, 2, (7,), 50, 25, 9)])
def test_eagle_mixed_features_matches_oracle(dev, n, d, sizes, pool, batch, steps):
  """Continuous + categorical (and purely categorical) eagle trajectories against the oracle with the
  shared Philox draws (laplace / gumbel-max categorical mutation, eagle_strategy.py:936-1011)."""
  rng = np.random.default_rng(51)
  sizes = np.asarray(sizes)
  dk = sizes.shape[0]
  x = rng.uniform(size=(n, d))
  z = np.stack([rng.integers(0, s, size=n) for s in sizes], axis=1).astype(np.int32)
  y = -np.sum((x - 0.3) ** 2, axis=1) - 0.3 * (z[:, 0] != 1) + 0.05 * rng.normal(size=n)
  po, pg = _params(d, dk)
  pred = go.precompute_predictive(po, x, y, z)
  dev.fit(x, y, pg, z=z)
  mask = np.ones(d, bool)
  radius = go.trust_radius(n, d, dk)
  score_fn = lambda xc, xz: go.score_with_aux(pred, xc, xz, tr_dim_mask=mask, categorical_dof=dk)[0]
  cfg_o = eo.EagleConfig()
  wc, wz, wr = eo.run_eagle_optimizer_mixed(score_fn, dim=d, sizes=sizes, pool_size=pool, batch_size=batch,
                                            max_evaluations=steps * batch, count=3, seed=11, cfg=cfg_o, prior_c=x, prior_z=z)
  from vizier_b200 import _lib
  cfg = _lib.EagleConfig(cfg_o.visibility, cfg_o.gravity, cfg_o.negative_gravity, cfg_o.perturbation,
                         cfg_o.perturbation_lower_bound, cfg_o.penalize_factor, cfg_o.normalization_scale,
                         cfg_o.prior_trials_pool_pct, pool, batch, steps * batch)
  bx, bz, br = dev.eagle_run(cfg, _gp().Acquisition(1.8, True, radius, mask), count=3, seed=11, prior=x, prior_z=z, cat_sizes=sizes)
  np.testing.assert_array_equal(bz, wz)
  np.testing.assert_allclose(br, wr, atol=1e-9)
  np.testing.assert_allclose(bx, wc, atol=1e-9)


def test_random_search_with_categoricals(dev):
  rng = np.random.default_rng(52)
  n, d, sizes, m = 80, 3, np.array([3, 6]), 4000
  x = rng.uniform(size=(n, d)); z = np.stack([rng.integers(0, s, size=n) for s in sizes], axis=1).astype(np.int32)
  y = rng.normal(size=n)
  po, pg = _params(d, 2)
  pred = go.precompute_predictive(po, x, y, z)
  dev.fit(x, y, pg, z=z)
  acq = _gp().Acquisition(1.8, True, go.trust_radius(n, d, 2))
  bx, bz, bs, bi = dev.random_search(m, acq, 2, seed=5, cat_sizes=sizes)
  xc = eo.philox_uniform(5, eo.STREAM_RANDOM_POOL, 0, m * d).reshape(m, d)
  xz = eo.uniform_categories(eo.philox_uniform(5, eo.STREAM_RANDOM_POOL_CAT, 0, m * 2).reshape(m, 2), sizes)
  want = go.score_with_aux(pred, xc, xz, categorical_dof=2)[0]
  order = go.top_k(want, 2)
  np.testing.assert_array_equal(bi, order)
  np.testing.assert_array_equal(bz, xz[order])
  np.testing.assert_array_equal(bx, xc[order])
  np.testing.assert_allclose(bs, want[order], atol=TOL)


@pytest.mark.parametrize('m', [1, 5000, 60_000])
def test_score_host_matches_device_path(dev, m):
  """The HOST-buffer entry point (chunked H2D pipelined against scoring) returns exactly what the
  device-buffer entry point returns."""
  n, d = 200, 8
  x, y, _ = _problem(n, d, 61)
  po, pg = _params(d)
  dev.fit(x, y, pg)
  acq = _gp().Acquisition(1.8, True, go.trust_radius(n, d, 0))
  xs = np.random.default_rng(62).uniform(size=(m, d))
  out = dev.score(xs, acq, with_aux=True)
  dev.synchronize()
  score = np.empty(m); mean = np.empty(m); sd = np.empty(m); linf = np.empty(m)
  dev.score_host(xs, acq, score_out=score, mean_out=mean, stddev_out=sd, linf_out=linf)
  np.testing.assert_allclose(score, out['score'].cpu().numpy(), atol=1e-12, rtol=0)
  np.testing.assert_allclose(mean, out['mean'].cpu().numpy(), atol=1e-12, rtol=0)
  np.testing.assert_allclose(sd, out['stddev'].cpu().numpy(), atol=1e-12, rtol=0)
  np.testing.assert_array_equal(linf, out['linf_distance'].cpu().numpy())
  pinned = torch.from_numpy(xs).pin_memory(); s2 = torch.empty(m, dtype=torch.float64).pin_memory()
  dev.score_host(pinned, acq, score_out=s2)
  want, _ = go.score_with_aux(go.precompute_predictive(po, x, y), xs[:256])
  np.testing.assert_allclose(s2.numpy()[:256], want, atol=TOL, rtol=0)


def test_nll_grad_d50_multiblock(dev):
  """C4-like shape (D=50, several 64-blocks) against the oracle, plus a directional finite
  difference at the full C4 size (N=2000) using the device loss only."""
  n, d = 600, 50
  rng = np.random.default_rng(71)
  x = rng.uniform(size=(n, d)); y = rng.normal(size=n)
  ls2 = np.exp(rng.uniform(np.log(0.3), np.log(5.0), size=d))
  po = go.GPParams(0.9, ls2, 3e-2); pg = _gp().GPHyperParams(0.9, ls2, 3e-2)
  want_l, want_g = go.loss_and_grad(po.to_vector(), x, y)
  xt = torch.from_numpy(x).cuda(); yt = torch.from_numpy(y).cuda()
  loss, grad, _ = dev.loss_and_grad(xt, yt, pg)
  assert abs(loss - want_l) < 1e-8 * abs(want_l)
  np.testing.assert_allclose(grad, want_g, atol=1e-7 * np.max(np.abs(want_g)), rtol=0)
  n = 2000
  x = rng.uniform(size=(n, d)); y = rng.normal(size=n)
  xt = torch.from_numpy(x).cuda(); yt = torch.from_numpy(y).cuda()
  theta = pg.to_vector()
  l0, g0, _ = dev.loss_and_grad(xt, yt, pg)
  direction = rng.normal(size=theta.shape) * theta
  h = 1e-6
  lp, _, _ = dev.loss_and_grad(xt, yt, _gp().GPHyperParams.from_vector(theta + h * direction, d, 0))
  lm, _, _ = dev.loss_and_grad(xt, yt, _gp().GPHyperParams.from_vector(theta - h * direction, d, 0))
  fd = (lp - lm) / (2 * h)
  assert abs(fd - g0 @ direction) < 1e-4 * max(1.0, abs(fd))


def test_nll_grad_c4_full_size(dev):
  """BASELINE C4 (N=2000, D=50, 52 hyper-parameters): loss and the whole gradient against the oracle."""
  n, d = 2000, 50
  rng = np.random.default_rng(72)
  x = rng.uniform(size=(n, d)); y = rng.normal(size=n)
  ls2 = np.exp(rng.uniform(np.log(0.3), np.log(5.0), size=d))
  po = go.GPParams(0.9, ls2, 3e-2); pg = _gp().GPHyperParams(0.9, ls2, 3e-2)
  want_l, want_g = go.loss_and_grad(po.to_vector(), x, y)
  xt = torch.from_numpy(x).cuda(); yt = torch.from_numpy(y).cuda()
  for _ in range(2):   # eager capture call, then the replayed graph
    loss, grad, retries = dev.loss_and_grad(xt, yt, pg)
    assert retries == 0
    assert abs(loss - want_l) < 1e-9 * abs(want_l)
    np.testing.assert_allclose(grad, want_g, atol=1e-8 * np.max(np.abs(want_g)), rtol=0)


def _two_models(dev, n, d, n_pending, seed, high_noise=False):
  from vizier_b200 import gp
  x, y, _ = _problem(n, d, seed)
  xp = np.random.default_rng(seed + 1).uniform(size=(n_pending, d))
  po, pg = _params(d)
  pred_a = go.precompute_predictive(po, x, y)
  xb = np.concatenate([x, xp]); yb = np.concatenate([y, np.zeros(n_pending)])
  pob = go.GPParams(po.signal_variance, po.continuous_length_scale_squared, 1e-10 if high_noise else po.observation_noise_variance)
  pgb = gp.GPHyperParams(pob.signal_variance, pob.continuous_length_scale_squared, pob.observation_noise_variance)
  pred_b = go.precompute_predictive(pob, xb, yb)
  dev_b = gp.DeviceGP(0, stream=dev.stream)
  dev.fit(x, y, pg)
  dev_b.fit(xb, yb, pgb)
  return x, pred_a, pred_b, dev_b


@pytest.mark.parametrize('mode,n,n_pending,tr_rows,high_noise', [(0, 30, 4, None, False), (1, 30, 4, 32, False),
                                                                (1, 150, 7, 152, True), (0, 150, 0, None, False)])
def test_ucb_pe_score(dev, mode, n, n_pending, tr_rows, high_noise):
  """vzgp_score_pe against UCBScoreFunction / PEScoreFunction restated in the oracle
  (gp_ucb_pe.py:344-381, :434-492, strict trust region :221-242)."""
  from vizier_b200 import gp
  d = 4
  x, pred_a, pred_b, dev_b = _two_models(dev, n, d, n_pending, 81, high_noise)
  xs = np.random.default_rng(82).uniform(size=(333, d))
  xs[:3] = x[:3]
  mask = np.array([True, True, False, True])
  rows = (n + n_pending) if tr_rows is None else tr_rows
  radius = go.trust_radius(rows, int(mask.sum()), 0)
  thr = go.ucb_threshold(pred_a, pred_b, 1.8)
  want, aux = go.ucb_pe_score(pred_a, pred_b, xs, mode=mode, threshold=thr, tr_dim_mask=mask, tr_rows=rows,
                              trust_radius_value=radius)
  pe = gp.UcbPeAcquisition(mode=mode, threshold=thr, trust_radius=radius, tr_dim_mask=mask, tr_rows=0 if tr_rows is None else tr_rows)
  out = dev.score_pe(dev_b, xs, pe)
  np.testing.assert_allclose(out['mean'].cpu().numpy(), aux['mean'], atol=TOL, rtol=0)
  np.testing.assert_allclose(out['stddev'].cpu().numpy(), aux['stddev'], atol=TOL, rtol=0)
  np.testing.assert_allclose(out['stddev_from_all'].cpu().numpy(), aux['stddev_from_all'], atol=1e-8 if high_noise else TOL, rtol=0)
  np.testing.assert_allclose(out['score'].cpu().numpy(), want, atol=1e-7 if high_noise else 1e-9, rtol=0)
  if radius <= 0.5:
    assert np.any(want < -1e3)
  dev_b.close()


def test_eagle_random_normalisation_with_pe_acquisition(dev):
  """GP-UCB-PE's optimiser configuration: RANDOM force normalisation (eagle_strategy.py:858-885) and
  the PE acquisition as scoring function, trajectory against the oracle with shared Philox draws."""
  from vizier_b200 import _lib, gp
  n, d, n_pending = 40, 3, 3
  x, pred_a, pred_b, dev_b = _two_models(dev, n, d, n_pending, 91)
  mask = np.ones(d, bool)
  rows = n + n_pending
  radius = go.trust_radius(rows, d, 0)
  thr = go.ucb_threshold(pred_a, pred_b, 1.8)
  cfg_o = eo.EagleConfig(visibility=3.678, gravity=3.028, negative_gravity=0.0304, perturbation=0.2334,
                         perturbation_lower_bound=7.376e-4, penalize_factor=0.7818, normalization_scale=1.989,
                         prior_trials_pool_pct=0.4235, mutate_normalization_type=1)
  pool, batch, steps = 25, 25, 7
  for mode in (0, 1):
    score_fn = lambda xc, xz: go.ucb_pe_score(pred_a, pred_b, xc, mode=mode, threshold=thr, tr_dim_mask=mask,
                                              tr_rows=rows, trust_radius_value=radius)[0]
    wc, _, wr = eo.run_eagle_optimizer_mixed(score_fn, dim=d, sizes=np.zeros(0, int), pool_size=pool, batch_size=batch,
                                             max_evaluations=steps * batch, count=2, seed=13, cfg=cfg_o, prior_c=x,
                                             prior_z=np.zeros((n, 0), np.int32))
    cfg = _lib.EagleConfig(cfg_o.visibility, cfg_o.gravity, cfg_o.negative_gravity, cfg_o.perturbation,
                           cfg_o.perturbation_lower_bound, cfg_o.penalize_factor, cfg_o.normalization_scale,
                           cfg_o.prior_trials_pool_pct, pool, batch, steps * batch, 1.0, 30.0, 0.98, 1)
    pe = gp.UcbPeAcquisition(mode=mode, threshold=thr, trust_radius=radius, tr_dim_mask=mask)
    bx, _, br = dev.eagle_run(cfg, pe, 2, 13, prior=x, other=dev_b)
    np.testing.assert_allclose(br, wr, atol=1e-8)
    np.testing.assert_allclose(bx, wc, atol=1e-8)
  dev_b.close()
