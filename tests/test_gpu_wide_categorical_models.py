"""Multi-model scoring and Eagle loops of models with more than 32 categorical features.

Scoring against the oracle on the general route (score_route 4): multi-metric means and scalarised UCB
(k_mean_multi's wide form), the separable model's scores and its NLL task-covariance gradient (the task Gram is
k_mean_multi on the trials), ensembles and stacks.  Dk = 40 splits into a full and a partial tile of 32 features,
Dk = 65 into three; pools of 4097 candidates cross the general route's 4096-candidate chunk.

Eagle: vzgp_eagle_run's ensemble, stack, GP-UCB-PE (single models and ensembles), multi-metric and separable variants
end on the replayed graph (eagle_route 2) with the winners of the host-stepped loop scored by the same model.
"""
import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from oracle import eagle_oracle as eo  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402
import separable_oracle as sepo  # noqa: E402
import stack_oracle as sto  # noqa: E402
import test_gpu_separable as tsep  # noqa: E402

GENERAL = 4                    # vzgp_score_route
EAGLE_GRAPH = 2                # vzgp_eagle_route
UCB = 1.8


def _gp():
  from vizier_b200 import gp
  return gp


def _params(dc, dk, k=0):
  """Member k's hyper-parameters as (oracle, device); categorical length scales of the order of Dk, so the Hamming
  term stays O(1) and K is far from the identity."""
  gp = _gp()
  sf2, sn2 = 0.8 + 0.2 * k, 2e-3 * (1 + k)
  ls2 = 0.3 * (1.0 + np.arange(dc) / max(dc, 1)) * (1 + 0.2 * k)
  lk = np.linspace(0.5, 1.5, dk) * dk / 4 * (1 + 0.1 * k)
  return go.GPParams(sf2, ls2, sn2, lk), gp.GPHyperParams(sf2, ls2, sn2, lk)


def _trials(n, dc, dk, seed, m=1):
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, dc))
  z = rng.integers(0, 3, size=(n, dk)).astype(np.int32)
  f = np.sin(3.0 * x.sum(1)) + 0.3 * np.cos(z[:, :7].sum(1)) - 0.2 * (z[:, -1] == 1)
  y = np.stack([f * (1 + 0.3 * k) + 0.2 * k * np.cos(3 * x[:, 0]) + 0.03 * rng.normal(size=n) for k in range(m)], 1)
  return x, (y[:, 0] if m == 1 else y), z


def _pool(mc, dc, dk, seed):
  rng = np.random.default_rng(seed)
  return rng.uniform(size=(mc, dc)), rng.integers(0, 3, size=(mc, dk)).astype(np.int32)


def _pick(mc):
  return np.unique(np.r_[np.arange(min(mc, 200)), np.arange(4090, 4100), mc - 1] % mc)


def _close(got, want):
  np.testing.assert_allclose(got, want, atol=1e-10 * max(1.0, float(np.max(np.abs(want)))), rtol=0)


def _weights(y, m, seed):
  rng = np.random.default_rng(seed)
  w = np.abs(rng.normal(size=(100, m)))
  w /= np.linalg.norm(w, axis=1, keepdims=True)
  ref = go.hv_reference_point(y)
  return w, ref, go.hv_max_scalarized(y, w, ref)


# ---------------------------------------------------------------------------------------------------------------------
# A. scoring against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dk,mc', [(40, 300), (40, 4097), (65, 4097)])
def test_multi_metric_scores(dk, mc):
  gp = _gp()
  x, y, z = _trials(150, 3, dk, dk, m=2)
  po, pg = _params(3, dk)
  dev = gp.DeviceGP(0)
  try:
    assert dev.fit(x, y, pg, z=z) == 0
    xs, zs = _pool(mc, 3, dk, mc + dk)
    pick = _pick(mc)
    mu, sd = go.predict(go.precompute_predictive(po, x, y, z), xs[pick], zs[pick])
    w, ref, best = _weights(y, 2, 1)
    for floor in (best, None):
      out = dev.score_multi(xs, gp.ScalarizedUcbAcquisition(w, ref, floor, UCB), zs=zs, with_aux=True)
      dev.synchronize()
      assert dev.get_int('score_route') == GENERAL
      _close(out['mean'].cpu().numpy().T[pick], mu)
      _close(out['stddev'].cpu().numpy()[pick], sd)
      _close(out['score'].cpu().numpy()[pick], go.scalarized_ucb(mu, sd, w, ref, floor))
  finally:
    dev.close()


@pytest.mark.parametrize('dk,mc', [(40, 4097), (65, 300)])
def test_separable_scores(dk, mc):
  gp = _gp()
  from vizier_b200 import task_kernels as tk
  x, y, z = _trials(120, 3, dk, dk + 1, m=2)
  po, _ = _params(3, dk)
  pg = gp.GPHyperParams(po.signal_variance, po.continuous_length_scale_squared, po.observation_noise_variance,
                        po.categorical_length_scale_squared, multitask_type=tk.LKJ, task_params=np.array([0.8, 0.9, 0.6]))
  sep = gp.SeparableGP(0, 2)
  try:
    assert sep.fit(x, y, pg, z=z) == 0
    xs, zs = _pool(mc, 3, dk, mc + dk + 1)
    pick = _pick(mc)
    mu, sd = sepo.marginals(po, pg.task_covariance(), x, y, xs[pick], z, zs[pick])
    w, ref, best = _weights(y, 2, 2)
    out = sep.score_multi(xs, gp.ScalarizedUcbAcquisition(w, ref, best, UCB), zs=zs, with_aux=True)
    sep.synchronize()
    assert {m.get_int('score_route') for m in sep.members} == {GENERAL}
    _close(out['mean'].cpu().numpy().T[pick], mu)
    _close(out['stddev'].cpu().numpy().T[pick], sd)
    _close(out['score'].cpu().numpy()[pick], sepo.scalarized_ucb(mu, sd, w, ref, best))
  finally:
    sep.close()


@pytest.mark.parametrize('n,dk,nv', [(40, 40, 40), (130, 40, 120), (130, 65, 130)])
def test_separable_nll_task_gradient(n, dk, nv):
  """vzgp_nll_grad_separable_batch: loss, base gradient and dL/dT (the task Gram of k_mean_multi's wide form)."""
  gp = _gp()
  from vizier_b200 import task_kernels as tk
  x, y, z = _trials(n, 3, dk, n + dk, m=2)
  valid = np.arange(n) < nv
  rng = np.random.default_rng(3)
  devs = [gp.DeviceGP(0) for _ in range(6)]
  try:
    for kind in tk.TYPES:
      ps, tcs, want = [], [], []
      for r in range(3):
        po, _ = _params(3, dk, r)
        t = sepo.task_cov(kind, tsep._theta(kind, 2, rng), 2)
        ps.append(gp.GPHyperParams(po.signal_variance, po.continuous_length_scale_squared, po.observation_noise_variance,
                                   po.categorical_length_scale_squared))
        tcs.append(t)
        want.append(sepo.loss_and_grad(po, t, x, y, z, valid))
      loss, grad, gt, st = tsep._raw_batch(devs, 2, ps, tcs, x, y, z, nv)
      for r in range(3):
        wl, wg, wt, wi = want[r]
        assert st[r] == wi == 0
        assert abs(loss[r] - wl) < 1e-9 * max(1.0, abs(wl))
        np.testing.assert_allclose(grad[r], wg, atol=1e-8 * max(1.0, np.max(np.abs(wg))), rtol=0)
        np.testing.assert_allclose(gt[r], wt, atol=1e-8 * max(1.0, np.max(np.abs(wt))), rtol=0)
  finally:
    for d in devs:
      d.close()


@pytest.mark.parametrize('dk,mc', [(40, 4097), (65, 300)])
def test_ensemble_scores(dk, mc):
  gp = _gp()
  x, y, z = _trials(110, 3, dk, dk + 2)
  ps = [_params(3, dk, k) for k in range(3)]
  ens = gp.EnsembleGP(0, 3)
  try:
    assert ens.fit(x, y, [pg for _, pg in ps], z=z) == 0
    xs, zs = _pool(mc, 3, dk, mc + dk + 2)
    pick = _pick(mc)
    mu, sd = go.predict_ensemble([go.precompute_predictive(po, x, y, z) for po, _ in ps], xs[pick], zs[pick])
    out = ens.score(xs, gp.Acquisition(UCB, False, 1.0), zs=zs, with_aux=True)
    ens.synchronize()
    assert {m.get_int('score_route') for m in ens.members} == {GENERAL}
    _close(out['mean'].cpu().numpy()[pick], mu)
    _close(out['stddev'].cpu().numpy()[pick], sd)
    _close(out['score'].cpu().numpy()[pick], mu + UCB * sd)
  finally:
    ens.close()


def _stack(dc, dk, e, seed):
  """Two levels (prior study, current study) of e members each: (StackedGP, oracle levels, top x, top z)."""
  gp = _gp()
  stack = gp.StackedGP(0)
  levels = []
  for l, n in enumerate((90, 50)):
    x, y, z = _trials(n, dc, dk, seed + l)
    resid_o = sto.residual_labels(levels, x, y, z)
    resid_d = y - stack.mean(x, z) if stack.levels else y
    np.testing.assert_allclose(resid_d, resid_o, rtol=0, atol=1e-9)
    ps = [_params(dc, dk, k + l) for k in range(e)]
    levels.append([go.precompute_predictive(po, x, resid_o, z) for po, _ in ps])
    level = stack.new_level(e)
    level.fit(x, resid_d, [pg for _, pg in ps] if e > 1 else ps[0][1], z=z)
    stack.push(level, n)
  return stack, levels, x, z


@pytest.mark.parametrize('e', [1, 2])
def test_stack_scores(e):
  gp = _gp()
  dk, mc = 40, 4097
  stack, levels, _, _ = _stack(3, dk, e, 7 + e)
  try:
    xs, zs = _pool(mc, 3, dk, 5)
    pick = _pick(mc)
    out = stack.score(xs, gp.Acquisition(UCB, False, 1.0), zs=zs, with_aux=True)
    stack.synchronize()
    assert {h.get_int('score_route') for h in stack._devices()} == {GENERAL}
    want, mean, sd, _ = sto.score(levels, xs[pick], zs[pick], coefficient=UCB)
    _close(out['mean'].cpu().numpy()[pick], mean)
    _close(out['stddev'].cpu().numpy()[pick], sd)
    _close(out['score'].cpu().numpy()[pick], want)
  finally:
    stack.close()


# ---------------------------------------------------------------------------------------------------------------------
# B. the Eagle variants: replayed graph, winners of the stepped loop scored by the same model
# ---------------------------------------------------------------------------------------------------------------------
STEPS, POOL, BATCH, COUNT, SEED = 6, 50, 25, 3, 9


def _config():
  from vizier_b200 import _lib
  c = eo.EagleConfig()
  return _lib.EagleConfig(c.visibility, c.gravity, c.negative_gravity, c.perturbation, c.perturbation_lower_bound,
                          c.penalize_factor, c.normalization_scale, c.prior_trials_pool_pct, POOL, BATCH, STEPS * BATCH,
                          c.categorical_perturbation_factor, c.pure_categorical_perturbation_factor,
                          c.prob_same_category_without_perturbation, c.mutate_normalization_type, 1)


def _stepped(owner, sizes, prior, prior_z, score):
  """The host-stepped loop on `owner` with every batch (and the prior trials) scored by `score(xs, zs)`."""
  gp = _gp()
  se = gp.SteppedEagle(owner, _config(), COUNT, SEED, n_prior=len(prior), cat_sizes=sizes)
  pt, pz = torch.from_numpy(prior).cuda(), torch.from_numpy(prior_z).cuda()
  se.seed(prior, prior_z, score(pt, pz))
  for _ in range(STEPS):
    xs, zs, rewards = se.ask()
    r = score(xs, zs)
    with torch.cuda.stream(owner._stream):
      rewards.copy_(r)
    se.tell()
  return se.end()


def _handles(model):
  return model._devices() if hasattr(model, '_devices') else [model]


def _check(owner, run, score, models, sizes, prior, prior_z):
  bx, bz, br = run()
  routes = {h.get_int('eagle_route') for m in models for h in _handles(m)} - {-1}
  assert routes == {EAGLE_GRAPH}, routes
  sx, sz, sr = _stepped(owner, sizes, prior, prior_z, score)
  np.testing.assert_allclose(br, sr, atol=1e-9 * max(1.0, float(np.max(np.abs(sr)))), rtol=0)
  np.testing.assert_allclose(bx, sx, atol=1e-9, rtol=0)
  np.testing.assert_array_equal(bz, sz)
  assert np.isfinite(br).all()


VARIANTS = ['ensemble', 'stack', 'stack-ensemble', 'pe', 'pe-ensemble', 'multi', 'separable']


@pytest.mark.parametrize('variant', VARIANTS)
def test_eagle_variants_on_graph(variant):
  gp = _gp()
  from vizier_b200 import task_kernels as tk
  dc, dk = 3, 40
  sizes = [2 + k % 4 for k in range(dk)]
  acq = gp.Acquisition(UCB, False, 1.0)
  opened = []
  try:
    if variant in ('ensemble', 'pe-ensemble'):
      x, y, z = _trials(80, dc, dk, 21)
      z = z % np.asarray(sizes, np.int32)
      ps = [_params(dc, dk, k) for k in range(3)]
      a = gp.EnsembleGP(0, 3); opened.append(a)
      a.fit(x, y, [pg for _, pg in ps], z=z)
      if variant == 'ensemble':
        _check(a, lambda: a.eagle_run(_config(), acq, COUNT, SEED, prior=x[:10], prior_z=z[:10], cat_sizes=sizes),
               lambda xs, zs: a.score(xs, acq, zs=zs)['score'], [a], sizes, x[:10], z[:10])
        return
      b = gp.EnsembleGP(0, 3, stream=a.stream); opened.append(b)
      b.fit(np.r_[x, x[:4] * 0.5], np.r_[y, np.zeros(4)], [pg for _, pg in ps], z=np.r_[z, z[:4]])
    elif variant == 'pe':
      x, y, z = _trials(80, dc, dk, 22)
      z = z % np.asarray(sizes, np.int32)
      _, pg = _params(dc, dk)
      a = gp.DeviceGP(0); opened.append(a)
      b = gp.DeviceGP(0, stream=a.stream); opened.append(b)
      a.fit(x, y, pg, z=z)
      b.fit(np.r_[x, x[:4] * 0.5], np.r_[y, np.zeros(4)], pg, z=np.r_[z, z[:4]])
    elif variant.startswith('stack'):
      stack, _, x, z = _stack(dc, dk, 2 if variant == 'stack-ensemble' else 1, 31)
      opened.append(stack)
      # categories of the trials stay within `sizes` only if they are below every size: 3 categories, sizes >= 2
      zc = z % np.asarray(sizes, np.int32)
      _check(stack, lambda: stack.eagle_run(_config(), acq, COUNT, SEED, prior=x[:10], prior_z=zc[:10], cat_sizes=sizes),
             lambda xs, zs: stack.score(xs, acq, zs=zs)['score'], [stack], sizes, x[:10], zc[:10])
      return
    else:
      x, y, z = _trials(90, dc, dk, 23, m=2)
      z = z % np.asarray(sizes, np.int32)
      po, pg = _params(dc, dk)
      w, ref, best = _weights(y, 2, 4)
      sc = gp.ScalarizedUcbAcquisition(w, ref, best, UCB)
      if variant == 'multi':
        m = gp.DeviceGP(0)
        opened.append(m)
        m.fit(x, y, pg, z=z)
      else:
        m = gp.SeparableGP(0, 2)
        opened.append(m)
        m.fit(x, y, gp.GPHyperParams(po.signal_variance, po.continuous_length_scale_squared,
                                     po.observation_noise_variance, po.categorical_length_scale_squared,
                                     multitask_type=tk.LKJ, task_params=np.array([0.8, 0.9, 0.6])), z=z)
      _check(m, lambda: m.eagle_run(_config(), sc, COUNT, SEED, prior=x[:10], prior_z=z[:10], cat_sizes=sizes),
             lambda xs, zs: m.score_multi(xs, sc, zs=zs)['score'], [m], sizes, x[:10], z[:10])
      return
    # GP-UCB-PE on single models or ensembles, both modes
    for mode in (0, 1):
      pe = gp.UcbPeAcquisition(mode=mode, ucb_coefficient=UCB, use_trust_region=False)
      _check(a, lambda: a.eagle_run(_config(), pe, COUNT, SEED, prior=x[:10], prior_z=z[:10], cat_sizes=sizes, other=b),
             lambda xs, zs: a.score_pe(b, xs, pe, zs=zs)['score'], [a, b], sizes, x[:10], z[:10])
  finally:
    for o in reversed(opened):
      o.close()
