"""The Eagle optimiser on the device against oracle/eagle_oracle.py with pool trimming, ties, non-finite rewards and an
active trust region, on every form of the loop (vzgp_get_int "eagle_route" is asserted in every case).

A. Lock step (tests/eagle_lockstep.py): the host-stepped loop runs k_eagle_suggest, k_eagle_update and
   k_eagle_seed_priors - the kernels of every form - with rewards chosen by the host, so each batch is compared with
   the oracle's and a wrong pool update shows when the fly is next visited.  tests/test_eagle_lockstep_host.py
   rehearses the same cases on the CPU.
B. The persistent, cooperative and graph forms score in-kernel.  They run a real acquisition with an explicit trust
   radius, one trust-region dimension off and tr_rows below the model's rows, and perturbation_lower_bound = 0.05
   (a fly is trimmed after 4 failed visits), for at most 16 steps; the winners must agree with the oracle's optimiser
   and with the stepped loop scored by the library's own scoring call to 1e-9.  Each case asserts on the oracle's side
   that between 20 % and 80 % of the scored candidates lay outside the region and that flies were trimmed early enough
   to be visited again.
"""
import dataclasses

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

import acq_oracle as ao  # noqa: E402
import eagle_lockstep as el  # noqa: E402
from oracle import eagle_oracle as eo  # noqa: E402
from oracle import gp_oracle as go  # noqa: E402

PERSISTENT, COOPERATIVE, GRAPH, STEPPED = 0, 1, 2, 3     # vzgp_eagle_route (include/vzgp.h)


def _mods():
  from vizier_b200 import _lib, gp
  return _lib, gp


def _config(cfg_o, pool, batch, steps, q=1):
  _lib, _ = _mods()
  return _lib.EagleConfig(cfg_o.visibility, cfg_o.gravity, cfg_o.negative_gravity, cfg_o.perturbation,
                          cfg_o.perturbation_lower_bound, cfg_o.penalize_factor, cfg_o.normalization_scale,
                          cfg_o.prior_trials_pool_pct, pool, batch, steps * batch, cfg_o.categorical_perturbation_factor,
                          cfg_o.pure_categorical_perturbation_factor, cfg_o.prob_same_category_without_perturbation,
                          cfg_o.mutate_normalization_type, q)


def _params(d, dk):
  _, gp = _mods()
  ls2 = 0.5 * (1 + np.arange(d) / max(d, 1))
  lk = np.linspace(0.6, 1.4, dk) if dk else None
  return go.GPParams(1.0, ls2, 1e-3, lk), gp.GPHyperParams(1.0, ls2, 1e-3, lk)


# ---------------------------------------------------------------------------------------------------------------------
# A. lock step over the host-stepped loop
# ---------------------------------------------------------------------------------------------------------------------
class DeviceLoop:
  """The ask / tell / end shape of eagle_lockstep.run over gp.SteppedEagle."""

  def __init__(self, dev, case: el.Case):
    _, gp = _mods()
    self.dev, self.case = dev, case
    self.se = gp.SteppedEagle(dev, _config(case.cfg, case.pool, case.batch, case.steps, case.q), case.count, case.seed,
                              n_prior=case.n_prior, cat_sizes=case.sizes or None)
    assert dev.get_int('eagle_route') == STEPPED

  def seed(self, pc, pz, r):
    self.se.seed(pc if self.case.dc else None, pz if self.case.sizes else None, r)

  def ask(self):
    xs, zs, self._r = self.se.ask()
    with torch.cuda.stream(self.dev.stream):
      xc = xs.cpu().numpy().copy()
      xz = zs.cpu().numpy().copy() if zs is not None else np.zeros((self.case.batch, 0), np.int32)
    return xc, xz

  def tell(self, r):
    with torch.cuda.stream(self.dev.stream):
      self._r.copy_(torch.from_numpy(np.ascontiguousarray(r, np.float64)))
    self.se.tell()

  def end(self):
    return self.se.end()


@pytest.mark.parametrize('case', el.CASES, ids=lambda c: c.name)
def test_stepped_loop_in_lock_step_with_oracle(case):
  _, gp = _mods()
  rng = np.random.default_rng(3)
  n, dk = 8, len(case.sizes)
  x = rng.uniform(size=(n, case.dc))
  z = np.stack([rng.integers(0, s, size=n) for s in case.sizes], axis=1).astype(np.int32) if dk else None
  dev = gp.DeviceGP(0)
  try:
    dev.fit(x, rng.normal(size=n), _params(case.dc, dk)[1], z=z)      # the handle only has to know Dc and Dk
    rep = el.run(case, DeviceLoop(dev, case))
    print(f'{case.name}: eagle_route {dev.get_int("eagle_route")} {rep}')
  finally:
    dev.close()


# ---------------------------------------------------------------------------------------------------------------------
# B. the fused forms: real scorer, active trust region, trimming
# ---------------------------------------------------------------------------------------------------------------------
CHEAP_TRIM = eo.EagleConfig(perturbation_lower_bound=0.05)     # 0.16 * 0.7^4 < 0.05: trimmed at the 4th failed visit
SIZES = (3, 4)
COUNT = 8


@dataclasses.dataclass(frozen=True)
class Fused:
  name: str
  route: int
  kind: str               # 'ucb', 'ei' (vzgp_set_acquisition: the GENERIC kernels), 'pe0', 'pe1' (GP-UCB-PE modes)
  n: int
  d: int
  pool: int
  batch: int
  radius: float
  dk: int = 0
  n_pending: int = 0      # rows of model B beyond model A's (GP-UCB-PE)

  @property
  def steps(self):
    return min(4 * (self.pool // self.batch) + 8, 16)


FUSED = [
    # persistent: np == 64, B <= 64.  N = 40 leaves 24 all-zero padded trial rows: the priors near the origin would be
    # inside the region if one of those rows were trusted.
    Fused('persistent-N40-nb1', PERSISTENT, 'ucb', 40, 4, 25, 25, 0.15),
    Fused('persistent-N64-nb2', PERSISTENT, 'ucb', 64, 4, 50, 25, 0.1),
    Fused('persistent-ei', PERSISTENT, 'ei', 40, 4, 50, 25, 0.15),
    Fused('persistent-pe0', PERSISTENT, 'pe0', 40, 4, 25, 25, 0.15, n_pending=6),
    Fused('persistent-pe1', PERSISTENT, 'pe1', 40, 4, 50, 25, 0.15, n_pending=6),
    Fused('persistent-dk2', PERSISTENT, 'ucb', 40, 3, 25, 25, 0.2, dk=2),
    # cooperative: one CTA per fly in eagle_suggest_cta, 64-candidate tiles
    Fused('cooperative-N130', COOPERATIVE, 'ucb', 130, 4, 50, 25, 0.08),
    Fused('cooperative-N300-B100', COOPERATIVE, 'ucb', 300, 5, 200, 100, 0.12),
    Fused('cooperative-B512', COOPERATIVE, 'ucb', 130, 4, 512, 512, 0.12),
    Fused('cooperative-ei', COOPERATIVE, 'ei', 130, 4, 50, 25, 0.08),
    Fused('cooperative-pe0', COOPERATIVE, 'pe0', 120, 4, 50, 25, 0.12, n_pending=10),    # np 128 and 192
    Fused('cooperative-pe1', COOPERATIVE, 'pe1', 120, 4, 25, 25, 0.12, n_pending=10),
    Fused('cooperative-dk2', COOPERATIVE, 'ucb', 130, 3, 50, 25, 0.15, dk=2),
    # graph: batches above 512 are scored by launch_score between k_eagle_suggest and k_eagle_update
    Fused('graph-B600', GRAPH, 'ucb', 700, 4, 1200, 600, 0.12),
]


def _fused_problem(c: Fused):
  """Trials away from the origin corner, pending points, priors = every trial (the untrusted last rows included) plus
  three points in the origin corner."""
  rng = np.random.default_rng(17)
  nb = c.n + c.n_pending
  x = rng.uniform(0.3, 0.7, size=(nb, c.d))
  z = np.stack([rng.integers(0, s, size=nb) for s in SIZES[:c.dk]], axis=1).astype(np.int32) if c.dk else None
  y = -np.sum((x[:c.n] - 0.85) ** 2, axis=1) + 0.05 * rng.normal(size=c.n)
  if c.dk:
    y -= 0.3 * (z[:c.n, 0] != 1)
  mask = np.ones(c.d, bool)
  mask[1] = False
  rows = nb - (2 if c.n_pending else 5)
  prior_c = np.concatenate([x[:c.n], rng.uniform(0.0, 0.08, size=(3, c.d))])
  prior_z = np.concatenate([z[:c.n], z[:3]]) if c.dk else np.zeros((c.n + 3, 0), np.int32)
  return x, y, z, mask, rows, prior_c, prior_z


def _fused_oracle(c: Fused):
  """The oracle's optimiser on the oracle's acquisition; returns its winners and the device-side acquisition spec."""
  x, y, z, mask, rows, prior_c, prior_z = _fused_problem(c)
  po, _ = _params(c.d, c.dk)
  pred_a = go.precompute_predictive(po, x[:c.n], y, None if z is None else z[:c.n])
  pred_b, thr = None, 0.0
  if c.n_pending:
    pred_b = go.precompute_predictive(po, x, np.r_[y, np.zeros(c.n_pending)], z)
    thr = go.ucb_threshold(pred_a, pred_b, 1.8)
  best = float(np.max(y))
  seen = {'calls': 0, 'scored': 0, 'outside': 0}

  def score(xc, xz):
    zs = xz if c.dk else None
    if c.kind in ('ucb', 'ei'):
      mu, sd = go.predict(pred_a, xc, zs)
      acq = mu + 1.8 * sd if c.kind == 'ucb' else ao.ei(mu, sd, best)
      dist = go.min_linf_distance(xc, x[:rows], mask)
      out, outside = go.apply_trust_region(acq, dist, c.radius), dist > c.radius
    else:
      out = go.ucb_pe_score(pred_a, pred_b, xc, zs, mode=int(c.kind[-1]), threshold=thr, tr_dim_mask=mask, tr_rows=rows,
                            trust_radius_value=c.radius)[0]
      outside = go.min_linf_distance(xc, x[:rows], mask) >= c.radius
    if seen['calls']:                   # the first call scores the priors
      seen['scored'] += outside.size
      seen['outside'] += int(np.sum(outside))
    seen['calls'] += 1
    return out

  watch = el.Watch(c.pool, c.batch, c.steps, CHEAP_TRIM)
  wc, wz, wr = eo.run_eagle_optimizer_mixed(score, dim=c.d, sizes=np.asarray(SIZES[:c.dk], np.int64), pool_size=c.pool,
                                            batch_size=c.batch, max_evaluations=c.steps * c.batch, count=COUNT, seed=5,
                                            cfg=CHEAP_TRIM, prior_c=prior_c, prior_z=prior_z, on_step=watch)
  share = seen['outside'] / seen['scored']
  rep = dict(outside=round(share, 3), trims=watch.trims, first_trim=min(watch.trim_steps, default=None), steps=c.steps)
  assert 0.2 <= share <= 0.8, rep
  assert watch.trims >= 3 and min(watch.trim_steps) < c.steps - 3, rep
  return (wc, wz, wr), rep, thr, best


def test_pe_pair_on_one_handle_takes_the_graph_form():
  """GP-UCB-PE with one handle as both models: the cooperative kernel keeps a workspace per member handle, so a shared
  handle must take the replayed graph."""
  c = next(f for f in FUSED if f.name == 'cooperative-pe1')
  _lib, gp = _mods()
  x, y, _, mask, _, prior_c, _ = _fused_problem(c)
  _, pg = _params(c.d, c.dk)
  dev = gp.DeviceGP(0)
  try:
    dev.fit(x[:c.n], y, pg)
    acq = gp.UcbPeAcquisition(mode=1, threshold=float(np.max(y)), trust_radius=c.radius, tr_dim_mask=mask, tr_rows=c.n)
    _, _, br = dev.eagle_run(_config(CHEAP_TRIM, c.pool, c.batch, c.steps), acq, COUNT, 5, other=dev, prior=prior_c)
    assert dev.get_int('eagle_route') == GRAPH
    assert np.all(np.isfinite(br))
  finally:
    dev.close()


@pytest.mark.parametrize('c', FUSED, ids=lambda c: c.name)
def test_fused_forms_with_trust_region_and_trimming(c):
  _lib, gp = _mods()
  x, y, z, mask, rows, prior_c, prior_z = _fused_problem(c)
  (wc, wz, wr), rep, thr, best = _fused_oracle(c)
  _, pg = _params(c.d, c.dk)
  dev = gp.DeviceGP(0)
  dev_b = gp.DeviceGP(0, stream=dev.stream) if c.n_pending else None
  try:
    dev.fit(x[:c.n], y, pg, z=None if z is None else z[:c.n])
    if dev_b is not None:
      dev_b.fit(x, np.r_[y, np.zeros(c.n_pending)], pg, z=z)
    if c.kind in ('ucb', 'ei'):
      spec = gp.AcqFnSpec(gp.AcqTermSpec(_lib.ACQ_EI, best_label=best, exploration=ao.EI_EXPLORATION)) if c.kind == 'ei' else None
      acq = gp.Acquisition(1.8, True, c.radius, mask, tr_rows=rows, acq_fn=spec)
      score = lambda xs, zs: dev.score(xs, acq, zs=zs)['score']
    else:
      acq = gp.UcbPeAcquisition(mode=int(c.kind[-1]), threshold=thr, trust_radius=c.radius, tr_dim_mask=mask, tr_rows=rows)
      score = lambda xs, zs: dev.score_pe(dev_b, xs, acq, zs=zs)['score']
    cfg = _config(CHEAP_TRIM, c.pool, c.batch, c.steps)
    kw = dict(prior=prior_c, prior_z=prior_z if c.dk else None, cat_sizes=SIZES[:c.dk] or None)
    bc, bz, br = dev.eagle_run(cfg, acq, COUNT, 5, other=dev_b, **kw)
    route = dev.get_int('eagle_route')
    print(f'{c.name}: eagle_route {route} {rep}')
    assert route == c.route
    np.testing.assert_allclose(br, wr, rtol=0, atol=1e-9)
    np.testing.assert_allclose(bc, wc, rtol=0, atol=1e-9)
    np.testing.assert_array_equal(bz, wz)

    # the same run through the stepped loop, scored by the library's scoring call
    se = gp.SteppedEagle(dev, cfg, COUNT, 5, n_prior=len(prior_c), cat_sizes=kw['cat_sizes'])
    pzt = torch.from_numpy(prior_z).cuda() if c.dk else None
    se.seed(prior_c, kw['prior_z'], score(torch.from_numpy(prior_c).cuda(), pzt))
    for _ in range(c.steps):
      xs, zs, rewards = se.ask()
      r = score(xs, zs)
      with torch.cuda.stream(dev.stream):
        rewards.copy_(r)
      se.tell()
    sc, sz, sr = se.end()
    assert dev.get_int('eagle_route') == STEPPED
    np.testing.assert_allclose(sr, br, rtol=0, atol=1e-9)
    np.testing.assert_allclose(sc, bc, rtol=0, atol=1e-9)
    np.testing.assert_array_equal(sz, bz)
  finally:
    dev.close()
    if dev_b is not None:
      dev_b.close()
