"""The Eagle optimiser's UNNORMALIZED force normalisation, its MULTIPLICATIVE perturbation and categorical features of
more than 64 values on the device, against tests/eagle_options_oracle.py, on every form of the loop (vzgp_get_int
"eagle_route" is asserted in every case).

A. Lock step over the host-stepped loop (k_eagle_suggest, k_eagle_suggest_wide, k_eagle_update): each batch equals
   the oracle's, continuous features within 1e-12 and categories exactly; rewards come from the schedules of
   tests/eagle_lockstep.py.
B. The persistent, cooperative and graph forms score in-kernel: their winners must agree with the oracle's optimiser
   on the oracle's UCB to 1e-9.
C. Random search, the designers on a space with 100- and 1000-value categorical parameters, and the perturbation type
   through VectorizedOptimizer (eagle_strategy_test.py:443-495).
"""
import dataclasses

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

import eagle_lockstep as el  # noqa: E402
import eagle_options_oracle as xo  # noqa: E402
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


def _trials(n, d, sizes, seed):
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, d))
  z = np.stack([rng.integers(0, s, size=n) for s in sizes], axis=1).astype(np.int32) if sizes else None
  return x, z


# ---------------------------------------------------------------------------------------------------------------------
# A. lock step over the host-stepped loop
# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class Step:
  case: el.Case
  pert: int = xo.ADDITIVE


def _s(name, schedule, dc, pool, batch, steps, count, pert=xo.ADDITIVE, **kw):
  return Step(el.Case(name, schedule, dc, pool, batch, steps, count, **kw), pert)


STEPS = [
    _s('unnorm-cont', 'decaying', 4, 10, 5, 50, 6, norm=2),
    _s('unnorm-mixed', 'quantised', 3, 20, 5, 30, 16, norm=2, sizes=(2, 65, 1000), n_prior=12),
    _s('unnorm-sets-q3', 'decaying', 5, 10, 5, 50, 3, norm=2, q=3, n_prior=9),
    _s('unnorm-sets-wide', 'improving', 21, 20, 5, 24, 3, norm=2, q=4),                 # 84 columns: k_eagle_suggest_wide
    _s('mult-cont', 'decaying', 4, 10, 5, 50, 6, pert=xo.MULTIPLICATIVE),
    _s('mult-mixed-random', 'quantised', 3, 20, 5, 30, 16, pert=xo.MULTIPLICATIVE, norm=1, sizes=(3, 100, 257)),
    _s('mult-sets-q3', 'decaying', 5, 10, 5, 50, 3, pert=xo.MULTIPLICATIVE, q=3, n_prior=9),
    _s('mult-sets-wide', 'improving', 21, 20, 5, 24, 3, pert=xo.MULTIPLICATIVE, q=4),
    _s('unnorm-mult-mixed', 'decaying', 2, 10, 5, 50, 4, pert=xo.MULTIPLICATIVE, norm=2, sizes=(65, 5)),
    _s('cat-65-100-257-1000', 'decaying', 3, 10, 5, 50, 4, sizes=(1, 64, 65, 100, 257, 1000), n_prior=20),
    _s('cat-only-big', 'quantised', 0, 20, 5, 30, 16, sizes=(65, 1000, 7), n_prior=30),
    _s('cat-only-big-random', 'decaying', 0, 10, 5, 50, 4, norm=1, sizes=(100, 2, 257)),
    _s('cat-big-B27', 'quantised', 3, 54, 27, 12, 8, sizes=(1000, 33)),                 # B % 8 != 0: a partial CTA
]


class DeviceLoop:
  """ask / tell / end over gp.SteppedEagle, started with the case's perturbation type on the handle."""

  def __init__(self, dev, st: Step):
    _, gp = _mods()
    c = st.case
    self.dev, self.case = dev, c
    dev.set_int('eagle_perturbation', st.pert)
    self.se = gp.SteppedEagle(dev, _config(c.cfg, c.pool, c.batch, c.steps, c.q), c.count, c.seed,
                              n_prior=c.n_prior, cat_sizes=c.sizes or None)
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


def _lockstep(st: Step, opt: DeviceLoop):
  """The oracle's runner with the device loop compared at every batch; returns the number of batches compared."""
  c = st.case
  state = {'t': -1 if c.n_prior else 0}
  pc, pz = el.priors(c)

  def score(xc, xz=None):
    t = state['t']
    state['t'] = t + 1
    xc = np.asarray(xc, np.float64).reshape(xc.shape[0], c.width)
    xz = np.zeros((xc.shape[0], 0), np.int32) if xz is None else np.asarray(xz, np.int32)
    r = el.rewards(c, t, xc, xz)
    if t < 0:
      opt.seed(xc, xz, r)
      return r
    gc, gz = opt.ask()
    np.testing.assert_allclose(gc, xc, rtol=0, atol=1e-12, err_msg=f'{c.name}: continuous batch of step {t}')
    np.testing.assert_array_equal(gz, xz, err_msg=f'{c.name}: categorical batch of step {t}')
    opt.tell(r)
    return r

  common = dict(pool_size=c.pool, batch_size=c.batch, max_evaluations=c.steps * c.batch, count=c.count, seed=c.seed,
                cfg=c.cfg, perturbation_type=st.pert)
  if c.q > 1:
    wc, wr = xo.run_sets(lambda x: score(x.reshape(x.shape[0], -1)), dim=c.dc, n_parallel=c.q,
                         prior_features=pc.reshape(-1, c.dc) if c.n_prior else None, **common)
    wc, wz = wc.reshape(c.count, c.width), np.zeros((c.count, 0), np.int32)
  else:
    wc, wz, wr = xo.run_mixed(score, dim=c.dc, sizes=np.asarray(c.sizes, np.int64), prior_c=pc if c.n_prior else None,
                              prior_z=pz if c.n_prior else None, **common)
  assert state['t'] == c.steps
  bc, bz, br = opt.se.end()
  np.testing.assert_array_equal(br, wr, err_msg=f'{c.name}: winners\' rewards')
  np.testing.assert_array_equal(bz, wz, err_msg=f'{c.name}: winners\' categories')
  np.testing.assert_allclose(bc, wc, rtol=0, atol=1e-12, err_msg=f'{c.name}: winners\' features')
  return state['t']


@pytest.mark.parametrize('st', STEPS, ids=lambda s: s.case.name)
def test_stepped_loop_in_lock_step_with_oracle(st):
  _, gp = _mods()
  c = st.case
  x, z = _trials(8, c.dc, c.sizes, 3)
  dev = gp.DeviceGP(0)
  try:
    dev.fit(x, np.random.default_rng(4).normal(size=8), _params(c.dc, len(c.sizes))[1], z=z)
    n = _lockstep(st, DeviceLoop(dev, st))
    print(f'{c.name}: {n} batches in lock step')
  finally:
    dev.close()


# ---------------------------------------------------------------------------------------------------------------------
# B. the fused forms: in-kernel UCB, winners against the oracle's optimiser
# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class Fused:
  name: str
  route: int
  n: int
  pool: int
  batch: int
  steps: int
  norm: int = 0
  pert: int = xo.ADDITIVE
  sizes: tuple = ()
  d: int = 3


_FORMS = [('persistent', PERSISTENT, 40, 50, 25, 12), ('cooperative', COOPERATIVE, 130, 50, 25, 12),
          ('graph', GRAPH, 700, 1200, 600, 5)]
_OPTS = [('unnorm', dict(norm=2)), ('mult', dict(pert=xo.MULTIPLICATIVE)),
         ('cat-65-1000', dict(sizes=(65, 1000))), ('unnorm-mult-cat100', dict(norm=2, pert=xo.MULTIPLICATIVE, sizes=(100,))),
         ('cat-only-257', dict(sizes=(257, 3), d=0))]
FUSED = [Fused(f'{f}-{o}', r, n, p, b, s, **kw) for f, r, n, p, b, s in _FORMS for o, kw in _OPTS]


@pytest.mark.parametrize('c', FUSED, ids=lambda c: c.name)
def test_fused_forms_against_oracle(c):
  _, gp = _mods()
  dk = len(c.sizes)
  x, z = _trials(c.n, c.d, c.sizes, 17)
  y = (-np.sum((x - 0.7) ** 2, axis=1) if c.d else np.zeros(c.n)) + 0.05 * np.random.default_rng(5).normal(size=c.n)
  if dk:
    y -= 0.3 * (z[:, 0] != 1)
  po, pg = _params(c.d, dk)
  pred = go.precompute_predictive(po, x, y, z)
  prior_c, prior_z = x[:10], (z[:10] if dk else np.zeros((10, 0), np.int32))

  def score(xc, xz):
    mu, sd = go.predict(pred, xc, xz if dk else None)
    return mu + 1.8 * sd

  cfg_o = eo.EagleConfig(mutate_normalization_type=c.norm, perturbation_lower_bound=0.05)
  wc, wz, wr = xo.run_mixed(score, dim=c.d, sizes=np.asarray(c.sizes, np.int64), pool_size=c.pool, batch_size=c.batch,
                            max_evaluations=c.steps * c.batch, count=6, seed=5, cfg=cfg_o, perturbation_type=c.pert,
                            prior_c=prior_c, prior_z=prior_z)
  dev = gp.DeviceGP(0)
  try:
    dev.fit(x, y, pg, z=z)
    dev.set_int('eagle_perturbation', c.pert)
    acq = gp.Acquisition(1.8, False, 1.0)
    bc, bz, br = dev.eagle_run(_config(cfg_o, c.pool, c.batch, c.steps), acq, 6, 5, prior=prior_c,
                               prior_z=prior_z if dk else None, cat_sizes=c.sizes or None)
    route = dev.get_int('eagle_route')
    print(f'{c.name}: eagle_route {route}, best {br[0]:.6f}')
    assert route == c.route
    np.testing.assert_allclose(br, wr, rtol=0, atol=1e-9)
    np.testing.assert_allclose(bc, wc, rtol=0, atol=1e-9)
    np.testing.assert_array_equal(bz, wz)
  finally:
    dev.close()


# ---------------------------------------------------------------------------------------------------------------------
# C. random search, the C checks, the designers, VectorizedOptimizer
# ---------------------------------------------------------------------------------------------------------------------
def test_random_search_past_64_categories():
  _, gp = _mods()
  sizes, d, m = (65, 3, 1000), 2, 5000
  x, z = _trials(30, d, sizes, 8)
  y = -np.sum((x - 0.4) ** 2, axis=1) - 0.2 * (z[:, 2] % 7 != 3)
  po, pg = _params(d, len(sizes))
  pred = go.precompute_predictive(po, x, y, z)
  dev = gp.DeviceGP(0)
  try:
    dev.fit(x, y, pg, z=z)
    bx, bz, bs, bi = dev.random_search(m, gp.Acquisition(1.8, False, 1.0), 8, 21, cat_sizes=sizes)
  finally:
    dev.close()
  xs = eo.philox_uniform(21, eo.STREAM_RANDOM_POOL, 0, m * d).reshape(m, d)
  zs = eo.uniform_categories(eo.philox_uniform(21, eo.STREAM_RANDOM_POOL_CAT, 0, m * len(sizes)).reshape(m, -1),
                             np.asarray(sizes))
  assert zs[:, 2].max() > 64 and np.all(zs < np.asarray(sizes))
  np.testing.assert_array_equal(bz, zs[bi])
  np.testing.assert_array_equal(bx, xs[bi])
  mu, sd = go.predict(pred, xs, zs)
  want = mu + 1.8 * sd
  np.testing.assert_allclose(bs, want[bi], rtol=0, atol=1e-9)
  np.testing.assert_array_equal(np.sort(bi), np.sort(np.argsort(-want, kind='stable')[:8]))


def test_library_rejects_bad_option_values():
  _lib, gp = _mods()
  x, z = _trials(10, 2, (70,), 1)
  dev = gp.DeviceGP(0)
  try:
    dev.fit(x, np.arange(10.0), _params(2, 1)[1], z=z)
    for bad in (-1, 2):
      with pytest.raises(_lib.VzgpError):
        dev.set_int('eagle_perturbation', bad)
    cfg = _config(eo.EagleConfig(mutate_normalization_type=3), 25, 25, 2)
    with pytest.raises(_lib.VzgpError):
      dev.eagle_run(cfg, gp.Acquisition(1.8, False, 1.0), 1, 0, cat_sizes=(70,))
    with pytest.raises(_lib.VzgpError):
      dev.eagle_run(_config(eo.EagleConfig(), 25, 25, 2), gp.Acquisition(1.8, False, 1.0), 1, 0, cat_sizes=(0,))
  finally:
    dev.close()


def _cat_problem(n_metrics=1):
  from vizier_b200 import vz
  p = vz.ProblemStatement()
  p.search_space.root.add_float_param('x0', 0.0, 1.0)
  p.search_space.root.add_float_param('x1', -2.0, 2.0)
  p.search_space.root.add_categorical_param('c100', [f'a{i}' for i in range(100)])
  p.search_space.root.add_categorical_param('c1000', [f'b{i}' for i in range(1000)])
  for k in range(n_metrics):
    goal = vz.ObjectiveMetricGoal.MAXIMIZE if k == 0 else vz.ObjectiveMetricGoal.MINIMIZE
    p.metric_information.append(vz.MetricInformation(name=f'm{k}', goal=goal))
  return p


def _value(params, name):
  v = params[name]
  return getattr(v, 'value', v)


def _label(params, k):
  x0, x1 = float(_value(params, 'x0')), float(_value(params, 'x1'))
  v = -(x0 - 0.3) ** 2 - 0.1 * x1 ** 2 - 0.5 * (int(_value(params, 'c100')[1:]) % 10 != 4)
  v -= 0.3 * (int(_value(params, 'c1000')[1:]) % 100 != 17)
  return float(v if k == 0 else -v + 0.1 * x0)


@pytest.mark.parametrize('designer', ['gp_bandit', 'gp_ucb_pe', 'gp_ucb_pe_two_metrics'])
def test_designers_suggest_on_large_categorical_spaces(designer):
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit, gp_ucb_pe
  n_metrics = 2 if designer.endswith('two_metrics') else 1
  p = _cat_problem(n_metrics)
  d = (gp_bandit.VizierGPBandit(p, rng=2) if designer == 'gp_bandit' else gp_ucb_pe.VizierGPUCBPEBandit(p, rng=2))
  tid = 1
  for _ in range(4):
    sugg = d.suggest(2)
    assert len(sugg) == 2
    done = []
    for s in sugg:
      assert p.search_space.contains(s.parameters)
      assert _value(s.parameters, 'c100') in {f'a{i}' for i in range(100)}
      assert _value(s.parameters, 'c1000') in {f'b{i}' for i in range(1000)}
      t = s.to_trial(tid); tid += 1
      t.complete(vz.Measurement({f'm{k}': _label(t.parameters, k) for k in range(n_metrics)}))
      done.append(t)
    d.update(vz.CompletedTrials(done), vz.ActiveTrials())


def test_vectorized_optimizer_perturbation_type():
  """eagle_strategy_test.py:443-495: the same run with ADDITIVE and MULTIPLICATIVE perturbations (score -sum(x) over
  two continuous and two categorical features, 50 evaluations) ends with winners more than 0.1 apart.  The setting
  belongs to each optimiser's run: ADDITIVE after MULTIPLICATIVE on the same handle repeats the first run."""
  from vizier_b200 import optimizers as vb
  _, gp = _mods()
  x, z = _trials(6, 2, (3, 4), 2)
  dev = gp.DeviceGP(0)
  try:
    dev.fit(x, np.zeros(6), _params(2, 2)[1], z=z)     # alpha = 0: the UCB with coefficient 0 is exactly 0
    acq = gp.Acquisition(0.0, False, 1.0)

    def run(kind, stepped, evaluations=50):
      cfg = vb.EagleStrategyConfig(continuous_feature_perturbation_type=kind)
      opt = vb.VectorizedOptimizer(vb.VectorizedEagleStrategyFactory(eagle_config=cfg), 2, 2, 25, evaluations, (3, 4))
      prior = (lambda xc, xz: -np.sum(xc, axis=1)) if stepped else None
      return opt(dev, acq, count=4, prior_acquisition=prior).features

    ADD, MUL = vb.ContinuousFeaturePerturbationType.ADDITIVE, vb.ContinuousFeaturePerturbationType.MULTIPLICATIVE
    add, mul = run(ADD, True), run(MUL, True)
    assert add.shape == mul.shape == (4, 2)
    assert np.max(np.abs(add - mul)) > 0.1
    np.testing.assert_array_equal(run(ADD, True), add)
    # the fused loop reads the same setting: a model of -sum(x) scored in the loop
    dev.fit(x, -np.sum(x, axis=1), _params(2, 2)[1], z=z)
    acq = gp.Acquisition(1.8, False, 1.0)
    fa, fm = run(ADD, False, 250), run(MUL, False, 250)
    assert np.max(np.abs(fa - fm)) > 1e-3
    np.testing.assert_array_equal(run(ADD, False, 250), fa)
  finally:
    dev.close()
