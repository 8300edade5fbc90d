"""Multi-metric GP-UCB-PE on the host: the tests-side oracle against the single-metric and scalarised oracles, the
ordering of the three promising-region aggregations, the prior-only degenerate case, the designer's constructor
checks and the register budget of the combine kernel."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import gp_oracle as go
import pe_multi_oracle as pmo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'vizier_b200', 'csrc')
AGGS = (pmo.AVERAGE, pmo.UNION, pmo.INTERSECTION)


def _nvcc():
  for c in (os.environ.get('NVCC'), shutil.which('nvcc'),
            os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc')):
    if c and os.path.isfile(c) and os.access(c, os.X_OK):
      return c
  return None


def _makefile_flags():
  """NVFLAGS of vizier_b200/csrc/Makefile with $(ARCH) expanded and $(EXTRA) empty."""
  text = open(os.path.join(CSRC, 'Makefile')).read()
  var = {m.group(1): m.group(2).strip() for m in re.finditer(r'^(\w+)\s*:=\s*(.*)$', text, re.M)}
  flags = var['NVFLAGS'].replace('$(ARCH)', var['ARCH']).replace('$(EXTRA)', '')
  assert '$(' not in flags, flags
  return flags.split()


def _models(n, n_pending, d, m, seed):
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, d))
  y = np.stack([np.sin(3 * x[:, 0] + k) - np.sum((x - 0.2 * k) ** 2, axis=1) for k in range(m)], axis=1)
  ls2 = 0.4 * (1 + np.arange(d) / d)
  po = go.GPParams(1.1, ls2, 2e-3)
  pred_a = go.precompute_predictive(po, x, y if m > 1 else y[:, 0])
  xb = np.concatenate([x, rng.uniform(size=(n_pending, d))])
  pred_b = go.precompute_predictive(po, xb, np.zeros(n + n_pending))
  xs = rng.uniform(size=(300, d))
  xs[:4] = x[:4]
  return rng, x, y, xb, xs, pred_a, pred_b


@pytest.mark.parametrize('agg', AGGS)
def test_single_metric_pe_equals_ucb_pe_oracle(agg):
  """With one metric every aggregation reduces to PEScoreFunction's single-metric branch."""
  _, _, _, xb, xs, pred_a, pred_b = _models(30, 5, 3, 1, 1)
  thr_single = go.ucb_threshold(pred_a, pred_b, 1.8)
  thr = pmo.ucb_thresholds_multi(pred_a, pred_b, 1.8)
  assert thr.shape == (1,) and thr[0] == thr_single
  mask = np.array([True, False, True])
  r = 0.2
  want, aux_w = go.ucb_pe_score(pred_a, pred_b, xs, mode=1, threshold=thr_single, tr_dim_mask=mask, tr_rows=32,
                                trust_radius_value=r)
  got, aux = pmo.ucb_pe_multi_score(pred_a, pred_b, xs, mode=1, thresholds=thr, region_penalty=agg, tr_dim_mask=mask,
                                    tr_rows=32, trust_radius_value=r)
  assert np.any(want < -1e3) and np.any(want > -1e3)
  np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)
  np.testing.assert_array_equal(aux['mean'][:, 0], aux_w['mean'])
  np.testing.assert_array_equal(aux['stddev_from_all'], aux_w['stddev_from_all'])


@pytest.mark.parametrize('m', [2, 3])
def test_ucb_mode_is_scalarized_ucb_then_trust_region(m):
  rng, _, y, xb, xs, pred_a, pred_b = _models(40, 6, 4, m, 2)
  w = np.abs(rng.normal(size=(100, m))); w /= np.linalg.norm(w, axis=1, keepdims=True)
  ref = go.hv_reference_point(y)
  best = go.hv_max_scalarized(y, w, ref)
  mask = np.ones(4, bool)
  r = 0.15
  mu, _ = go.predict(pred_a, xs)
  _, sd_b = go.predict(pred_b, xs)
  dist = go.min_linf_distance(xs, xb[:42], mask)
  for floor in (best, None):
    raw = go.scalarized_ucb(mu, sd_b, w, ref, floor, 1.8)
    want = np.where((dist < r) | (r > 0.5), raw, -1e4 - dist)
    got, _ = pmo.ucb_pe_multi_score(pred_a, pred_b, xs, mode=0, weights=w, reference_point=ref, max_scalarized=floor,
                                    tr_rows=42, trust_radius_value=r)
    np.testing.assert_array_equal(got, want)
    assert np.any(got < -1e3) and np.any(got > -1e3)
  # the floor only ever raises the score
  hi, _ = pmo.ucb_pe_multi_score(pred_a, pred_b, xs, mode=0, weights=w, reference_point=ref, max_scalarized=best,
                                 use_trust_region=False)
  lo, _ = pmo.ucb_pe_multi_score(pred_a, pred_b, xs, mode=0, weights=w, reference_point=ref, use_trust_region=False)
  assert np.all(hi >= lo) and np.any(hi > lo)


@pytest.mark.parametrize('m', [2, 3, 8])
def test_intersection_le_average_le_union(m):
  _, _, _, _, xs, pred_a, pred_b = _models(35, 3, 3, m, 3)
  thr = pmo.ucb_thresholds_multi(pred_a, pred_b)
  s = {agg: pmo.ucb_pe_multi_score(pred_a, pred_b, xs, mode=1, thresholds=thr, region_penalty=agg,
                                   use_trust_region=False)[0] for agg in AGGS}
  assert np.all(s[pmo.INTERSECTION] <= s[pmo.AVERAGE] + 1e-12)
  assert np.all(s[pmo.AVERAGE] <= s[pmo.UNION] + 1e-12)
  assert np.any(s[pmo.INTERSECTION] < s[pmo.UNION])


@pytest.mark.parametrize('agg', AGGS)
def test_prior_only_score_is_stddev_of_b(agg):
  """No completed trial: model A is the prior (mean 0, stddev sqrt(sf2 + sn2)) and every threshold is the prior mean 0,
  so each penalty is min(0.5 stddev_A, 0) = 0 and the PE score is stddev_B."""
  rng = np.random.default_rng(4)
  sd_b = rng.uniform(0.1, 1.0, size=50)
  m = 3
  got = pmo.combine(np.zeros((50, m)), np.full(50, np.sqrt(1.1 + 2e-3)), sd_b, mode=1, thresholds=np.zeros(m),
                    region_penalty=agg)
  np.testing.assert_allclose(got, sd_b, rtol=1e-15, atol=0)


def _problem(n_metrics):
  from vizier_b200 import vz
  p = vz.ProblemStatement()
  for i in range(2):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  for k in range(n_metrics):
    goal = vz.ObjectiveMetricGoal.MINIMIZE if k == 1 else vz.ObjectiveMetricGoal.MAXIMIZE
    p.metric_information.append(vz.MetricInformation(name=f'metric{k}', goal=goal))
  return p


def test_designer_constructor_defaults_and_errors():
  from vizier_b200.designers import gp_ucb_pe as ucbpe
  cfg = ucbpe.UCBPEConfig()
  assert cfg.multimetric_promising_region_penalty_type == ucbpe.MultimetricPromisingRegionPenaltyType.AVERAGE
  assert cfg.multitask_type == 'INDEPENDENT'
  for penalty in ucbpe.MultimetricPromisingRegionPenaltyType:
    ucbpe.VizierGPUCBPEBandit(_problem(2), rng=1,
                              config=ucbpe.UCBPEConfig(multimetric_promising_region_penalty_type=penalty))
  ucbpe.VizierGPUCBPEBandit(_problem(8), rng=1)
  with pytest.raises(ValueError):
    ucbpe.VizierGPUCBPEBandit(_problem(2), config=ucbpe.UCBPEConfig(optimize_set_acquisition_for_exploration=True))
  with pytest.raises(NotImplementedError):
    ucbpe.VizierGPUCBPEBandit(_problem(2), mixes_linear_kernel=True)
  with pytest.raises(NotImplementedError):
    ucbpe.VizierGPUCBPEBandit(_problem(2), ensemble_size=2)
  with pytest.raises(NotImplementedError):
    ucbpe.VizierGPUCBPEBandit(_problem(2), config=ucbpe.UCBPEConfig(multitask_type='SEPARABLE_NORMAL_TASK_KERNEL_PRIOR'))
  with pytest.raises(NotImplementedError):
    ucbpe.VizierGPUCBPEBandit(_problem(9))
  with pytest.raises(ValueError):
    ucbpe.VizierGPUCBPEBandit(_problem(2), config=ucbpe.UCBPEConfig(multimetric_promising_region_penalty_type='max'))
  # one metric: the set-PE batches and the linear kernel stay available
  ucbpe.VizierGPUCBPEBandit(_problem(1), config=ucbpe.UCBPEConfig(optimize_set_acquisition_for_exploration=True))
  ucbpe.VizierGPUCBPEBandit(_problem(1), mixes_linear_kernel=True)


def test_region_penalty_codes_match_the_header():
  from vizier_b200 import _lib
  from vizier_b200.designers import gp_ucb_pe as ucbpe
  text = open(os.path.join(ROOT, 'include', 'vzgp.h')).read()
  codes = {k: int(v) for k, v in re.findall(r'VZGP_REGION_(\w+)\s*=\s*(\d+)', text)}
  assert codes == {'AVERAGE': _lib.REGION_AVERAGE, 'UNION': _lib.REGION_UNION, 'INTERSECTION': _lib.REGION_INTERSECTION}
  assert codes == {'AVERAGE': pmo.AVERAGE, 'UNION': pmo.UNION, 'INTERSECTION': pmo.INTERSECTION}
  for member, code in ucbpe._REGION_PENALTY_CODE.items():
    assert codes[member.name] == code
  fields = [f for f, _ in _lib.PeMultiParams._fields_]
  body = re.search(r'typedef struct vzgp_pe_multi_params \{(.*?)\} vzgp_pe_multi_params;', text, re.S).group(1)
  body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
  declared = [re.findall(r'(\w+)\s*$', d.strip())[0] for piece in body.split(';') if piece.strip()
              for d in piece.split(',')]
  assert fields == declared


@pytest.fixture(scope='module')
def multi_ptxas_report(tmp_path_factory):
  nvcc = _nvcc()
  if nvcc is None:
    pytest.skip('nvcc not found')
  out = tmp_path_factory.mktemp('multi_ptxas')
  cmd = [nvcc] + _makefile_flags() +['-Xptxas', '-v', '-c', os.path.join(CSRC, 'multi.cu'), '-o', str(out / 'multi.o')]
  res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
  assert res.returncode == 0, res.stderr[-4000:]
  report = {}
  for m in re.finditer(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", res.stderr):
    report[m.group(1)] = {'stack': int(m.group(2)), 'spill_stores': int(m.group(3)), 'spill_loads': int(m.group(4))}
  return report


@pytest.mark.parametrize('kernel', ['k_pe_multi_combine', 'k_scalarize'])
def test_combine_kernels_have_no_spills_and_no_stack_frame(multi_ptxas_report, kernel):
  names = [n for n in multi_ptxas_report if re.match(rf'_ZN4vzgp{len(kernel)}{kernel}E', n)]
  assert len(names) == 1, sorted(multi_ptxas_report)
  r = multi_ptxas_report[names[0]]
  assert r == {'stack': 0, 'spill_stores': 0, 'spill_loads': 0}, r
