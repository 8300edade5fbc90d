"""CPU checks of the q-acquisition oracle (tests/qacq_oracle.py::qacq_score and its Monte Carlo stage) and of what
the designer rejects at construction.

The oracle restates csrc/score_q.cu draw for draw, so the GPU tests compare the kernels with it; here it is pinned
against closed forms: at q = 1 QEI / QPI / QUCB are Monte Carlo estimates of EI (exploration 0.01), PI and UCB, and
with independent points E[max] has a one-dimensional integral.  Also: the reference's own known answers
(acquisitions_test.py:279-335) on tfd.Normal moments, the jitter ladder, and the ptxas report of the two kernels."""
import math
import os

import numpy as np
import pytest
import scipy.integrate as si
import scipy.stats as st

import qacq_oracle as qo

S = 20000


def _one_point(mu, sd, kind, **kw):
  return qo.qacq_from_moments(np.array([[[mu]]]), np.array([[[[sd * sd]]]]), kind=kind, **kw)[0][0]


def _mc_se(values_sd, n):
  return values_sd / math.sqrt(n)


@pytest.mark.parametrize('mu,sd,best', [(0.1, 1.0, 0.2), (-0.3, 0.4, 0.1), (1.2, 0.2, 1.0)])
def test_q1_matches_analytic_ei_pi_ucb_within_4_standard_errors(mu, sd, best):
  imp = mu - best - qo.QEI_EXPLORATION
  ei = imp * st.norm.cdf(imp / sd) + sd * st.norm.pdf(imp / sd)
  ei2 = (imp * imp + sd * sd) * st.norm.cdf(imp / sd) + imp * sd * st.norm.pdf(imp / sd)
  got = _one_point(mu, sd, qo.QACQ_QEI, best_label=best, num_samples=S, seed=5)
  assert abs(got - ei) < 4 * _mc_se(math.sqrt(ei2 - ei * ei), S)
  pi = st.norm.cdf((mu - best) / sd)
  got = _one_point(mu, sd, qo.QACQ_QPI, best_label=best, num_samples=S, seed=6)
  assert abs(got - pi) < 4 * _mc_se(math.sqrt(pi * (1 - pi)), S)
  # QUCB(c sqrt(pi / 2)) = UCB(c): c sqrt(pi/2) |z| sd has mean c sd and variance c^2 sd^2 (pi/2 - 1)
  c = 1.8
  got = _one_point(mu, sd, qo.QACQ_QUCB, coefficient=c * math.sqrt(math.pi / 2), num_samples=S, seed=7)
  assert abs(got - (mu + c * sd)) < 4 * _mc_se(c * sd * math.sqrt(math.pi / 2 - 1), S)


def test_q2_independent_points_match_expected_max_by_integration():
  mu, sd = np.array([0.2, -0.1]), np.array([0.5, 0.8])
  cdf = lambda t: st.norm.cdf((t - mu[0]) / sd[0]) * st.norm.cdf((t - mu[1]) / sd[1])
  lo, hi = -10.0, 10.0
  emax = hi - si.quad(cdf, lo, hi, limit=200)[0] + lo * cdf(lo)
  emax2 = 2 * si.quad(lambda t: t * (1 - cdf(t)), 0, hi, limit=200)[0] - 2 * si.quad(lambda t: t * cdf(t), lo, 0, limit=200)[0]
  cov = np.diag(sd * sd)[None, None]
  got = qo.qacq_from_moments(mu[None, None], cov, kind=qo.QACQ_QEI, best_label=-np.inf, num_samples=S, seed=9)[0][0]
  assert abs(got - emax) < 4 * _mc_se(math.sqrt(emax2 - emax * emax), S)
  # QEI with a finite best: E[max(max_j f_j - best - 0.01, 0)]
  best = 0.3
  t0 = best + qo.QEI_EXPLORATION
  qei = si.quad(lambda t: 1 - cdf(t), t0, hi, limit=200)[0]
  got = qo.qacq_from_moments(mu[None, None], cov, kind=qo.QACQ_QEI, best_label=best, num_samples=S, seed=10)[0][0]
  assert abs(got - qei) < 4 * _mc_se(0.6, S)
  # QPI: P(max_j f_j > best)
  qpi = 1 - cdf(best)
  got = qo.qacq_from_moments(mu[None, None], cov, kind=qo.QACQ_QPI, best_label=best, num_samples=S, seed=11)[0][0]
  assert abs(got - qpi) < 4 * _mc_se(math.sqrt(qpi * (1 - qpi)), S)


def test_reference_known_answers_on_normal_moments():
  """acquisitions_test.py:279-335: QEI of N(0.1, 1) with best 0.2 is 0.346 (atol 1e-2 there); QPI agrees with PI and
  QUCB(c sqrt(pi / 2)) with UCB(c) within 1e-2 at 5000 samples."""
  qei = _one_point(0.1, 1.0, qo.QACQ_QEI, best_label=0.2, num_samples=5000, seed=0)
  assert abs(qei - 0.346) < 2e-2
  mu, sd, best = np.array([0.3, -0.2, 1.1]), np.array([0.9, 0.5, 0.3]), 0.1
  for j in range(3):
    qpi = _one_point(mu[j], sd[j], qo.QACQ_QPI, best_label=best, num_samples=5000, seed=1)
    assert abs(qpi - st.norm.cdf((mu[j] - best) / sd[j])) < 2.5e-2
    qucb = _one_point(mu[j], sd[j], qo.QACQ_QUCB, coefficient=1.8 * math.sqrt(math.pi / 2), num_samples=5000, seed=2)
    assert abs(qucb - (mu[j] + 1.8 * sd[j])) < 4 * _mc_se(1.8 * sd[j] * math.sqrt(math.pi / 2 - 1), 5000)


def test_jitter_ladder_retries_then_gives_up():
  ok_after_retry = np.array([[1.0, 1.0], [1.0, 1.0 - 5e-5]])     # eigenvalue about -2.5e-5: the first shift fixes it
  hopeless = np.array([[1.0, 0.0], [0.0, -10.0]])
  l, ok = qo.qacq_cholesky(np.stack([ok_after_retry, hopeless, np.eye(2)]))
  assert ok.tolist() == [True, False, True]
  np.testing.assert_allclose(l[0] @ l[0].T, ok_after_retry + 1e-4 * np.eye(2), rtol=1e-12)
  assert np.isnan(l[1]).all()
  np.testing.assert_array_equal(l[2], np.eye(2))
  score = qo.qacq_from_moments(np.zeros((1, 3, 2)), np.stack([ok_after_retry, hopeless, np.eye(2)])[None],
                               kind=qo.QACQ_QEI, best_label=0.0, num_samples=10, seed=0)[0]
  assert np.isfinite(score[[0, 2]]).all() and np.isnan(score[1])


def test_draws_depend_on_position_not_set_index():
  mean = np.tile(np.array([0.1, 0.3, -0.2]), (1, 4, 1))
  cov = np.tile(0.5 * np.eye(3) + 0.1, (1, 4, 1, 1))
  s = qo.qacq_from_moments(mean, cov, kind=qo.QACQ_QEI, best_label=0.0, num_samples=50, seed=4, period=2)[0]
  assert s[0] == s[2] and s[1] == s[3] and s[0] != s[1]


def test_box_muller_normals_are_standard_normal():
  z = qo.qacq_normals(123, np.arange(200_000, dtype=np.uint64))
  assert abs(z.mean()) < 0.01 and abs(z.std() - 1) < 0.01
  assert st.kstest(z, 'norm').pvalue > 1e-3


def test_member_draw_mixes_members():
  """E = 2 members with disjoint means: the mixture's QUCB-free expectation E[max f] lands between them."""
  mean = np.array([[[0.0]], [[10.0]]])
  cov = np.full((2, 1, 1, 1), 1e-6)
  got = qo.qacq_from_moments(mean, cov, kind=qo.QACQ_QEI, best_label=-np.inf, num_samples=4000, seed=8)[0][0]
  assert abs(got - 5.0) < 4 * 5.0 / math.sqrt(4000)


# ---------------------------------------------------------------- designer construction (no GPU needed)
def _problem():
  from vizier_b200 import vz
  p = vz.ProblemStatement()
  p.search_space.root.add_float_param('x0', 0.0, 1.0)
  p.search_space.root.add_float_param('x1', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='obj', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  return p


def test_designer_construction_accepts_and_rejects():
  from vizier_b200 import acquisitions as acq
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit
  qei = acq.bayesian_scoring_function_factory(lambda d: acq.QEI(acq.get_best_labels(d.labels)))
  qucb = acq.bayesian_scoring_function_factory(lambda d: acq.QUCB())
  qpi = acq.bayesian_scoring_function_factory(lambda d: acq.QPI(acq.get_best_labels(d.labels), num_samples=50))
  for f in (qei, qucb, qpi):
    gp_bandit.VizierGPBandit(_problem(), scoring_function_factory=f, scoring_function_is_parallel=True)
  # a pointwise acquisition with the parallel flag, and the default UCB
  with pytest.raises(NotImplementedError):
    gp_bandit.VizierGPBandit(_problem(), scoring_function_is_parallel=True,
                             scoring_function_factory=acq.bayesian_scoring_function_factory(lambda d: acq.UCB()))
  with pytest.raises(NotImplementedError):
    gp_bandit.VizierGPBandit(_problem(), scoring_function_is_parallel=True)
  # a q-acquisition without the flag
  with pytest.raises(NotImplementedError):
    gp_bandit.VizierGPBandit(_problem(), scoring_function_factory=qei)
  # multi-metric
  p = _problem()
  p.metric_information.append(vz.MetricInformation(name='obj2', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  with pytest.raises(NotImplementedError):
    gp_bandit.VizierGPBandit(p, scoring_function_factory=qei, scoring_function_is_parallel=True)
  # priors
  d = gp_bandit.VizierGPBandit(_problem(), scoring_function_factory=qei, scoring_function_is_parallel=True)
  with pytest.raises(NotImplementedError):
    d.set_priors([])


def test_lowering():
  from vizier_b200 import _lib
  from vizier_b200 import acquisitions as acq
  q = acq.lower_parallel_acquisition(acq.QEI(np.array([0.5]), num_samples=77), use_trust_region=True, trust_radius=0.3)
  assert (q.kind, q.best_label, q.num_samples, q.use_trust_region, q.trust_radius) == (_lib.QACQ_QEI, 0.5, 77, True, 0.3)
  q = acq.lower_parallel_acquisition(acq.QPI(acq.get_best_labels(acq.PaddedArray(np.zeros((0, 1))))))
  assert q.kind == _lib.QACQ_QPI and q.best_label == -np.inf
  q = acq.lower_parallel_acquisition(acq.QUCB(2.5))
  assert q.kind == _lib.QACQ_QUCB and q.coefficient == 2.5 and q.num_samples == 100
  with pytest.raises(NotImplementedError):
    acq.lower_parallel_acquisition(acq.EI(0.0))
  with pytest.raises(NotImplementedError):
    acq.lower_acquisition(acq.QEI(0.0))


# ---------------------------------------------------------------- ptxas report of score_q.cu
def test_qacq_kernels_compile_without_spills(tmp_path):
  import re
  import shutil
  import subprocess
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  csrc = os.path.join(root, 'vizier_b200', 'csrc')
  nvcc = next((c for c in (os.environ.get('NVCC'), shutil.which('nvcc'),
                           os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc'))
               if c and os.path.isfile(c) and os.access(c, os.X_OK)), None)
  if nvcc is None:
    pytest.skip('nvcc not found')
  text = open(os.path.join(csrc, 'Makefile')).read()
  var = {m.group(1): m.group(2).strip() for m in re.finditer(r'^(\w+)\s*:=\s*(.*)$', text, re.M)}
  flags = var['NVFLAGS'].replace('$(ARCH)', var['ARCH']).replace('$(EXTRA)', '').split()
  res = subprocess.run([nvcc] + flags + ['-Xptxas', '-v', '-c', os.path.join(csrc, 'score_q.cu'), '-o',
                        str(tmp_path / 'score_q.o')], cwd=csrc, capture_output=True, text=True)
  assert res.returncode == 0, res.stderr[-4000:]
  report = {m.group(1): (int(m.group(2)), int(m.group(3)), int(m.group(4))) for m in re.finditer(
      r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
      res.stderr)}
  for name in ('_ZN4vzgp14k_qset_momentsENS_8QMomArgsE', '_ZN4vzgp9k_qacq_mcENS_7QMcArgsE'):
    assert name in report, sorted(report)
    assert report[name] == (0, 0, 0), (name, report[name])
