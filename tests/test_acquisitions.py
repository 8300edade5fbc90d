"""CPU checks of the acquisition functions a VizierGPBandit can score with: the oracle and the host lowering
(evaluated with NumPy) against the reference's own known answers (acquisitions_test.py), the lowering of every
preset, and the NotImplementedError of what the device does not evaluate."""
import json
import os

import numpy as np
import pytest

import acq_oracle as ao
from vizier_b200 import _lib
from vizier_b200 import acquisitions as acq
from vizier_b200 import vz
from vizier_b200.designers import gp_bandit

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, 'golden', 'acquisition_known_answers.json')))


def _data(labels):
  return acq.ModelData(features=None, labels=acq.PaddedArray.as_padded(np.asarray(labels, np.float64)))


def _build(case):
  kind = case['acquisition']
  if kind == 'UCB':
    return acq.UCB(case['coefficient'])
  if kind == 'LCB':
    return acq.LCB(case['coefficient'])
  if kind in ('EI', 'PI'):
    best = acq.get_best_labels(acq.PaddedArray.as_padded(np.asarray(case['labels'])))
    return acq.EI(best) if kind == 'EI' else acq.PI(best)
  return getattr(acq.AcquisitionTrustRegion, kind)(_data(case['labels']))


@pytest.mark.parametrize('case', GOLDEN['cases'], ids=lambda c: c['name'])
def test_known_answers(case):
  fn = _build(case)
  mu, sd = np.array([GOLDEN['mean']]), np.array([GOLDEN['stddev']])
  tol = case.get('delta', 5e-8)
  got_oracle = float(ao.evaluate(fn, mu, sd)[0])
  got_lowered = float(ao.evaluate_spec(acq.lower_acquisition(fn), mu, sd)[0])
  assert abs(got_oracle - case['expected']) <= tol, got_oracle
  assert abs(got_lowered - case['expected']) <= tol, got_lowered


def test_lowering_matches_oracle_on_a_grid():
  rng = np.random.default_rng(0)
  mu = rng.normal(size=2000)
  sd = np.abs(rng.normal(size=2000))
  sd[:50] = 0.0                                   # the clamped-variance rule
  labels = rng.normal(size=(17, 1))
  fns = [acq.UCB(1.3), acq.LCB(0.7), acq.EI(acq.get_best_labels(_data(labels).labels)),
         acq.PI(acq.get_best_labels(_data(labels).labels))]
  fns += [getattr(acq.AcquisitionTrustRegion, p)(_data(labels))
          for p in ('default_ucb_pi', 'default_ucb_lcb', 'default_ucb_lcb_wide', 'default_ucb_lcb_delay_tr')]
  for fn in fns:
    want = ao.evaluate(fn, mu, sd)
    got = ao.evaluate_spec(acq.lower_acquisition(fn), mu, sd)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-13, err_msg=type(fn).__name__)
  # sd = 0: EI = max(imp, 0), PI = (imp > 0)
  best = float(np.max(labels))
  np.testing.assert_array_equal(ao.ei(mu[:50], sd[:50], best), np.maximum(mu[:50] - best - 0.01, 0.0))
  np.testing.assert_array_equal(ao.pi(mu[:50], sd[:50], best), (mu[:50] - best > 0).astype(float))


def test_lowering_resolves_threshold_and_delay():
  f = acq.lower_acquisition(acq.AcquisitionTrustRegion.default_ucb_lcb(_data([[1.0], [2.0], [6.0]])))
  assert f.thresholding.kind == _lib.ACQ_LCB and f.threshold == 2.0   # min(mean 3, median 2)
  assert f.main.kind == _lib.ACQ_UCB and f.main.coefficient == 1.8 and f.bad_acq_value == -1e4
  # at most apply_tr_after labels: main only
  f = acq.lower_acquisition(acq.AcquisitionTrustRegion.default_ucb_lcb_delay_tr(_data([[1.0]] * 5)))
  assert f.thresholding is None
  assert acq.lower_acquisition(acq.AcquisitionTrustRegion.default_ucb_lcb_delay_tr(_data([[1.0]] * 6))).thresholding
  # no labels at all: the threshold is NaN
  assert acq.lower_acquisition(acq.AcquisitionTrustRegion.default_ucb_pi(_data(np.zeros((0, 1))))).thresholding is None
  f = acq.lower_acquisition(acq.AcquisitionTrustRegion.default_ucb_pi(_data([[3.0]])))
  assert f.thresholding.kind == _lib.ACQ_PI and f.threshold == 0.3 and f.thresholding.best_label == 3.0
  e = acq.lower_acquisition(acq.EI(acq.get_best_labels(_data([[0.5], [0.25]]).labels)))
  assert (e.main.kind, e.main.best_label, e.main.exploration) == (_lib.ACQ_EI, 0.5, 0.01)
  # an empty study: best label -inf, scored by the posterior mean
  e = acq.lower_acquisition(acq.EI(acq.get_best_labels(_data(np.zeros((0, 1))).labels)))
  assert (e.main.kind, e.main.coefficient) == (_lib.ACQ_UCB, 0.0)


def test_ctypes_struct_layout():
  import ctypes as C
  assert C.sizeof(_lib.AcqTerm) == 32
  assert _lib.AcqFn.thresholding.offset == 40 and _lib.AcqFn.threshold.offset == 72 and C.sizeof(_lib.AcqFn) == 88


class QEI:      # stands for an acquisition the device does not evaluate
  best_labels = 0.0


def _problem():
  p = vz.ProblemStatement()
  for i in range(2):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='obj', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  return p


@pytest.mark.parametrize('factory', [
    acq.bayesian_scoring_function_factory(lambda d: QEI()),
    acq.bayesian_scoring_function_factory(lambda d: acq.AcquisitionTrustRegion(
        acq.UCB(), QEI(), bad_acq_value=-1e4, labels=d.labels)),
    lambda data, predictive, cfv, use_tr: (lambda xs: xs),
])
def test_unsupported_scoring_functions_raise_at_construction(factory):
  with pytest.raises(NotImplementedError):
    gp_bandit.VizierGPBandit(_problem(), scoring_function_factory=factory)


def test_parallel_scoring_raises_and_supported_factories_construct():
  with pytest.raises(NotImplementedError):
    gp_bandit.VizierGPBandit(_problem(), scoring_function_is_parallel=True)
  for f in (lambda d: acq.EI(acq.get_best_labels(d.labels)), lambda d: acq.PI(acq.get_best_labels(d.labels)),
            lambda d: acq.LCB(), acq.AcquisitionTrustRegion.default_ucb_pi, acq.AcquisitionTrustRegion.default_ucb_lcb,
            acq.AcquisitionTrustRegion.default_ucb_lcb_wide, acq.AcquisitionTrustRegion.default_ucb_lcb_delay_tr):
    gp_bandit.VizierGPBandit(_problem(), scoring_function_factory=acq.bayesian_scoring_function_factory(f))
