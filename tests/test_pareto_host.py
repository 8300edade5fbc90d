"""CPU tests of the Pareto / hypervolume feature: the NumPy oracle against the reference's own known answers
(tests/golden/pareto_known_answers.json), the host logic of `multimetric.ParetoFrontier` driven by the oracle, the
argument checks of `vizier_b200.multimetric` (raised before any device work), the agreement of the header, the ctypes
table and the Makefile, and the ptxas report of pareto.cu."""
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import pareto_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'vizier_b200', 'csrc')
G = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'pareto_known_answers.json')))
ENTRY_POINTS = {'vzgp_pareto_optimal_against': 8, 'vzgp_pareto_rank': 5, 'vzgp_cum_hypervolume_origin': 7}


# ---------------------------------------------------------------------------------------------------------------------
# the oracle reproduces the reference's known answers
# ---------------------------------------------------------------------------------------------------------------------
def test_oracle_pareto_rank_known_answer():
  g = G['pareto_rank']
  np.testing.assert_array_equal(po.pareto_rank(np.array(g['ys'])), g['rank'])
  # rank 0 is the frontier
  np.testing.assert_array_equal(po.is_frontier(np.array(g['ys'])), np.array(g['rank']) == 0)


def test_oracle_frontier_known_answers():
  g = G['is_pareto_optimal']
  pts = np.array(g['points'], dtype=float)
  np.testing.assert_array_equal(po.is_frontier(pts), g['optimal'])
  np.testing.assert_array_equal(po.is_frontier(np.vstack([pts, g['added']])), g['optimal_with_added'])
  u = G['update_pareto_optimal']
  both = np.append(np.array(u['current'], float), np.array(u['incremental'], float), axis=0)
  np.testing.assert_array_equal(po.is_frontier(both).nonzero()[0], u['indices'])


def test_oracle_optimal_against_known_answers():
  g = G['is_pareto_optimal_against']
  pts, against = np.array(g['points'], float), np.array(g['against'], float)
  np.testing.assert_array_equal(po.is_pareto_optimal_against(pts, against, strict=True), g['strict'])
  np.testing.assert_array_equal(po.is_pareto_optimal_against(pts, against, strict=False), g['non_strict'])


def test_oracle_nan_and_inf_rows():
  ys = np.array([[np.nan, 5.0], [0.0, 0.0], [np.inf, np.inf], [-np.inf, 1.0], [1.0, np.nan]])
  # the NaN rows are never dominated and dominate nothing; (inf, inf) dominates every row without a NaN
  np.testing.assert_array_equal(po.is_frontier(ys), [True, False, True, False, True])
  np.testing.assert_array_equal(po.pareto_rank(ys), [0, 1, 0, 1, 0])
  # a row does not strictly dominate itself, but does weakly
  np.testing.assert_array_equal(po.is_pareto_optimal_against(ys[2:3], ys[2:3], strict=False), [False])
  np.testing.assert_array_equal(po.is_pareto_optimal_against(ys[2:3], ys[2:3], strict=True), [True])


def test_oracle_cum_hypervolume_matches_its_definition():
  rng = np.random.default_rng(0)
  pts, vec = rng.uniform(0.1, 2.0, size=(37, 3)), rng.uniform(0.1, 1.0, size=(700, 3))
  want = np.mean(np.maximum.accumulate(np.min(pts[None] / vec[:, None], axis=2), axis=1) ** 3, axis=0)
  np.testing.assert_allclose(po.cum_hypervolume_origin(pts, vec), want, rtol=1e-13)
  pts[5, 1] = np.nan
  got = po.cum_hypervolume_origin(pts, vec)
  assert np.all(np.isfinite(got[:5])) and np.all(np.isnan(got[5:]))


# ---------------------------------------------------------------------------------------------------------------------
# ParetoFrontier's host logic, with the oracle as its cumulative-hypervolume base
# ---------------------------------------------------------------------------------------------------------------------
def _frontier(points, origin, **kw):
  from vizier_b200 import multimetric
  return multimetric.ParetoFrontier(np.asarray(points, float), np.asarray(origin, float),
                                    cum_hypervolume_base=po.cum_hypervolume_origin, **kw)


def test_pareto_frontier_two_point_identity():
  g = G['two_point_hypervolume']
  np.random.seed(0)
  for c in g['cases']:
    pf = _frontier([[c['x'], c['y']], [c['y'], c['x']]], g['origin'])
    assert abs(float(pf.hypervolume()) - c['expected']) <= g['delta'], c


def test_pareto_frontier_cumulative_curve():
  np.random.seed(1)
  points = np.random.normal(size=(100, 4))
  pf = _frontier(points, np.zeros(4))
  cum = pf.hypervolume(is_cumulative=True)
  assert len(cum) == len(points)
  assert np.all(np.diff(cum) >= 0)
  assert cum[-1] == pytest.approx(float(pf.hypervolume()))
  # additional points are appended after the frontier's own
  extra = np.random.normal(size=(10, 4))
  assert len(pf.hypervolume(additional_points=extra, is_cumulative=True)) == 110


def test_pareto_frontier_dimension_mismatch():
  g = G['dimension_mismatch']
  with pytest.raises(ValueError, match=g['message']):
    _frontier(g['points'], g['origin_3d'])
  pf = _frontier(g['points'], g['origin'])
  with pytest.raises(ValueError, match=g['message']):
    pf.hypervolume(additional_points=np.array(g['origin_3d'], float)[..., np.newaxis])


# ---------------------------------------------------------------------------------------------------------------------
# argument checks of the Python layer (no device needed: they raise before any)
# ---------------------------------------------------------------------------------------------------------------------
def test_python_argument_errors():
  torch = pytest.importorskip('torch')
  from vizier_b200 import multimetric as mm
  a2, a3 = np.zeros((4, 2)), np.zeros((4, 3))
  with pytest.raises(ValueError, match='points have 2 metrics but against has 3'):
    mm.is_pareto_optimal_against(a2, a3, strict=True)
  with pytest.raises(ValueError, match='points have 2 metrics but the vectors have 3'):
    mm.cum_hypervolume_origin(a2, a3)
  with pytest.raises(ValueError, match='2-D'):
    mm.is_frontier(np.zeros(5))
  with pytest.raises(ValueError, match='2-D'):
    mm.pareto_rank(np.zeros((2, 3, 4)))
  with pytest.raises(ValueError, match='metrics'):
    mm.pareto_rank(np.zeros((3, 65)))
  with pytest.raises(ValueError, match='metrics'):
    mm.get_frontier(np.zeros((3, 0)))
  with pytest.raises(TypeError, match='float64 CUDA'):
    mm.pareto_rank(torch.zeros((3, 2), dtype=torch.float64))
  with pytest.raises(TypeError):
    mm.is_pareto_optimal_against(a2, a2)   # strict is keyword-only and required, as in the reference


# ---------------------------------------------------------------------------------------------------------------------
# header, ctypes table and Makefile
# ---------------------------------------------------------------------------------------------------------------------
def test_header_ctypes_and_makefile_agree():
  from vizier_b200 import _lib
  header = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'vzgp.h')).read(), flags=re.S)
  for name, nargs in ENTRY_POINTS.items():
    m = re.search(rf'\bint\s+{name}\s*\(([^)]*)\)\s*;', header)
    assert m, name
    assert len(m.group(1).split(',')) == nargs, name
    assert len(_lib.SIGNATURES[name][1]) == nargs, name
  text = open(os.path.join(CSRC, 'Makefile')).read()
  srcs = re.search(r'^SRCS\s*:=\s*(.*)$', text, re.M).group(1).split()
  assert 'pareto.cu' in srcs
  assert re.search(r'^int vzgp_pareto_rank\(', open(os.path.join(CSRC, 'c_abi.cu')).read(), re.M)


def _nvcc():
  for c in (os.environ.get('NVCC'), shutil.which('nvcc'),
            os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc')):
    if c and os.path.isfile(c) and os.access(c, os.X_OK):
      return c
  return None


def test_pareto_kernels_have_no_spills_or_stack_frame(tmp_path):
  nvcc = _nvcc()
  if nvcc is None:
    pytest.skip('nvcc not found')
  text = open(os.path.join(CSRC, 'Makefile')).read()
  var = {m.group(1): m.group(2).strip() for m in re.finditer(r'^(\w+)\s*:=\s*(.*)$', text, re.M)}
  flags = var['NVFLAGS'].replace('$(ARCH)', var['ARCH']).replace('$(EXTRA)', '').split()
  res = subprocess.run([nvcc] + flags + ['-Xptxas', '-v', '-c', os.path.join(CSRC, 'pareto.cu'), '-o',
                        str(tmp_path / 'pareto.o')], cwd=CSRC, capture_output=True, text=True)
  assert res.returncode == 0, res.stderr[-4000:]
  found = 0
  for m in re.finditer(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", res.stderr):
    if 'k_pareto_dominance' in m.group(1) or 'k_cum_hypervolume' in m.group(1):
      found += 1
      assert (int(m.group(2)), int(m.group(3)), int(m.group(4))) == (0, 0, 0), m.group(0)
  assert found == 16, res.stderr[-2000:]   # 7 metric widths x (frontier, rank), the hypervolume and its reduction
