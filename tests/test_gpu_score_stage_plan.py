"""k_score's phase-1 shared-memory plan on both sides of each dc where it switches, against the oracle.

Phase 1 aliases the operand ring with the K* staging buffers (TMA stores), the candidates and three trial buffers.
Three staging buffers fit up to Dc = 45, two up to Dc = 61, and from Dc = 62 there is one, where each 64-column
step waits for the previous step's store (score.cu, stg_buffers).  The cases run the split and cluster routes, with
and without the trust-region distance (both k_score instances), and with categorical features, through the same
checks as test_gpu_score_routes.py: score, mean and stddev within 1e-10 of oracle/gp_oracle.py, the L-inf distance
bit for bit.
"""
import pytest

torch = pytest.importorskip('torch')
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason='no CUDA device')]

from test_gpu_score_routes import HALF1, Case, _t, dev, geom  # noqa: E402,F401  (dev, geom: fixtures)
from test_gpu_score_routes import test_score_route_matches_oracle as _check_route  # noqa: E402

CASES = [
    pytest.param(Case('split', 300, d, _t(9), last=40), id=f'D{d}-split') for d in (45, 46, 61, 62)
] + [
    pytest.param(Case('cluster', 200, d, HALF1, radius=None), id=f'D{d}-cluster') for d in (45, 46, 61, 62)
] + [
    pytest.param(Case('cluster', 130, d, HALF1, last=11, dk=3, mask_off=(7,)), id=f'D{d}-cluster-dk3') for d in (61, 62)
]


@pytest.mark.parametrize('c', CASES)
def test_stage_plan_edges_match_oracle(dev, geom, c):  # noqa: F811
  _check_route(dev, geom, c)
