"""clock64 breakdown of k_score on the C2 pool (N=1000, D=20, M=100k) - needs the instrumented library
(`make -C vizier_b200/csrc timing`, then VZGP_LIB=vizier_b200/_lib/libvzgp_timing.so).

Usage: score_timing.py [N D] [--trust-region].  --trust-region scores with a trust radius of 0.3, which
runs the k_score<true> instance (L-inf distance); bench.py times that instance at N=100.

Counters are summed over all CTAs and reported per tile: phase 1 (K* tile), the gate after it, phase 2
(DMMA slab stream), the whole tile (all of math warp 0), the average math warp's wait on the full
barriers (ring starved: operand feed too slow) and the producer's wait on the empty barriers (ring full:
the math warps are the limit).  Phase 1 is split into d2 (without --trust-region: the norms and the DMMA cross
term of the centred form, timed to the last DMMA's result; with it: the difference-first loop), Matern + mu, the scratch stores (K* written
to the shared-memory staging buffer, plus the TMA store issue) and the waits: barriers, cp.async and the TMA
stores (math warp 0).  Between builds whose d2 forms differ, phase 1 as a whole is the fair comparison: where the
work of one part moves, its latency can show up in the next counter."""
import ctypes as C
import json
import sys
import numpy as np
import torch

sys.path.insert(0, '.')
from vizier_b200 import _lib, gp  # noqa: E402

MATH_WARPS = 8
COUNTERS = 11


def main():
  n, d, m = 1000, 20, 100_000
  args = [a for a in sys.argv[1:] if a != '--trust-region']
  if len(args) >= 2:
    n, d = int(args[0]), int(args[1])
  rng = np.random.default_rng(0)
  x = rng.uniform(size=(n, d))
  y = -np.sum((x - 0.3) ** 2, axis=1)
  dev = gp.DeviceGP(0)
  dev.fit(x, y, gp.GPHyperParams(1.0, 0.5 * (1 + np.arange(d) / d), 1e-3))
  dev.set_int('score_i8', 0)
  pools = [dev.random_pool(m, d, seed=s) for s in range(4)]
  acq = gp.Acquisition(1.8, True, 0.3) if '--trust-region' in sys.argv else gp.Acquisition(1.8, False, 0.0)
  lib = _lib.load()
  lib.vzgp_debug_score_timing.restype = C.c_int
  buf = (C.c_ulonglong * COUNTERS)()
  out = None
  for p in pools[:2]:
    out = dev.score(p, acq, out=out)
  dev.synchronize()
  assert lib.vzgp_debug_score_timing(buf, 1) == 0
  passes = 8
  e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
  e0.record(dev._stream)
  for it in range(passes):
    out = dev.score(pools[it % 4], acq, out=out)
  e1.record(dev._stream)
  dev.synchronize()
  assert lib.vzgp_debug_score_timing(buf, 0) == 0
  t = np.array(buf[:], dtype=np.float64)
  tiles = max(t[0], 1.0)
  per_tile = {'phase1': t[1] / tiles, 'gate': t[3] / tiles, 'phase2': t[2] / tiles, 'tile': t[4] / tiles,
              'full_wait_per_math_warp': t[5] / MATH_WARPS / tiles, 'empty_wait_producer': t[6] / tiles,
              'phase1_d2': t[7] / tiles, 'phase1_matern_mu': t[8] / tiles, 'phase1_stores': t[9] / tiles,
              'phase1_waits': t[10] / tiles}
  res = {'ms_per_pass': e0.elapsed_time(e1) / passes, 'tiles_per_pass': tiles / passes,
         'cycles_per_tile': {k: int(round(v)) for k, v in per_tile.items()},
         'full_wait_share_of_phase2': round(per_tile['full_wait_per_math_warp'] / max(per_tile['phase2'], 1.0), 4),
         'empty_wait_share_of_phase2': round(per_tile['empty_wait_producer'] / max(per_tile['phase2'], 1.0), 4)}
  print(json.dumps(res))


if __name__ == '__main__':
  main()
