"""clock64 breakdown of k_score_i8 (CTA 0) - needs the instrumented library (`make -C vizier_b200/csrc timing`,
then VZGP_LIB=vizier_b200/_lib/libvzgp_timing.so)."""
import ctypes as C
import json
import sys
import numpy as np
import torch

sys.path.insert(0, '.')
from vizier_b200 import _lib, gp  # noqa: E402

NAMES = {0: 'phase1', 3: 'tile', 12: 'k_wait_kfree'}


def main():
  n, d, m = 1000, 20, 100_000
  if len(sys.argv) > 2:
    n, d = int(sys.argv[1]), int(sys.argv[2])
  rng = np.random.default_rng(0)
  x = rng.uniform(size=(n, d))
  y = -np.sum((x - 0.3) ** 2, axis=1)
  dev = gp.DeviceGP(0)
  dev.fit(x, y, gp.GPHyperParams(1.0, 0.5 * (1 + np.arange(d) / d), 1e-3))
  dev.set_int('score_i8', 1)
  pools = [dev.random_pool(m, d, seed=s) for s in range(4)]
  acq = gp.Acquisition(1.8, False, 0.0)
  lib = _lib.load()
  buf = (C.c_longlong * 16)()
  out = None
  for p in pools[:2]:
    out = dev.score(p, acq, out=out)
  dev.synchronize()
  lib.vzgp_debug_i8_timing.restype = C.c_int
  assert lib.vzgp_debug_i8_timing(buf, 1) == 0
  e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
  e0.record(dev._stream)
  for it in range(8):
    out = dev.score(pools[it % 4], acq, out=out)
  e1.record(dev._stream)
  dev.synchronize()
  assert lib.vzgp_debug_i8_timing(buf, 0) == 0
  t = np.array(buf[:], dtype=np.int64)
  tiles = max(int(t[15]), 1)
  res = {'ms_per_pass': e0.elapsed_time(e1) / 8, 'tiles_cta0': tiles,
         'cycles_per_tile': {k: int(t[i] // tiles) for i, k in NAMES.items()}}
  print(json.dumps(res))


if __name__ == '__main__':
  main()
