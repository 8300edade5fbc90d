"""k_score (DMMA) against k_score_i8 (wgmma int8 split) on the C2 pool: CUDA-event time per pass."""
import json
import sys
import numpy as np
import torch

sys.path.insert(0, '.')
from vizier_b200 import gp  # noqa: E402


def main():
  n, d, m = 1000, 20, 100_000
  if len(sys.argv) > 2:
    n, d = int(sys.argv[1]), int(sys.argv[2])
  rng = np.random.default_rng(0)
  x = rng.uniform(size=(n, d))
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  dev = gp.DeviceGP(0)
  dev.fit(x, y, gp.GPHyperParams(1.0, 0.5 * (1 + np.arange(d) / d), 1e-3))
  pools = [dev.random_pool(m, d, seed=s) for s in range(10)]   # 160 MB > L2
  acq = gp.Acquisition(1.8, False, 0.0)
  res = {}
  outs = {}
  for mode in (0, 1):
    dev.set_int('score_i8', mode)
    out = None
    for p in pools[:3]:
      out = dev.score(p, acq, out=out)
    dev.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(dev._stream):
      e0.record(dev._stream)
      for it in range(20):
        out = dev.score(pools[it % 10], acq, out=out)
      e1.record(dev._stream)
    dev.synchronize()
    ms = e0.elapsed_time(e1) / 20
    res['i8' if mode else 'dmma'] = {'ms': ms, 'cand_per_s': m / ms * 1e3}
    outs[mode] = dev.score(pools[0], acq, with_aux=True)
    dev.synchronize()
  diff = (outs[0]['stddev'] - outs[1]['stddev']).abs().max().item()
  res['max_abs_sigma_diff'] = diff
  res['config'] = {'n': n, 'd': d, 'm': m}
  print(json.dumps(res))


if __name__ == '__main__':
  main()
