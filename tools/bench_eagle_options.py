"""Cost of the Eagle strategy options in one `vzgp_eagle_run`: categorical features past 64 values, UNNORMALIZED force
normalisation against MEAN, MULTIPLICATIVE perturbation against ADDITIVE.

Each form of the loop runs one Eagle optimisation of 200 steps against a fitted GP (UCB, no trust region):
  persistent   N = 50,   Dc = 20, B = 25,  P = 50     (k_eagle_persistent64)
  cooperative  N = 1000, Dc = 20, B = 25,  P = 100    (k_eagle_grid)
  graph        N = 1000, Dc = 20, B = 600, P = 1200   (k_eagle_suggest / scoring / k_eagle_update from a CUDA graph)
with one extra categorical feature of 64, 65 or 1000 values (Dk = 1), and with Dk = 0 under the four combinations of
{MEAN, UNNORMALIZED} x {ADDITIVE, MULTIPLICATIVE}.  Variants of one form alternate within each round, so drift of the
card affects them alike; the median over rounds is reported in ms per run, with the route each run took.

Prints one JSON line with the card name and power limit read in the same run.  Usage:
  python tools/bench_eagle_options.py [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FORMS = {'persistent': (50, 25, 50), 'cooperative': (1000, 25, 100), 'graph': (1000, 600, 1200)}   # N, B, P
STEPS = 200
DC = 20
VARIANTS = [('cat64', 64, 0, 0), ('cat65', 65, 0, 0), ('cat1000', 1000, 0, 0),
            ('mean-additive', 0, 0, 0), ('unnormalized-additive', 0, 2, 0),
            ('mean-multiplicative', 0, 0, 1), ('unnormalized-multiplicative', 0, 2, 1)]   # name, size, norm, pert


def _card():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                          text=True, check=True).stdout.strip().splitlines()[0]
  except Exception as e:  # pylint: disable=broad-except
    return f'unknown ({e})'


def _fitted(n, size, seed=0):
  from vizier_b200 import gp
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, DC))
  z = rng.integers(0, size, size=(n, 1)).astype(np.int32) if size else None
  y = -np.sum((x - 0.3) ** 2, axis=1) - (0.3 * (z[:, 0] % 5 != 2) if size else 0.0)
  dev = gp.DeviceGP(0)
  dev.fit(x, y, gp.GPHyperParams(1.0, np.full(DC, 0.5), 1e-3, np.array([1.0]) if size else None), z=z)
  return dev


def one_run_ms(dev, form, size, norm, pert):
  from vizier_b200 import _lib, gp
  n, b, p = FORMS[form]
  cfg = _lib.EagleConfig(0.45, 1.5, 0.008, 0.16, 7e-5, 0.7, 0.5, 0.96, p, b, STEPS * b, 1.0, 30.0, 0.98, norm, 1)
  dev.set_int('eagle_perturbation', pert)
  dev.synchronize()
  t0 = time.perf_counter()
  dev.eagle_run(cfg, gp.Acquisition(1.8, False, 1.0), 1, 7, cat_sizes=[size] if size else None)   # ends in a sync
  return (time.perf_counter() - t0) * 1e3, dev.get_int('eagle_route')


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--rounds', type=int, default=5)
  args = ap.parse_args()
  import torch
  assert torch.cuda.is_available(), 'bench_eagle_options needs a CUDA device'
  out = {'card': _card(), 'steps_per_run': STEPS, 'dc': DC, 'forms': {}}
  for form, (n, b, p) in FORMS.items():
    devs = {s: _fitted(n, s) for s in sorted({v[1] for v in VARIANTS})}
    times = {v[0]: [] for v in VARIANTS}
    routes = {}
    for name, size, norm, pert in VARIANTS:           # warm-up: workspaces, modules
      one_run_ms(devs[size], form, size, norm, pert)
    for _ in range(args.rounds):
      for name, size, norm, pert in VARIANTS:
        ms, routes[name] = one_run_ms(devs[size], form, size, norm, pert)
        times[name].append(ms)
    out['forms'][form] = {'N': n, 'B': b, 'P': p,
                          'ms_median': {k: round(float(np.median(v)), 3) for k, v in times.items()},
                          'ms_all': {k: [round(t, 3) for t in v] for k, v in times.items()}, 'route': routes}
    for d in devs.values():
      d.close()
  print(json.dumps(out), flush=True)


if __name__ == '__main__':
  main()
