"""Wall time of one ARD fit with Adam (ard.OptaxTrain) on the device, three ways on the same data:

  fused   every epoch of every restart in one launch of `vzgp_ard_adam_small` (csrc/ard_adam.cu);
  host    the host-stepped epochs: one `vzgp_nll_grad` evaluation per restart and epoch (k_nll_grad_small, a launch and
          a synchronisation each), SoftClip and Adam in NumPy;
  lbfgsb  today's default ARD, `ard.train_gp` with ScipyLbfgsB (maxiter 50, restarts on up to 8 handles).

Sizes: N in {16, 32, 64} trials, D in {10, 20} continuous features, R in {4, 64} restarts, 500 epochs.  The variants
run alternately, `--reps` times each, and the median wall time (host clock around work that ends in a device
synchronisation) is reported.  Prints one JSON line with the card's name and power limit.

  python tools/bench_adam_ard.py [--epochs 500] [--reps 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _card():
  import torch
  name = torch.cuda.get_device_name(0)
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
    power, clock = (s.strip() for s in out.split(','))
  except Exception:  # pylint: disable=broad-except
    power = clock = 'unknown'
  return name, power, clock


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--epochs', type=int, default=500)
  ap.add_argument('--reps', type=int, default=3)
  ap.add_argument('--sizes', default='16,32,64')
  ap.add_argument('--dims', default='10,20')
  ap.add_argument('--restarts', default='4,64')
  a = ap.parse_args()
  import torch
  if not torch.cuda.is_available():
    raise SystemExit('bench_adam_ard needs a CUDA device')
  from vizier_b200 import ard, gp

  name, power, clock = _card()
  dev = gp.DeviceGP(0)
  rows = []
  for n in (int(s) for s in a.sizes.split(',')):
    for d in (int(s) for s in a.dims.split(',')):
      rng = np.random.default_rng(n * 100 + d)
      x = rng.uniform(size=(n, d))
      y = np.sin(3.0 * x.sum(1)) - np.sum((x - 0.4) ** 2, 1) + 0.05 * rng.normal(size=n)
      xt = torch.from_numpy(x).cuda()
      yt = torch.from_numpy(y).cuda()
      lo, hi = gp.param_bounds(d, 0)
      for r in (int(s) for s in a.restarts.split(',')):
        inits = ard.log_uniform_init(np.random.default_rng(r), d, 0, r)
        fused = ard.OptaxTrain(ard.adam(5e-2), epochs=a.epochs)
        host = ard.OptaxTrain(ard.adam(5e-2), epochs=a.epochs)
        fn = dev.make_loss_fn(xt, yt)

        def run_fused():
          fused.fit(dev, xt, yt, None, inits, lo, hi, best_n=1)

        def run_host():
          host(inits, fn, list(zip(lo, hi)), best_n=1)

        def run_lbfgsb():
          ard.train_gp(dev, xt, yt, rng=np.random.default_rng(r), random_restarts=r)

        variants = {'fused': run_fused, 'host': run_host, 'lbfgsb': run_lbfgsb}
        for f in variants.values():   # warm-up: modules, buffers, worker handles
          f()
        torch.cuda.synchronize()
        times = {k: [] for k in variants}
        for _ in range(a.reps):
          for k, f in variants.items():
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
        med = {k: statistics.median(v) for k, v in times.items()}
        assert fused.last_metrics['route'] == 'fused'
        diff = float(np.nanmax(np.abs(fused.last_metrics['loss'] - host.last_metrics['loss'])
                               / np.abs(host.last_metrics['loss'])))
        row = {'n': n, 'd': d, 'restarts': r, 'epochs': a.epochs,
               'fused_ms': round(1e3 * med['fused'], 3), 'host_ms': round(1e3 * med['host'], 3),
               'lbfgsb_ms': round(1e3 * med['lbfgsb'], 3),
               'fused_us_per_epoch': round(1e6 * med['fused'] / a.epochs, 2),
               'host_us_per_epoch': round(1e6 * med['host'] / a.epochs, 2),
               'host_over_fused': round(med['host'] / med['fused'], 2),
               'lbfgsb_over_fused': round(med['lbfgsb'] / med['fused'], 2),
               'max_rel_loss_diff_fused_vs_host': diff}
        rows.append(row)
        print(json.dumps(row), file=sys.stderr)
  print(json.dumps({'bench': 'adam_ard', 'gpu': name, 'power_limit': power, 'max_sm_clock': clock,
                    'reps': a.reps, 'rows': rows}))


if __name__ == '__main__':
  main()
