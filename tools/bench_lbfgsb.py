"""Cost of the L-BFGS-B acquisition optimiser (optimizers.LBFGSBOptimizerFactory, vzgp_score_grad).

1. `suggest(1)` of VizierGPBandit on N random completed trials of a D-dimensional quadratic, (N, D) = (50, 4) and
   (1000, 20), with the default LBFGSBOptimizerFactory (25 restarts, maxiter 100) and, in the same run, the default
   Eagle optimiser.  First call (ARD + optimiser) and second call (optimiser only: no new trial).
2. For the L-BFGS-B optimiser alone on the fitted model: the number of lock-step rounds, the device time per round
   (CUDA events around the batched `score_grad` call and its one device-to-host copy) and the host driver time per
   round (the rest of the wall time: SciPy's setulb calls and the Python around them).
3. `vzgp_score_grad` at M = 25 and M = 100 000 candidates, N = 1000, D = 20, CUDA events, median of `--reps`, with the
   FLOP count per candidate 2 N^2 (W = K* L^-T and V = W L^-1, triangular) + 12 N D (K* row, d2 and the gradient
   contraction) over kernel time.

Prints one JSON line with the card name and power limit read in the same run.  Usage:
  python tools/bench_lbfgsb.py [--reps 20]
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


def _card():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                          text=True, check=True).stdout.strip().splitlines()[0]
  except Exception as e:  # pylint: disable=broad-except
    return f'unknown ({e})'


def _designer(n, d, factory, seed=0):
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit
  p = vz.ProblemStatement()
  for i in range(d):
    p.search_space.root.add_float_param(f'x{i:02d}', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='obj', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  kw = {} if factory is None else {'acquisition_optimizer_factory': factory}
  des = gp_bandit.VizierGPBandit.from_problem(p, seed=seed, **kw)
  rng = np.random.default_rng(seed)
  trials = []
  for t in range(n):
    x = rng.uniform(size=d)
    tr = vz.Trial(parameters={f'x{i:02d}': float(x[i]) for i in range(d)})
    tr.complete(vz.Measurement({'obj': float(-np.sum((x - 0.3) ** 2) + 0.01 * rng.normal())}))
    trials.append(tr)
  des.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  return des


def _suggest_times(des):
  out = []
  for _ in range(2):
    t0 = time.perf_counter()
    des.suggest(1)
    out.append(time.perf_counter() - t0)
  return out


def _round_split(des):
  """Rounds, device ms / round and host ms / round of one L-BFGS-B run on the designer's fitted model."""
  import torch
  from vizier_b200 import optimizers as vb
  dev = des._dev
  cont, _, labels = des._trials_to_data(des._trials)
  acq = des._acquisition(cont.shape[0], labels, features=None)
  opt = vb.LBFGSBOptimizerFactory()(des._converter)
  inner = dev.score_grad
  device_ms = []

  def timed(xs, a, with_aux=False):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record(dev.stream)
    out = inner(xs, a, with_aux)
    e.record(dev.stream)
    e.synchronize()
    device_ms.append(s.elapsed_time(e))
    return out

  dev.score_grad = timed
  try:
    t0 = time.perf_counter()
    opt(dev, acq, count=1, seed=1)
    wall = (time.perf_counter() - t0) * 1e3
  finally:
    del dev.score_grad
  dev_total = float(np.sum(device_ms))
  # the round's device-to-host copy runs after the event pair, so its time is counted as host time
  return {'rounds': opt.rounds, 'device_ms_per_round': dev_total / opt.rounds,
          'host_ms_per_round': (wall - dev_total) / opt.rounds, 'optimizer_ms': wall}


def _score_grad_times(reps):
  import torch
  from vizier_b200 import gp
  n, d = 1000, 20
  rng = np.random.default_rng(0)
  x = rng.uniform(size=(n, d))
  y = -np.sum((x - 0.3) ** 2, axis=1)
  dev = gp.DeviceGP(0)
  dev.fit(x, y, gp.GPHyperParams(1.0, np.full(d, 0.5), 1e-3))
  acq = gp.Acquisition(1.8, True, 0.3)
  res = {}
  for m in (25, 100_000):
    xs = torch.from_numpy(rng.uniform(size=(m, d))).to(dev.device)
    dev.score_grad(xs, acq)
    dev.synchronize()
    times = []
    for _ in range(reps):
      s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      s.record(dev.stream)
      dev.score_grad(xs, acq)
      e.record(dev.stream)
      e.synchronize()
      times.append(s.elapsed_time(e))
    ms = float(np.median(times))
    flops = m * (2.0 * n * n + 12.0 * n * d)
    res[f'M={m}'] = {'ms': ms, 'gflop': flops / 1e9, 'tflop_per_s': flops / (ms * 1e-3) / 1e12}
  dev.close()
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=20)
  args = ap.parse_args()
  from vizier_b200 import optimizers as vb
  out = {'card': _card()}
  for n, d in ((50, 4), (1000, 20)):
    key = f'N={n},D={d}'
    lb = _designer(n, d, vb.LBFGSBOptimizerFactory())
    eg = _designer(n, d, None)
    out[key] = {'lbfgsb_suggest_s': _suggest_times(lb), 'eagle_suggest_s': _suggest_times(eg),
                'lbfgsb_rounds': _round_split(lb)}
  out['score_grad_N=1000_D=20'] = _score_grad_times(args.reps)
  out['card_after'] = _card()
  print(json.dumps(out))


if __name__ == '__main__':
  main()
