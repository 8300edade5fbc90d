"""Throughput of the parallel (q-) acquisitions.

1. `vzgp_score_qsets` (QEI) at N = 1000 trials, D = 20, q = 4, S = 100 samples over 25 000 sets (100 000 points):
   sets per second from CUDA events around whole calls, then one `torch.profiler` run of its own that splits a call
   into the W product (k_gemm_nt_tri), k_qset_moments, k_qacq_mc and the rest (K* and padding).
2. One `suggest(4)` of VizierGPBandit with parallel QEI at 1000 completed trials in D = 16 (the Eagle optimiser's set
   form holds q * D <= 64 features per fly), the GP already fitted by a first suggest, so the timed call is the set
   optimisation: 75 000 evaluations of the default Eagle optimiser.

Prints one JSON line with the card name and power limit read in the same run.  Usage:
  python tools/bench_qacq.py [--reps 10]
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


def _score_sets(reps):
  import torch
  from torch.profiler import ProfilerActivity, profile
  from vizier_b200 import _lib
  from vizier_b200 import gp
  rng = np.random.default_rng(0)
  n, d, q, n_sets = 1000, 20, 4, 25_000
  x = rng.uniform(size=(n, d))
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  dev = gp.DeviceGP(0)
  dev.fit(x, y, gp.GPHyperParams(1.0, np.full(d, 0.5), 1e-3))
  xs = dev.random_pool(n_sets * q, d, seed=1)
  qa = gp.QAcquisition(_lib.QACQ_QEI, best_label=float(y.max()), num_samples=100)
  for _ in range(3):
    dev.score_qsets(xs, q, qa, seed=3)
  dev.synchronize()
  times = []
  for _ in range(reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record(dev.stream)
    dev.score_qsets(xs, q, qa, seed=3)
    e.record(dev.stream)
    e.synchronize()
    times.append(s.elapsed_time(e))
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    dev.score_qsets(xs, q, qa, seed=3)
    dev.synchronize()
  kernels = {}
  for ev in prof.key_averages():
    if ev.device_type is not None and 'CUDA' in str(ev.device_type) and ev.count > 0:
      name = ev.key
      for k in ('k_gemm_nt_tri', 'k_qset_moments', 'k_qacq_mc'):
        if k in name:
          name = k
      t = getattr(ev, 'device_time_total', None) or getattr(ev, 'cuda_time_total', 0.0)
      kernels[name] = kernels.get(name, 0.0) + t / 1000.0
  dev.close()
  med = float(np.median(times))
  return {'setup': f'N={n}, D={d}, q={q}, S=100, {n_sets} sets ({n_sets * q} points), QEI',
          'call_ms': {'median': med, 'min': float(np.min(times)), 'max': float(np.max(times))},
          'sets_per_s': n_sets / (med / 1000.0),
          'kernel_ms_one_call': {k: round(v, 4) for k, v in sorted(kernels.items(), key=lambda kv: -kv[1])}}


def _suggest_s():
  from vizier_b200 import acquisitions as acq
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit
  p = vz.ProblemStatement()
  d = 16
  for i in range(d):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='obj', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  des = gp_bandit.VizierGPBandit.from_problem(
      p, seed=0, scoring_function_is_parallel=True,
      scoring_function_factory=acq.bayesian_scoring_function_factory(lambda d: acq.QEI(acq.get_best_labels(d.labels))))
  rng = np.random.default_rng(5)
  trials = []
  for i in range(1000):
    xv = rng.uniform(size=d)
    t = vz.Trial(parameters={f'x{j}': float(xv[j]) for j in range(d)}, id=i + 1)
    t.complete(vz.Measurement({'obj': float(-np.sum((xv - 0.3) ** 2))}))
    trials.append(t)
  des.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  t0 = time.perf_counter()
  des.suggest(4)                     # ARD fit + set optimisation
  first = time.perf_counter() - t0
  t0 = time.perf_counter()
  out = des.suggest(4)               # the fit is re-used: set optimisation only
  assert len(out) == 4
  return {'first_suggest_s': first, 'suggest_s': time.perf_counter() - t0}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=10)
  args = ap.parse_args()
  res = {'card': _card(), 'score_qsets': _score_sets(args.reps), 'suggest4_parallel_qei_n1000': _suggest_s()}
  print(json.dumps(res), flush=True)


if __name__ == '__main__':
  main()
