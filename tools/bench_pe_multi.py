"""Cost of the multi-metric GP-UCB-PE scorer next to the single-metric one.

1. `vzgp_score_pe_multi` (PE mode, AVERAGE, and UCB mode with S = 1000 scalarisations) against `vzgp_score_pe` on the
   same 100 000-candidate pool at N = 1000 trials, D = 20, n_metrics in {2, 4}: CUDA events around whole calls, the
   variants run alternately, median of `--reps`; then one `torch.profiler` run per multi-metric mode that splits a
   call into k_score (the two sigma products), k_mean_multi, k_pe_multi_combine and the rest.
2. One `suggest(1)` of VizierGPUCBPEBandit at 1000 completed trials with 2 metrics (ARD + Eagle), and a second one that
   re-runs the same work on the same data.

Prints one JSON line with the card name and power limit read in the same run.  Usage:
  python tools/bench_pe_multi.py [--reps 10]
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


def _kernel_split(fn):
  import torch
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    fn()
    torch.cuda.synchronize()
  kernels = {}
  for ev in prof.key_averages():
    if ev.device_type is not None and 'CUDA' in str(ev.device_type) and ev.count > 0:
      name = ev.key
      for k in ('k_score_finalize', 'k_score', 'k_mean_multi', 'k_pe_multi_combine'):
        if k in name:
          name = k
          break
      t = getattr(ev, 'device_time_total', None) or getattr(ev, 'cuda_time_total', 0.0)
      kernels[name] = kernels.get(name, 0.0) + t / 1000.0
  return {k: round(v, 4) for k, v in sorted(kernels.items(), key=lambda kv: -kv[1])}


def _score(reps, n_metrics):
  import torch
  from vizier_b200 import gp
  rng = np.random.default_rng(0)
  n, n_pending, d, m = 1000, 10, 20, 100_000
  x = rng.uniform(size=(n, d))
  y = np.stack([-np.sum((x - 0.1 * (k + 1)) ** 2, axis=1) + 0.05 * rng.normal(size=n) for k in range(n_metrics)], 1)
  params = gp.GPHyperParams(1.0, np.full(d, 0.5), 1e-3)
  a1, a = gp.DeviceGP(0), gp.DeviceGP(0)
  b = gp.DeviceGP(0, stream=a.stream)
  b1 = gp.DeviceGP(0, stream=a1.stream)
  a1.fit(x, y[:, 0], params)
  a.fit(x, y, params)
  xb = np.concatenate([x, rng.uniform(size=(n_pending, d))])
  b.fit(xb, np.zeros(n + n_pending), params)
  b1.fit(xb, np.zeros(n + n_pending), params)
  xs = a.random_pool(m, d, seed=1)
  torch.cuda.synchronize()
  mask = np.ones(d, bool)
  single = gp.UcbPeAcquisition(mode=1, threshold=0.0, trust_radius=0.3, tr_dim_mask=mask)
  w = np.abs(rng.normal(size=(1000, n_metrics))); w /= np.linalg.norm(w, axis=1, keepdims=True)
  ref = y.min(0) - 0.01 * (y.max(0) - y.min(0))
  pe = gp.UcbPeMultiAcquisition(n_metrics=n_metrics, mode=1, thresholds=np.zeros(n_metrics), trust_radius=0.3,
                                tr_dim_mask=mask)
  ucb = gp.UcbPeMultiAcquisition(n_metrics=n_metrics, mode=0, trust_radius=0.3, tr_dim_mask=mask,
                                 scalarization=gp.ScalarizedUcbAcquisition(w, ref, None, 1.8))
  variants = {'score_pe': lambda: a1.score_pe(b1, xs, single),
              'score_pe_multi_pe': lambda: a.score_pe_multi(b, xs, pe),
              'score_pe_multi_ucb': lambda: a.score_pe_multi(b, xs, ucb)}
  for f in variants.values():
    f(); f()
  times = {k: [] for k in variants}
  for _ in range(reps):             # alternate the variants so drift hits all of them alike
    for k, f in variants.items():
      st = torch.cuda.current_stream()
      s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      torch.cuda.synchronize()
      s.record(st)
      f()                           # synchronous: returns after the device finished
      e.record(st)
      e.synchronize()
      times[k].append(s.elapsed_time(e))
  out = {k: {'median_ms': float(np.median(v)), 'min_ms': float(np.min(v)), 'max_ms': float(np.max(v))}
         for k, v in times.items()}
  out['kernel_ms_one_call'] = {k: _kernel_split(variants[k]) for k in ('score_pe_multi_pe', 'score_pe_multi_ucb')}
  for h in (b1, b, a1, a):
    h.close()
  return out


def _suggest():
  from vizier_b200 import vz
  from vizier_b200.designers import gp_ucb_pe
  p = vz.ProblemStatement()
  d = 20
  for i in range(d):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='gain', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  p.metric_information.append(vz.MetricInformation(name='cost', goal=vz.ObjectiveMetricGoal.MINIMIZE))
  rng = np.random.default_rng(5)
  trials = []
  for i in range(1000):
    xv = rng.uniform(size=d)
    t = vz.Trial(parameters={f'x{j}': float(xv[j]) for j in range(d)}, id=i + 1)
    t.complete(vz.Measurement({'gain': float(-np.sum((xv - 0.3) ** 2)), 'cost': float(np.sum((xv - 0.6) ** 2))}))
    trials.append(t)
  des = gp_ucb_pe.VizierGPUCBPEBandit.from_problem(p, seed=0)
  des.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  res = {}
  for run in ('first', 'second'):
    t0 = time.perf_counter()
    out = des.suggest(1)            # ARD on both metrics + Eagle with 75 000 evaluations
    res[f'{run}_suggest1_s'] = time.perf_counter() - t0
    assert len(out) == 1
    res[f'{run}_use_ucb'] = out[0].metadata.ns('google_gp_ucb_pe_bandit').ns('prediction_in_warped_y_space')['use_ucb']
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=10)
  args = ap.parse_args()
  res = {'card': _card(), 'setup': 'N=1000, D=20, 100000 candidates, PE trust radius 0.3, S=1000'}
  for nm in (2, 4):
    res[f'score_n_metrics_{nm}'] = _score(args.reps, nm)
  res['suggest1_two_metrics_n1000'] = _suggest()
  print(json.dumps(res), flush=True)


if __name__ == '__main__':
  main()
