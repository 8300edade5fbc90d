"""Cost of the acquisition functions on the scoring path, on bench.py's C2 setup (N = 1000 trials, D = 20, M = 100 000
candidates).

1. Default path (UCB) against another build: runs `bench.py --no-suggest --no-cpu` alternately in this tree and in
   `--other-tree` (a built checkout of another commit), `--rounds` times each, and reports the k_score kernel time of
   every run, so the spread of each build is visible next to the difference.
2. k_score time under EI, and under the ucb_pi preset, against UCB in one process (CUDA events, alternating), and
   one default `suggest()` of VizierGPBandit with and without an EI scoring function.

Prints one JSON line with the card name and power limit.  Usage:
  python tools/bench_acq.py [--other-tree path/to/other/checkout] [--rounds 3] [--reps 50]
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
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    return q
  except Exception as e:  # pylint: disable=broad-except
    return f'unknown ({e})'


def _find(obj, key):
  if isinstance(obj, dict):
    if key in obj:
      return obj[key]
    for v in obj.values():
      r = _find(v, key)
      if r is not None:
        return r
  return None


def _bench_kernel_ms(tree, steps):
  out = subprocess.run([sys.executable, os.path.join(tree, 'bench.py'), '--gpus', '1', '--steps', str(steps), '--warmup', '3',
                        '--no-suggest', '--no-cpu'], capture_output=True, text=True, cwd=tree)
  lines = [l for l in out.stdout.splitlines() if l.startswith('{')]
  if out.returncode != 0 or not lines:
    raise RuntimeError(f'bench.py failed ({out.returncode}): {out.stderr[-2000:]}')
  return float(_find(json.loads(lines[-1]), 'kernel_ms'))


def _in_process(reps):
  import torch
  from vizier_b200 import acquisitions as acq
  from vizier_b200 import gp
  rng = np.random.default_rng(0)
  n, d, m = 1000, 20, 100_000
  x = rng.uniform(size=(n, d))
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  dev = gp.DeviceGP(0)
  dev.set_int('score_i8', 0)
  dev.fit(x, y, gp.GPHyperParams(1.0, np.full(d, 0.5), 1e-3))
  xs = dev.random_pool(m, d, seed=1)
  data = acq.ModelData(None, acq.PaddedArray.as_padded(y[:, None]))
  acqs = {'ucb': gp.Acquisition(1.8, False, 1.0),
          'ei': gp.Acquisition(1.8, False, 1.0, acq_fn=acq.lower_acquisition(acq.EI(acq.get_best_labels(data.labels)))),
          'ucb_pi': gp.Acquisition(1.8, False, 1.0,
                                   acq_fn=acq.lower_acquisition(acq.AcquisitionTrustRegion.default_ucb_pi(data)))}
  out = {'score': torch.empty(m, dtype=torch.float64, device=dev.device)}
  times = {k: [] for k in acqs}
  for k, a in acqs.items():      # warm up every variant
    for _ in range(3):
      dev.score(xs, a, out=out)
  dev.synchronize()
  for _ in range(reps):
    for k, a in acqs.items():
      dev.score(xs, a, out=out)   # switch the handle's acquisition outside the timed window
      s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      s.record(dev.stream)
      dev.score(xs, a, out=out)
      e.record(dev.stream)
      e.synchronize()
      times[k].append(s.elapsed_time(e))
  dev.close()
  return {k: {'median_ms': float(np.median(v)), 'min_ms': float(np.min(v)), 'max_ms': float(np.max(v))} for k, v in times.items()}


def _suggest_s(with_ei):
  from vizier_b200 import acquisitions as acq
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit
  p = vz.ProblemStatement()
  for i in range(20):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='obj', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  kw = {}
  if with_ei:
    kw['scoring_function_factory'] = acq.bayesian_scoring_function_factory(lambda d: acq.EI(acq.get_best_labels(d.labels)))
  des = gp_bandit.VizierGPBandit.from_problem(p, seed=0, **kw)
  rng = np.random.default_rng(5)
  trials = []
  for i in range(100):
    xv = rng.uniform(size=20)
    t = vz.Trial(parameters={f'x{j}': float(xv[j]) for j in range(20)}, id=i + 1)
    t.complete(vz.Measurement({'obj': float(-np.sum((xv - 0.3) ** 2))}))
    trials.append(t)
  des.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  des.suggest(1)                     # fits the GP and compiles nothing: the timed call re-uses the fit
  t0 = time.perf_counter()
  des.suggest(1)
  return time.perf_counter() - t0


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--other-tree', default=None, help='built checkout of the commit to compare the default path against')
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--steps', type=int, default=200)
  ap.add_argument('--reps', type=int, default=50)
  args = ap.parse_args()
  res = {'card': _card(), 'setup': 'N=1000, D=20, M=100000 (bench.py C2)'}
  if args.other_tree:
    runs = {'this': [], 'other': []}
    for _ in range(args.rounds):
      runs['other'].append(_bench_kernel_ms(os.path.abspath(args.other_tree), args.steps))
      runs['this'].append(_bench_kernel_ms(ROOT, args.steps))
    res['ucb_k_score_ms_bench'] = runs
  res['k_score_ms_in_process'] = _in_process(args.reps)
  res['suggest_s'] = {'ucb': _suggest_s(False), 'ei': _suggest_s(True)}
  print(json.dumps(res), flush=True)


if __name__ == '__main__':
  main()
