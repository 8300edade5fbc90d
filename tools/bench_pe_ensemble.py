"""Cost of GP-UCB-PE over uniform ensembles next to the single-model scorer.

1. `vzgp_score_pe` against `vzgp_score_pe_ensemble` for E = 1..5 on the same 100 000-candidate pool at N = 1000
   trials, D = 20 (PE mode, strict trust radius 0.3): CUDA events around whole calls, the variants run alternately,
   median of `--reps`.
2. The default Eagle loop (75 000 evaluations, batches of 25) at N = 1000 in the cooperative form at E = 1 (a pair of
   models) and E = 3, and at E = 3 in the replayed-graph form (VZGP_EAGLE_GRID=0 is read once per process, so that
   form runs in a child process).
3. One `suggest(1)` of VizierGPUCBPEBandit at 1000 completed trials with ensemble_size 1 and 3 (ARD + Eagle).

Prints one JSON line with the card name and power limit read in the same run.  Usage:
  python tools/bench_pe_ensemble.py [--reps 10]
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

N, N_PENDING, D, M = 1000, 10, 20, 100_000


def _card():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                          text=True, check=True).stdout.strip().splitlines()[0]
  except Exception as e:  # pylint: disable=broad-except
    return f'unknown ({e})'


def _ensembles(e, rng):
  from vizier_b200 import gp
  x = rng.uniform(size=(N, D))
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=N)
  xb = np.concatenate([x, rng.uniform(size=(N_PENDING, D))])
  yb = np.concatenate([y, np.zeros(N_PENDING)])
  params = [gp.GPHyperParams(1.0 + 0.1 * k, np.full(D, 0.5 + 0.05 * k), 1e-3) for k in range(e)]
  a = gp.EnsembleGP(0, e)
  b = gp.EnsembleGP(0, e, stream=a.stream)
  a.fit(x, y, params)
  b.fit(xb, yb, params)
  return x, a, b


def _timed(fn):
  import torch
  st = torch.cuda.current_stream()
  s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  s.record(st)
  fn()                              # synchronous: returns after the device finished
  e.record(st)
  e.synchronize()
  return s.elapsed_time(e)


def _score(reps):
  import torch
  from vizier_b200 import gp
  rng = np.random.default_rng(0)
  pe = gp.UcbPeAcquisition(mode=1, threshold=0.0, trust_radius=0.3, tr_dim_mask=np.ones(D, bool))
  models = {e: _ensembles(e, rng) for e in range(1, 6)}
  xs = models[1][1].members[0].random_pool(M, D, seed=1)
  torch.cuda.synchronize()
  a1, b1 = models[1][1].members[0], models[1][2].members[0]
  variants = {'score_pe': lambda: a1.score_pe(b1, xs, pe)}
  for e, (_, a, b) in models.items():
    variants[f'score_pe_ensemble_e{e}'] = lambda a=a, b=b: a.score_pe(b, xs, pe)
  for f in variants.values():
    f(); f()
  times = {k: [] for k in variants}
  for _ in range(reps):             # alternate the variants so drift hits all of them alike
    for k, f in variants.items():
      times[k].append(_timed(f))
  for _, a, b in models.values():
    b.close(); a.close()
  return {k: {'median_ms': float(np.median(v)), 'min_ms': float(np.min(v)), 'max_ms': float(np.max(v))}
          for k, v in times.items()}


def _eagle(reps, e=3):
  """Median wall time of the default Eagle loop at E members in whichever form this process takes."""
  from vizier_b200 import optimizers as vb
  from vizier_b200 import gp
  from vizier_b200.designers import gp_ucb_pe
  rng = np.random.default_rng(3)
  x, a, b = _ensembles(e, rng)
  opt = vb.VectorizedOptimizer(vb.VectorizedEagleStrategyFactory(eagle_config=gp_ucb_pe.default_eagle_config), D, 0,
                               25, 75_000, ())
  cfg = opt._eagle_config()   # pylint: disable=protected-access
  pe = gp.UcbPeAcquisition(mode=1, threshold=0.0, trust_radius=0.3, tr_dim_mask=np.ones(D, bool))
  a.eagle_run(cfg, pe, 1, 0, prior=x, other=b)
  times = [_timed(lambda s=s: a.eagle_run(cfg, pe, 1, s, prior=x, other=b)) for s in range(reps)]
  route = a.members[0].get_int('eagle_route')
  b.close(); a.close()
  return {'eagle_route': route, 'median_ms': float(np.median(times)), 'min_ms': float(np.min(times))}


def _suggest(ensemble_size):
  from vizier_b200 import vz
  from vizier_b200.designers import gp_ucb_pe
  p = vz.ProblemStatement()
  for i in range(D):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='gain', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  rng = np.random.default_rng(5)
  trials = []
  for i in range(N):
    xv = rng.uniform(size=D)
    t = vz.Trial(parameters={f'x{j}': float(xv[j]) for j in range(D)}, id=i + 1)
    t.complete(vz.Measurement({'gain': float(-np.sum((xv - 0.3) ** 2))}))
    trials.append(t)
  des = gp_ucb_pe.VizierGPUCBPEBandit.from_problem(p, seed=0, ensemble_size=ensemble_size)
  des.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  res = {}
  for run in ('first', 'second'):
    t0 = time.perf_counter()
    out = des.suggest(1)            # ARD + Eagle with 75 000 evaluations
    res[f'{run}_suggest1_s'] = time.perf_counter() - t0
    assert len(out) == 1
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=10)
  ap.add_argument('--eagle-only', action='store_true', help='time the Eagle loop alone (used for the graph form)')
  args = ap.parse_args()
  if args.eagle_only:
    print('EAGLE ' + json.dumps(_eagle(args.reps)), flush=True)
    return
  res = {'card': _card(), 'setup': f'N={N}, D={D}, {M} candidates, PE mode, strict trust radius 0.3'}
  res['score'] = _score(args.reps)
  res['eagle_e1_cooperative'] = _eagle(args.reps, 1)
  res['eagle_e3_cooperative'] = _eagle(args.reps)
  env = dict(os.environ, VZGP_EAGLE_GRID='0')
  proc = subprocess.run([sys.executable, os.path.abspath(__file__), '--eagle-only', '--reps', str(args.reps)], env=env,
                        capture_output=True, text=True, check=True)
  line = [ln for ln in proc.stdout.splitlines() if ln.startswith('EAGLE ')][-1]
  res['eagle_e3_graph'] = json.loads(line[len('EAGLE '):])
  res['suggest1_n1000'] = {f'ensemble_size_{e}': _suggest(e) for e in (1, 3)}
  print(json.dumps(res), flush=True)


if __name__ == '__main__':
  main()
