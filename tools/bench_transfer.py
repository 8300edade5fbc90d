"""Cost of transfer-learning stacks whose levels are ensembles or multi-metric models.

1. One scoring pass over 100 000 candidates (UCB, trust radius 0.3) on stacks of L in {2, 3} levels: every prior level
   fitted on N = 1000 trials and the current (top) level on 200, D = 20; E = 1 (`vzgp_score_stack`), E = 3 and E = 5
   (`vzgp_score_stack_ensemble`), and a two-metric stack of two levels (`vzgp_score_stack_multi`, 1000 scalarisations).
   CUDA events around whole calls, the variants run alternately, median of `--reps`.
2. The default Eagle loop (75 000 evaluations, batches of 25) on the two-level E = 3 stack (replayed graph).
3. One `suggest(1)` of VizierGPBandit(ensemble_size=3) with one prior study of 1000 trials and 200 current trials
   (ARD of the top level + Eagle), first and second call.

Prints one JSON line with the card name and power limit read in the same run.  Usage:
  python tools/bench_transfer.py [--reps 10]
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

N_PRIOR, N_TOP, D, M = 1000, 200, 20, 100_000


def _card():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                          text=True, check=True).stdout.strip().splitlines()[0]
  except Exception as e:  # pylint: disable=broad-except
    return f'unknown ({e})'


def _stack(n_levels, e, rng, n_metrics=1):
  from vizier_b200 import gp
  stack = gp.StackedGP(0)
  x = None
  for l in range(n_levels):
    n = N_TOP if l == n_levels - 1 else N_PRIOR
    x = rng.uniform(size=(n, D))
    y = -np.sum((x - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
    if n_metrics > 1:
      y = np.stack([y * (1 + m) for m in range(n_metrics)], axis=1)
    y = y - stack.mean(x) if stack.levels else y
    params = [gp.GPHyperParams(1.0 + 0.1 * k, np.full(D, 0.5 + 0.05 * k), 1e-3) for k in range(e)]
    level = stack.new_level(e)
    level.fit(x, y, params if e > 1 else params[0])
    stack.push(level, n)
  return stack, x


def _timed(fn):
  import torch
  st = torch.cuda.current_stream()
  s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  s.record(st)
  fn()
  e.record(st)
  e.synchronize()
  return s.elapsed_time(e)


def _score(reps):
  import torch
  from vizier_b200 import gp
  rng = np.random.default_rng(0)
  acq = gp.Acquisition(1.8, True, 0.3)
  stacks = {(l, e): _stack(l, e, rng)[0] for l in (2, 3) for e in (1, 3, 5)}
  multi = _stack(2, 1, rng, n_metrics=2)[0]
  w = np.abs(rng.normal(size=(1000, 2)))
  sc = gp.ScalarizedUcbAcquisition(w / np.linalg.norm(w, axis=1, keepdims=True), np.array([-2.0, -4.0]), None, 1.8)
  xs = stacks[(2, 1)]._lead().random_pool(M, D, seed=1)
  torch.cuda.synchronize()

  def run(s):
    s.score(xs, acq)
    s.synchronize()

  def run_multi():
    multi.score_multi(xs, sc)
    multi.synchronize()

  variants = {f'L{l}_E{e}': (lambda s=s: run(s)) for (l, e), s in stacks.items()}
  variants['L2_two_metrics'] = run_multi
  for f in variants.values():
    f(); f()
  times = {k: [] for k in variants}
  for _ in range(reps):             # alternate the variants so drift hits all of them alike
    for k, f in variants.items():
      times[k].append(_timed(f))
  for s in list(stacks.values()) + [multi]:
    s.close()
  return {k: {'median_ms': float(np.median(v)), 'min_ms': float(np.min(v)), 'max_ms': float(np.max(v))}
          for k, v in times.items()}


def _eagle(reps):
  from vizier_b200 import gp
  from vizier_b200 import optimizers as vb
  rng = np.random.default_rng(3)
  stack, x_top = _stack(2, 3, rng)
  opt = vb.VectorizedOptimizer(vb.VectorizedEagleStrategyFactory(), D, 0, 25, 75_000, ())
  cfg = opt._eagle_config()   # pylint: disable=protected-access
  acq = gp.Acquisition(1.8, True, 0.3)
  stack.eagle_run(cfg, acq, 1, 0, prior=x_top)
  times = [_timed(lambda s=s: stack.eagle_run(cfg, acq, 1, s, prior=x_top)) for s in range(reps)]
  route = stack._lead().get_int('eagle_route')
  stack.close()
  return {'eagle_route': route, 'median_ms': float(np.median(times)), 'min_ms': float(np.min(times))}


def _suggest():
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit
  p = vz.ProblemStatement()
  for i in range(D):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='gain', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  rng = np.random.default_rng(5)

  def trials(n, start):
    out = []
    for i in range(n):
      xv = rng.uniform(size=D)
      t = vz.Trial(parameters={f'x{j}': float(xv[j]) for j in range(D)}, id=start + i)
      t.complete(vz.Measurement({'gain': float(-np.sum((xv - 0.3) ** 2))}))
      out.append(t)
    return out

  des = gp_bandit.VizierGPBandit.from_problem(p, seed=0, ensemble_size=3)
  t0 = time.perf_counter()
  des.set_priors([vz.CompletedTrials(trials(N_PRIOR, 1))])
  res = {'set_priors_s': time.perf_counter() - t0}
  des.update(vz.CompletedTrials(trials(N_TOP, 10_000)), vz.ActiveTrials())
  for run in ('first', 'second'):
    t0 = time.perf_counter()
    out = des.suggest(1)
    res[f'{run}_suggest1_s'] = time.perf_counter() - t0
    assert len(out) == 1
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=10)
  args = ap.parse_args()
  res = {'card': _card(),
         'setup': f'prior levels N={N_PRIOR}, top N={N_TOP}, D={D}, {M} candidates, UCB, trust radius 0.3'}
  res['score'] = _score(args.reps)
  res['eagle_l2_e3'] = _eagle(max(3, args.reps // 2))
  res['suggest1_e3_one_prior'] = _suggest()
  print(json.dumps(res), flush=True)


if __name__ == '__main__':
  main()
