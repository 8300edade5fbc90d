"""Cost of MaxValueEntropySearch (vzgp_mes_fit and the MES branch of the scoring epilogues).

a. `vzgp_score` at C2 (N = 1000, D = 20, M = 100 000, the k_score route): UCB, EI and MES (K = 100) alternating,
   CUDA events, median of `--reps`.
b. The small-pool route at M = 512, same acquisitions.
c. `vzgp_mes_fit` (K = 100) at N = 50 and N = 1000.
d. Second-call `suggest(1)` of VizierGPBandit with the default Eagle optimiser at N = 50, D = 4: UCB vs MES.
e. One L-BFGS-B round (`score_grad` on 25 points) at N = 1000, D = 20 with MES.

Prints one JSON line with the card name and power limit read in the same run.  Usage:
  python tools/bench_mes.py [--reps 5]
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


def _events_ms(fn, reps, stream):
  import torch
  out = []
  for _ in range(reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    fn()
    b.record(stream)
    b.synchronize()
    out.append(a.elapsed_time(b))
  return out


def _model(n, d, seed=0):
  from vizier_b200 import gp
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, d))
  y = -np.sum((x - 0.3) ** 2, axis=1) + 0.01 * rng.normal(size=n)
  dev = gp.DeviceGP(0)
  dev.fit(x, y, gp.GPHyperParams(1.0, 0.5 * np.ones(d) * max(1.0, d / 4), 1e-3))
  return dev, float(np.max(y))


def _score_table(dev, best, m, d, reps):
  import torch
  from vizier_b200 import _lib, gp
  xs = torch.from_numpy(np.random.default_rng(1).uniform(size=(m, d))).cuda()
  radius = 0.3
  acqs = {'ucb': gp.Acquisition(1.8, True, radius),
          'ei': gp.Acquisition(1.8, True, radius, acq_fn=gp.AcqFnSpec(gp.AcqTermSpec(_lib.ACQ_EI, best_label=best,
                                                                                     exploration=0.01))),
          'mes': gp.Acquisition(1.8, True, radius, acq_fn=gp.MES)}
  res = {k: [] for k in acqs}
  out = {}
  ys = dev.mes_fit(best).cpu().numpy()
  for name, a in acqs.items():   # warm-up
    if name == 'mes':
      dev.set_mes(ys)             # back to MES after EI (set_mes copies the samples; it launches no scoring)
    out = dev.score(xs, a, out=out if out else None)
  dev.synchronize()
  for _ in range(reps):
    for name, a in acqs.items():
      if name == 'mes':
        dev.set_mes(ys)
        dev.synchronize()
      res[name] += _events_ms(lambda a=a: dev.score(xs, a, out=out), 1, dev.stream)
  route = dev.get_int('score_route')
  return {k: float(np.median(v)) for k, v in res.items()} | {'route': route}


def _designer(n, d, mes, factory=None, seed=0):
  from vizier_b200 import acquisitions as acq, vz
  from vizier_b200.designers import gp_bandit
  p = vz.ProblemStatement()
  for i in range(d):
    p.search_space.root.add_float_param(f'x{i:02d}', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='obj', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  kw = {} if factory is None else {'acquisition_optimizer_factory': factory}
  if mes:
    kw['scoring_function_factory'] = acq.MaxValueEntropySearch.scoring_fn_factory
  des = gp_bandit.VizierGPBandit.from_problem(p, seed=seed, **kw)
  rng = np.random.default_rng(seed)
  trials = []
  for _ in range(n):
    x = rng.uniform(size=d)
    tr = vz.Trial(parameters={f'x{i:02d}': float(x[i]) for i in range(d)})
    tr.complete(vz.Measurement({'obj': float(-np.sum((x - 0.3) ** 2) + 0.01 * rng.normal())}))
    trials.append(tr)
  des.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  return des


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=5)
  args = ap.parse_args()
  import torch
  from vizier_b200 import gp
  out = {'card': _card()}
  dev, best = _model(1000, 20)
  dev.set_int('score_i8', 0)
  out['a_c2_score_ms'] = _score_table(dev, best, 100_000, 20, args.reps)
  out['b_small_pool_ms'] = _score_table(dev, best, 512, 20, max(args.reps, 20))
  for n in (50, 1000):
    dv, bl = (dev, best) if n == 1000 else _model(n, 20)
    dv.mes_fit(bl)
    dv.synchronize()
    out[f'c_mes_fit_N{n}_ms'] = float(np.median(_events_ms(lambda dv=dv, bl=bl: dv.mes_fit(bl), max(args.reps, 10),
                                                          dv.stream)))
  for name in ('ucb', 'mes'):
    des = _designer(50, 4, name == 'mes')
    des.suggest(1)
    t0 = time.perf_counter()
    des.suggest(1)
    out[f'd_suggest_N50_D4_{name}_s'] = time.perf_counter() - t0
  xs = torch.from_numpy(np.random.default_rng(2).uniform(size=(25, 20))).cuda()
  dev.mes_fit(best)
  a = gp.Acquisition(1.8, True, 0.3, acq_fn=gp.MES)
  dev.score_grad(xs, a)
  dev.synchronize()
  out['e_lbfgsb_round_N1000_D20_mes_ms'] = float(np.median(_events_ms(
      lambda: dev.score_grad(xs, a)['_flat'].cpu(), max(args.reps, 10), dev.stream)))
  print(json.dumps(out))


if __name__ == '__main__':
  main()
