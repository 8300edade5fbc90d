"""Cost of categorical features past 32: the tiled (wide) kernel forms and the general scoring route against the
narrow forms at Dk = 32.

At N = 1000 trials and Dc = 4 continuous features, for each Dk in {32, 33, 64, 128, 256} (3 categories per feature):
  score    one scoring pass over 100 000 candidates (UCB; Dk = 32 takes k_score, Dk > 32 the general route 4)
  nll      one NLL + gradient evaluation (the replayed graph)
  eagle    one default Eagle loop: 75 000 evaluations, batch 25, the designer's pool size
  suggest  VizierGPBandit.suggest(1) on a study of 1000 completed trials (ARD fit + Eagle), after a warm-up suggest
The sizes alternate within each round, so drift of the card affects them alike; the median over rounds is reported in
ms, with the routes taken and the ratio of each size to Dk = 32.

Prints one JSON line with the card name and power limit read in the same run.  Usage:
  python tools/bench_wide_categorical.py [--rounds 3] [--dks 32,33,64,128,256] [--no-suggest]
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

N, DC, M = 1000, 4, 100_000


def _card():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                          text=True, check=True).stdout.strip().splitlines()[0]
  except Exception as e:  # pylint: disable=broad-except
    return f'unknown ({e})'


def _data(n, dk, seed):
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, DC))
  z = rng.integers(0, 3, size=(n, dk)).astype(np.int32)
  y = -np.sum((x - 0.3) ** 2, axis=1) - 0.3 * np.mean(z[:, :8] != 1, axis=1) + 0.01 * rng.normal(size=n)
  return x, y, z


class Case:
  def __init__(self, dk):
    import torch
    from vizier_b200 import gp
    from vizier_b200 import optimizers as vb
    self.dk = dk
    x, y, z = _data(N, dk, dk)
    self.hp = gp.GPHyperParams(1.0, np.full(DC, 0.5), 1e-3, np.full(dk, dk / 4.0))
    self.dev = gp.DeviceGP(0)
    self.dev.fit(x, y, self.hp, z=z)
    xs, _, zs = _data(M, dk, dk + 1)
    self.xs, self.zs = (torch.from_numpy(a).cuda() for a in (xs, zs))
    self.xt, self.yt, self.zt = (torch.from_numpy(a).cuda() for a in (x, y, z))
    self.nll = gp.DeviceGP(0)
    self.acq = gp.Acquisition(1.8, False, 1.0)
    opt = vb.VectorizedOptimizer(vb.VectorizedEagleStrategyFactory(), DC, dk, categorical_sizes=(3,) * dk)
    self.cfg = opt._eagle_config()   # pylint: disable=protected-access

  def score(self):
    self.dev.synchronize()
    t0 = time.perf_counter()
    self.dev.score(self.xs, self.acq, zs=self.zs)
    self.dev.synchronize()
    return (time.perf_counter() - t0) * 1e3, self.dev.get_int('score_route')

  def nll_eval(self):
    t0 = time.perf_counter()
    self.nll.loss_and_grad(self.xt, self.yt, self.hp, z=self.zt)   # returns host values: synchronous
    return (time.perf_counter() - t0) * 1e3, self.nll.get_int('nll_route')

  def eagle(self):
    self.dev.synchronize()
    t0 = time.perf_counter()
    self.dev.eagle_run(self.cfg, self.acq, 1, 7, cat_sizes=(3,) * self.dk)   # ends in a sync
    return (time.perf_counter() - t0) * 1e3, self.dev.get_int('eagle_route')

  def close(self):
    self.dev.close()
    self.nll.close()


def _designer(dk):
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit
  p = vz.ProblemStatement()
  for i in range(DC):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  for i in range(dk):
    p.search_space.root.add_categorical_param(f'c{i}', ['a', 'b', 'c'])
  p.metric_information.append(vz.MetricInformation(name='m', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  x, y, z = _data(N, dk, 3 * dk)
  trials = []
  for t in range(N):
    params = {f'x{i}': float(x[t, i]) for i in range(DC)}
    params.update({f'c{i}': 'abc'[z[t, i]] for i in range(dk)})
    tr = vz.Trial(parameters=params, id=t + 1)
    tr.complete(vz.Measurement({'m': float(y[t])}))
    trials.append(tr)
  d = gp_bandit.VizierGPBandit(p, rng=1)
  d.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  return d


def _suggest_ms(d):
  t0 = time.perf_counter()
  d.suggest(1)
  return (time.perf_counter() - t0) * 1e3


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--dks', default='32,33,64,128,256')
  ap.add_argument('--no-suggest', action='store_true')
  args = ap.parse_args()
  import torch
  assert torch.cuda.is_available(), 'bench_wide_categorical needs a CUDA device'
  dks = [int(v) for v in args.dks.split(',')]
  out = {'card': _card(), 'N': N, 'Dc': DC, 'M': M, 'rounds': args.rounds, 'ms_median': {}, 'route': {},
         'ratio_to_dk32': {}}
  cases = {dk: Case(dk) for dk in dks}
  parts = {'score': Case.score, 'nll': Case.nll_eval, 'eagle': Case.eagle}
  times = {k: {dk: [] for dk in dks} for k in parts}
  for dk in dks:                       # warm-up: modules, workspaces, graph captures
    for f in parts.values():
      f(cases[dk])
  for _ in range(args.rounds):
    for dk in dks:
      for k, f in parts.items():
        ms, route = f(cases[dk])
        times[k][dk].append(ms)
        out['route'].setdefault(k, {})[dk] = route
  for c in cases.values():
    c.close()
  if not args.no_suggest:
    times['suggest'] = {dk: [] for dk in dks}
    designers = {dk: _designer(dk) for dk in dks}
    for dk in dks:
      _suggest_ms(designers[dk])
    for _ in range(args.rounds):
      for dk in dks:
        times['suggest'][dk].append(_suggest_ms(designers[dk]))
  for k, per in times.items():
    med = {dk: float(np.median(v)) for dk, v in per.items()}
    out['ms_median'][k] = {dk: round(v, 3) for dk, v in med.items()}
    if 32 in med:
      out['ratio_to_dk32'][k] = {dk: round(v / med[32], 3) for dk, v in med.items()}
  print(json.dumps(out), flush=True)


if __name__ == '__main__':
  main()
