"""Cost of wide set flies (n_parallel = q points of Dc features, width q * Dc up to 1024) in the Eagle optimiser.

1. The suggest kernel alone: CUDA events around `vzgp_eagle_ask` (one k_eagle_suggest launch each, k_eagle_suggest_wide
   above 64 coordinates) over many steps of the host-stepped loop after the pool's first pass, B = 25, P = 100 and
   3000, widths 60, 80, 320 and 1024.
2. The whole set-PE optimiser (`optimize_sets`, GP-UCB-PE's default Eagle config, 75 000 evaluations) at N = 1000,
   Dc = 20, q = 3, 4, 8, 16, and at Dc = 64, q = 16 (width 1024): wall time, then a separate torch.profiler run that
   splits one run into k_eagle_suggest[_wide], the kernels of vzgp_score_set_pe, k_eagle_update, copies, and the host
   time left over.
3. `suggest(4)` of VizierGPBandit with parallel QEI at Dc = 20 (second call: the ARD fit of the first is re-used).
4. --ab LIB: k_eagle_suggest at width 60 (q = 3) and one persistent single-point Eagle run (N = 50, D = 4) with this
   build and with LIB, alternating in separate processes, to compare an older build of the library on the same card.

Prints one JSON line with the card name and power limit read in the same run.  Usage:
  python tools/bench_set_flies.py [--ab path/to/other/libvzgp.so] [--rounds 3]
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
WIDTHS = ((3, 20), (4, 20), (16, 20), (16, 64))    # (q, Dc): widths 60, 80, 320, 1024


def _card():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                          text=True, check=True).stdout.strip().splitlines()[0]
  except Exception as e:  # pylint: disable=broad-except
    return f'unknown ({e})'


def _fitted(dc, n=50, seed=0):
  from vizier_b200 import gp
  rng = np.random.default_rng(seed)
  x = rng.uniform(size=(n, dc))
  dev = gp.DeviceGP(0)
  dev.fit(x, -np.sum((x - 0.3) ** 2, axis=1), gp.GPHyperParams(1.0, np.full(dc, 0.5), 1e-3))
  return dev, x


def suggest_kernel_us(q, dc, pool, steps=200):
  """Mean k_eagle_suggest time (us) over `steps` asks after the first pass; rewards from a cheap torch expression."""
  import torch
  from vizier_b200 import _lib, gp
  dev, _ = _fitted(dc)
  nb = pool // 25
  cfg = _lib.EagleConfig(0.45, 1.5, 0.008, 0.16, 7e-5, 0.7, 0.5, 0.96, pool, 25, (nb + steps) * 25, 1.0, 30.0, 0.98, 1, q)
  se = gp.SteppedEagle(dev, cfg, 1, 7)
  total = 0.0
  for t in range(nb + steps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record(dev.stream)
    xs, _, rewards = se.ask()
    e.record(dev.stream)
    with torch.cuda.stream(dev.stream):
      rewards.copy_(-((xs - 0.3) ** 2).sum(dim=1))
    se.tell()
    if t >= nb:
      e.synchronize()
      total += s.elapsed_time(e)
  se.end()
  dev.close()
  return 1000.0 * total / steps


def _set_pe_models(n, dc, n_pend=5):
  from vizier_b200 import gp
  rng = np.random.default_rng(1)
  x = rng.uniform(size=(n + n_pend, dc))
  y = -np.sum((x[:n] - 0.3) ** 2, axis=1) + 0.05 * rng.normal(size=n)
  pg = gp.GPHyperParams(1.0, np.full(dc, 0.5), 1e-3)
  dev_a = gp.DeviceGP(0)
  dev_b = gp.DeviceGP(0, stream=dev_a.stream)
  dev_a.fit(x[:n], y, pg)
  dev_b.fit(x, np.r_[y, np.zeros(n_pend)], pg)
  pe = gp.UcbPeAcquisition(mode=1, explore_coefficient=0.5, penalty_coefficient=10.0, threshold=float(np.max(y)) - 0.1,
                           use_trust_region=True, trust_radius=0.4, tr_rows=n + n_pend)
  return dev_a, dev_b, pe


def _profiler_warmup():
  """The first profiled region of a process pays the profiler's set-up (seconds); keep it out of the splits."""
  import torch
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]):
    torch.zeros(1, device='cuda').add_(1)
    torch.cuda.synchronize()


def set_pe_run(q, n=1000, dc=20):
  from torch.profiler import ProfilerActivity, profile
  from vizier_b200 import optimizers as vb
  from vizier_b200.designers import gp_ucb_pe
  dev_a, dev_b, pe = _set_pe_models(n, dc)
  opt = vb.VectorizedOptimizer(vb.VectorizedEagleStrategyFactory(eagle_config=gp_ucb_pe.default_eagle_config), dc, 0,
                               25, 75_000)
  opt.optimize_sets(dev_a, dev_b, pe, n_parallel=q, seed=1)      # warm-up
  t0 = time.perf_counter()
  opt.optimize_sets(dev_a, dev_b, pe, n_parallel=q, seed=2)
  wall = time.perf_counter() - t0
  t0 = time.perf_counter()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    opt.optimize_sets(dev_a, dev_b, pe, n_parallel=q, seed=2)
  prof_wall = time.perf_counter() - t0
  split = {'suggest': 0.0, 'score_set_pe': 0.0, 'update': 0.0, 'copies': 0.0}
  for ev in prof.key_averages():
    if ev.device_type is None or 'CUDA' not in str(ev.device_type) or ev.count == 0:
      continue
    t = (getattr(ev, 'device_time_total', None) or getattr(ev, 'cuda_time_total', 0.0)) / 1e6
    name = ev.key
    if 'k_eagle_suggest' in name:
      split['suggest'] += t
    elif 'k_eagle_update' in name:
      split['update'] += t
    elif 'emcpy' in name.lower() or 'copy' in name.lower() or 'elementwise' in name.lower() or 'fill' in name.lower():
      split['copies'] += t
    else:
      split['score_set_pe'] += t
  split['host'] = prof_wall - sum(split.values())
  steps = (75_000 - 1) // 25 + 1
  dev_a.close()
  dev_b.close()
  return {'wall_s': round(wall, 4), 'profiled_wall_s': round(prof_wall, 4),
          'per_step_us': {k: round(1e6 * v / steps, 2) for k, v in split.items()}}


def qei_suggest4(dc=20, n=100):
  from vizier_b200 import acquisitions as acq
  from vizier_b200 import vz
  from vizier_b200.designers import gp_bandit
  p = vz.ProblemStatement()
  for i in range(dc):
    p.search_space.root.add_float_param(f'x{i}', 0.0, 1.0)
  p.metric_information.append(vz.MetricInformation(name='obj', goal=vz.ObjectiveMetricGoal.MAXIMIZE))
  des = gp_bandit.VizierGPBandit.from_problem(
      p, seed=0, scoring_function_is_parallel=True,
      scoring_function_factory=acq.bayesian_scoring_function_factory(lambda d: acq.QEI(acq.get_best_labels(d.labels))))
  rng = np.random.default_rng(5)
  trials = []
  for i in range(n):
    xv = rng.uniform(size=dc)
    t = vz.Trial(parameters={f'x{j}': float(xv[j]) for j in range(dc)}, id=i + 1)
    t.complete(vz.Measurement({'obj': float(-np.sum((xv - 0.3) ** 2))}))
    trials.append(t)
  des.update(vz.CompletedTrials(trials), vz.ActiveTrials())
  t0 = time.perf_counter()
  des.suggest(4)
  first = time.perf_counter() - t0
  t0 = time.perf_counter()
  assert len(des.suggest(4)) == 4
  return {'setup': f'N={n}, Dc={dc}, QEI, q=4, 75 000 evaluations', 'first_suggest_s': round(first, 4),
          'suggest_s': round(time.perf_counter() - t0, 4)}


def persistent_run_ms(reps=5):
  """One single-point Eagle run on the persistent route (N = 50, D = 4, 75 000 evaluations), median of reps."""
  from vizier_b200 import _lib, gp
  dev, _ = _fitted(4)
  cfg = _lib.EagleConfig(0.45, 1.5, 0.008, 0.16, 7e-5, 0.7, 0.5, 0.96, 50, 25, 75_000)
  acq = gp.Acquisition(1.8, True, 0.3)
  dev.eagle_run(cfg, acq, 1, 3)
  times = []
  for _ in range(reps):
    t0 = time.perf_counter()
    dev.eagle_run(cfg, acq, 1, 3)
    times.append(time.perf_counter() - t0)
  assert dev.get_int('eagle_route') == 0
  dev.close()
  return 1000.0 * float(np.median(times))


def _narrow_child():
  print(json.dumps({'suggest_w60_P100_us': suggest_kernel_us(3, 20, 100, steps=400),
                    'suggest_w60_P3000_us': suggest_kernel_us(3, 20, 3000, steps=100),
                    'persistent_ms': persistent_run_ms()}), flush=True)


def _ab(other_lib, rounds):
  out = {'this': [], 'other': []}
  for _ in range(rounds):
    for key, lib in (('this', None), ('other', other_lib)):
      env = dict(os.environ)
      env.pop('VZGP_LIB', None)
      if lib:
        env['VZGP_LIB'] = lib
      res = subprocess.run([sys.executable, os.path.abspath(__file__), '--narrow-child'], env=env, capture_output=True,
                           text=True, check=True)
      out[key].append(json.loads(res.stdout.strip().splitlines()[-1]))
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--ab', default=None, help='another build of libvzgp.so to alternate with at width 60')
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--narrow-child', action='store_true', help=argparse.SUPPRESS)
  args = ap.parse_args()
  if args.narrow_child:
    _narrow_child()
    return
  res = {'card': _card()}
  res['k_eagle_suggest_us'] = {f'P{p}_w{q * dc}': round(suggest_kernel_us(q, dc, p, steps=200 if p < 1000 else 60), 2)
                               for p in (100, 3000) for q, dc in WIDTHS}
  _profiler_warmup()
  res['set_pe_n1000_dc20'] = {f'q{q}': set_pe_run(q) for q in (3, 4, 8, 16)}
  res['set_pe_n1000_dc64'] = {'q16': set_pe_run(16, dc=64)}     # width 1024
  res['qei_suggest4'] = qei_suggest4()
  if args.ab:
    res['ab_width60'] = _ab(args.ab, args.rounds)
  print(json.dumps(res), flush=True)


if __name__ == '__main__':
  main()
