"""Device time of the Pareto kernels (pareto.cu) against the NumPy oracle on the same inputs.

a. Self-frontier (`vzgp_pareto_optimal_against` with points == against, strict) and `vzgp_pareto_rank` at
   N in {10^4, 10^5}, M in {2, 8}, uniform random points.
b. `vzgp_cum_hypervolume_origin` at N = V = 10^4, M in {2, 3}: uniform points, unit directions in the positive
   orthant (as `ParetoFrontier` draws them).
Every shape is warmed up, then timed with CUDA events around `--reps` back-to-back launches on the handle's stream
(median of `--rounds`).  The device outputs are checked against oracle/pareto_oracle.py at the timed sizes; at
N = 10^5 the oracle runs on a sample of `--sample` rows (against all N rows) and its time is that of the sample.
Floors: the compares of all pairs (2 M per pair: p <= a and a > p) at one FP64 compare per FP64 lane per clock
(132 SMs x 64 lanes x the maximum SM clock), and for the hypervolume N V M divisions at that same rate (a division
takes several FP64 instructions, so this floor is loose) or its DRAM bytes at 3.35 TB/s, whichever is larger.
Prints one JSON line, with the card's name, power limit and maximum SM clock read in the same run.  Usage:
  python tools/bench_pareto.py [--reps 20] [--rounds 3] [--sample 1000]
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

HBM_BYTES_PER_S = 3.35e12
FP64_LANES_PER_SM = 64


def _card():
  out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
  name, power, clock = [s.strip() for s in out.split(',')]
  return name, power, float(clock.split()[0]) * 1e6


def _events_ms(fn, reps, rounds, stream):
  import torch
  times = []
  for _ in range(rounds):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for _ in range(reps):
      fn()
    b.record(stream)
    b.synchronize()
    times.append(a.elapsed_time(b) / reps)
  return float(np.median(times))


def _wall_s(fn):
  t = time.perf_counter()
  out = fn()
  return out, time.perf_counter() - t


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--sample', type=int, default=1000)
  args = ap.parse_args()
  import torch
  from oracle import pareto_oracle as po
  from vizier_b200 import _lib, gp
  assert torch.cuda.is_available(), 'bench_pareto.py needs a CUDA device'
  name, power, clock = _card()
  dev = gp.DeviceGP(0)
  lib, h, stream = dev._lib, dev._h, dev.stream   # pylint: disable=protected-access
  sms = dev.get_int('sm_count')
  compares_per_s = sms * FP64_LANES_PER_SM * clock
  rows = []

  for n in (10_000, 100_000):
    for m in (2, 8):
      rng = np.random.default_rng(n + m)
      pts = rng.random((n, m))
      t = torch.from_numpy(pts).cuda()
      opt = torch.empty(n, dtype=torch.uint8, device='cuda')
      rank = torch.empty(n, dtype=torch.int32, device='cuda')
      torch.cuda.synchronize()
      frontier = lambda: _lib.check('vzgp_pareto_optimal_against', lib.vzgp_pareto_optimal_against(
          h, t.data_ptr(), n, t.data_ptr(), n, m, 1, opt.data_ptr()))
      ranks = lambda: _lib.check('vzgp_pareto_rank', lib.vzgp_pareto_rank(h, t.data_ptr(), n, m, rank.data_ptr()))
      frontier(); ranks(); dev.synchronize()
      f_ms = _events_ms(frontier, args.reps, args.rounds, stream)
      r_ms = _events_ms(ranks, args.reps, args.rounds, stream)
      got_opt, got_rank = opt.cpu().numpy().astype(bool), rank.cpu().numpy()
      sample = np.arange(n) if n <= 10_000 else np.sort(rng.choice(n, size=args.sample, replace=False))
      want_opt, f_host = _wall_s(lambda: po.is_pareto_optimal_against(pts[sample], pts, strict=True))
      want_rank, r_host = _wall_s(lambda: np.sum(po.domination_matrix(pts[sample], pts, strict=True), axis=1))
      floor_ms = 2.0 * m * n * n / compares_per_s * 1e3
      rows.append({'kernel': 'self-frontier', 'n': n, 'm': m, 'device_ms': round(f_ms, 4),
                   'all_pairs_compare_floor_ms': round(floor_ms, 4), 'frontier_size': int(got_opt.sum()),
                   'oracle_rows': len(sample), 'oracle_s': round(f_host, 3),
                   'agrees': bool(np.array_equal(got_opt[sample], want_opt))})
      rows.append({'kernel': 'pareto_rank', 'n': n, 'm': m, 'device_ms': round(r_ms, 4),
                   'all_pairs_compare_floor_ms': round(floor_ms, 4), 'share_of_floor': round(floor_ms / r_ms, 3),
                   'oracle_rows': len(sample), 'oracle_s': round(r_host, 3),
                   'agrees': bool(np.array_equal(got_rank[sample], want_rank))})

  for m in (2, 3):
    n = v = 10_000
    rng = np.random.default_rng(m)
    pts = rng.uniform(0.0, 2.0, size=(n, m))
    vec = np.abs(rng.normal(size=(v, m)))
    vec /= np.linalg.norm(vec, axis=1)[:, None]
    tp, tv = torch.from_numpy(pts).cuda(), torch.from_numpy(vec).cuda()
    out = torch.empty(n, dtype=torch.float64, device='cuda')
    torch.cuda.synchronize()
    hv = lambda: _lib.check('vzgp_cum_hypervolume_origin', lib.vzgp_cum_hypervolume_origin(
        h, tp.data_ptr(), n, m, tv.data_ptr(), v, out.data_ptr()))
    hv(); dev.synchronize()
    ms = _events_ms(hv, args.reps, args.rounds, stream)
    got = out.cpu().numpy()
    want, host_s = _wall_s(lambda: po.cum_hypervolume_origin(pts, vec))
    divisions = float(n) * v * m
    ctas = -(-v // min(4096, -(-max(-(-v // (4 * sms)), 1) // 8) * 8))
    dram = 8.0 * (n * m + v * m + 2 * ctas * n + n)
    floor_ms = max(divisions / compares_per_s, dram / HBM_BYTES_PER_S) * 1e3
    rows.append({'kernel': 'cum_hypervolume', 'n': n, 'v': v, 'm': m, 'device_ms': round(ms, 4),
                 'divisions_per_s': f'{divisions / (ms * 1e-3):.3e}', 'floor_ms': round(floor_ms, 4),
                 'oracle_s': round(host_s, 3), 'max_rel_err': float(np.max(np.abs(got - want) / np.abs(want))),
                 'agrees': bool(np.allclose(got, want, rtol=1e-12, atol=0))})

  dev.close()
  print(json.dumps({'card': name, 'power_limit': power, 'max_sm_clock_hz': clock, 'sm_count': sms, 'rows': rows}))
  if not all(r['agrees'] for r in rows):
    sys.exit(1)


if __name__ == '__main__':
  main()
