"""Records seeded host-stepped Eagle runs on the fly widths D <= 64 into tests/golden/eagle_narrow_flies.json.

Set flies wider than 64 coordinates run `k_eagle_suggest_wide`, which walks a fly in 64-column chunks; flies of at most
64 coordinates (single points, categorical features, narrow sets) stay on `k_eagle_suggest` and must compute what they
computed before wide flies existed: tests/test_gpu_set_flies.py re-runs these cases and requires the winners and their
rewards to be bit-identical to the fixture, which was written on an H100 by the library before that change.

Each case runs `gp.SteppedEagle` (k_eagle_seed_priors, k_eagle_suggest, k_eagle_update) with rewards computed on the
host by `reward` from the batch the device suggested, so the fixture depends on the optimiser's kernels only.

  python tools/make_set_flies_golden.py [OUT.json]      (on an H100, after build())
"""
import dataclasses
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)


@dataclasses.dataclass(frozen=True)
class Case:
  name: str
  dc: int                 # continuous features of one point
  pool: int
  batch: int
  steps: int
  count: int
  q: int = 1              # n_parallel: points per fly
  sizes: tuple = ()       # categorical feature sizes
  norm: int = 0           # mutate_normalization_type: 0 MEAN, 1 RANDOM
  n_prior: int = 0        # prior flies
  seed: int = 13


CASES = [
    Case('q1-categorical', 5, 50, 25, 40, 6, sizes=(3, 7, 2, 40), n_prior=30),
    Case('q1-random', 8, 100, 25, 40, 6, norm=1, n_prior=20),
    Case('q1-random-D40', 40, 50, 25, 30, 4, norm=1),                  # lanes own columns lane and lane + 32
    Case('set-q3-D60', 20, 75, 25, 40, 4, q=3, n_prior=12),
    Case('set-q4-D60-random', 15, 50, 25, 30, 4, q=4, norm=1),
    Case('set-q2-D64', 32, 50, 25, 30, 3, q=2, n_prior=8),
]


def reward(case: Case, xc, xz):
  """Smooth in every continuous coordinate, a step in every categorical one."""
  out = np.zeros(xc.shape[0])
  w = 1.0 + np.arange(xc.shape[1]) % 3
  out -= np.sum(w * (xc - 0.3) ** 2, axis=1) / np.sum(w)
  if xz.shape[1]:
    out -= 0.3 * np.mean(xz != 1, axis=1)
  return out


def run(case: Case):
  """Winners (continuous [count, q * Dc], categorical [count, Dk]) and their rewards [count] of one seeded run."""
  import torch
  from vizier_b200 import _lib, gp
  rng = np.random.default_rng(case.seed)
  dk = len(case.sizes)
  width = case.q * case.dc
  dev = gp.DeviceGP(0)
  try:
    n = 8
    x = rng.uniform(size=(n, case.dc))
    z = np.stack([rng.integers(0, s, size=n) for s in case.sizes], axis=1).astype(np.int32) if dk else None
    ls2 = 0.5 * np.ones(case.dc)
    dev.fit(x, rng.normal(size=n), gp.GPHyperParams(1.0, ls2, 1e-3, np.ones(dk) if dk else None), z=z)
    cfg = _lib.EagleConfig(0.45, 1.5, 0.008, 0.16, 7e-5, 0.7, 0.5, 0.96, case.pool, case.batch,
                           case.steps * case.batch, 1.0, 30.0, 0.98, case.norm, case.q)
    se = gp.SteppedEagle(dev, cfg, case.count, case.seed, n_prior=case.n_prior, cat_sizes=list(case.sizes) or None)
    if case.n_prior:
      pc = rng.uniform(size=(case.n_prior, width))
      pz = np.stack([rng.integers(0, s, size=case.n_prior) for s in case.sizes], axis=1).astype(np.int32) \
          if dk else np.zeros((case.n_prior, 0), np.int32)
      se.seed(pc, pz if dk else None, reward(case, pc, pz))
    for _ in range(case.steps):
      xs, zs, rewards = se.ask()
      with torch.cuda.stream(dev.stream):
        xc = xs.cpu().numpy()
        xz = zs.cpu().numpy() if zs is not None else np.zeros((case.batch, 0), np.int32)
        rewards.copy_(torch.from_numpy(reward(case, xc, xz)))
      se.tell()
    return se.end()
  finally:
    dev.close()


def main(out_path):
  import torch
  result = {'device': torch.cuda.get_device_name(0), 'cases': {}}
  for case in CASES:
    bc, bz, br = run(case)
    result['cases'][case.name] = {'features': [float(v).hex() for v in bc.ravel()],
                                  'categorical': [int(v) for v in bz.ravel()],
                                  'rewards': [float(v).hex() for v in br.ravel()]}
    print(case.name, br)
  os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
  with open(out_path, 'w') as f:
    json.dump(result, f, indent=1)
  print('wrote', out_path)


if __name__ == '__main__':
  main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, 'tests', 'golden', 'eagle_narrow_flies.json'))
