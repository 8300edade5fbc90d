"""Host build of k_score's branch-free Matern-5/2 (vizier_b200/csrc/matern_fast.cuh) against long double.

The header compiles as plain C++, with the MUFU.RSQ64H seed modelled by truncation to high words.  Over 1.2e7
points with d2 in [0, 2e5] (uniform in d2, log-uniform from 1e-12, uniform in s up to past 708), each of three
signal variances: the kernel value is within 4 ulp of sf2 (1 + s + s^2/3) exp(-s) evaluated in long double at
the same s, s = sqrt(5 d2) rounds like IEEE sqrt, and every s above 708 gives 0."""
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'vizier_b200', 'csrc')

HARNESS = r'''
#include "matern_fast.cuh"
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
static uint64_t st = 88172645463325252ull;
static double u01() { st ^= st << 13; st ^= st >> 7; st ^= st << 17; return (st >> 11) * (1.0 / 9007199254740992.0); }
int main(int argc, char** argv) {
  const long n = atol(argv[1]);
  const double sf2s[3] = {1.0, 2.7, 0.013};
  double worst = 0, worst_d2 = 0;
  long sqrt_off = 0, sqrt_off_big = 0, zero_above = 0, nonzero_above = 0;
  const double fixed[] = {0.0, 1e-320, 1e-101, 708.0 * 708.0 / 5, 2e5};
  for (long i = 0; i < n; ++i) {
    double d2;
    if (i < 5) d2 = fixed[i];
    else if (i % 3 == 0) d2 = 2e5 * u01();
    else if (i % 3 == 1) d2 = pow(10.0, -12 + 17.3 * u01());
    else { const double s = 720 * u01(); d2 = s * s / 5; }
    if (d2 > 2e5) d2 = 2e5;
    const double sf2 = sf2s[(i / 3) % 3];
    const double x = 5.0 * d2;
    const double s = vzgp::matern_sqrt(x), want_s = x < 1e-100 ? 0.0 : sqrt(x);
    if (s != want_s) { ++sqrt_off; if (fabs(s - want_s) > fabs(nextafter(want_s, INFINITY) - want_s)) ++sqrt_off_big; }
    const double k = vzgp::matern_of_s(s, sf2);
    if (s > 708.0) { if (k == 0.0) ++zero_above; else ++nonzero_above; continue; }
    const long double S = s;
    const long double K = (long double)sf2 * (1.0L + S + S * S / 3.0L) * expl(-S);
    const double kd = (double)K, ulp = nextafter(kd, INFINITY) - kd;
    const double e = (double)(fabsl((long double)k - K) / ulp);
    if (e > worst) { worst = e; worst_d2 = d2; }
  }
  printf("{\"max_ulp\": %.6f, \"at_d2\": %.17g, \"sqrt_off\": %ld, \"sqrt_off_more_than_1ulp\": %ld, "
         "\"zero_above_708\": %ld, \"nonzero_above_708\": %ld}\n", worst, worst_d2, sqrt_off, sqrt_off_big, zero_above,
         nonzero_above);
  return 0;
}
'''


def _compiler():
  for c in (os.environ.get('CXX'), 'g++', 'c++', 'clang++'):
    if c and shutil.which(c):
      return c
  return None


@pytest.mark.skipif(_compiler() is None, reason='no host C++ compiler')
@pytest.mark.skipif(not sys.platform.startswith('linux') or np.finfo(np.longdouble).nmant < 63,
                    reason='needs an x87 80-bit long double')
def test_matern_fast_host_within_4_ulp(tmp_path):
  src = tmp_path / 'matern_fast_host.cpp'
  exe = tmp_path / 'matern_fast_host'
  src.write_text(HARNESS)
  # no contraction: the sequence's fma are explicit, every other product and sum rounds on its own as on the GPU
  subprocess.run([_compiler(), '-O2', '-std=c++17', '-ffp-contract=off', '-I', CSRC, str(src), '-o', str(exe)], check=True)
  out = json.loads(subprocess.run([str(exe), '12000000'], check=True, capture_output=True, text=True).stdout)
  print(out)
  assert out['max_ulp'] <= 4.0, out
  assert out['nonzero_above_708'] == 0 and out['zero_above_708'] > 0, out
  # the Goldschmidt step leaves ~2^-36 relative error, the fma correction rounds like IEEE sqrt except within
  # ~2^-70 of a rounding midpoint: a handful of 1-ulp misses at most, never more than 1 ulp
  assert out['sqrt_off_more_than_1ulp'] == 0 and out['sqrt_off'] <= 5, out
