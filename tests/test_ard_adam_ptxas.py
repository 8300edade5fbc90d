"""The fused Adam ARD kernel's launch size is exactly what `vzgp_ard_adam_small_supported` counts.

`k_ard_adam_small` keeps everything it shares in dynamic shared memory, so the dynamic size the launcher requests is
the CTA's whole shared-memory footprint and the predicate that picks the fused route compares that size with the
227 KiB a CTA may use on sm_90.  This test compiles ard_adam.cu with the Makefile's flags plus -Xptxas -v and checks
that ptxas reports no static shared memory (and no spills or stack frame) for both forms; then that the predicate,
which needs no GPU, refuses the wide-categorical shapes just past the limit and accepts those within it."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'vizier_b200', 'csrc')
MAX_CTA_SMEM = 227 * 1024


def _nvcc():
  for c in (os.environ.get('NVCC'), shutil.which('nvcc'),
            os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc')):
    if c and os.path.isfile(c) and os.access(c, os.X_OK):
      return c
  return None


def _makefile_flags():
  text = open(os.path.join(CSRC, 'Makefile')).read()
  var = {m.group(1): m.group(2).strip() for m in re.finditer(r'^(\w+)\s*:=\s*(.*)$', text, re.M)}
  flags = var['NVFLAGS'].replace('$(ARCH)', var['ARCH']).replace('$(EXTRA)', '')
  assert '$(' not in flags, flags
  return flags.split()


@pytest.fixture(scope='module')
def ptxas_report(tmp_path_factory):
  nvcc = _nvcc()
  if nvcc is None:
    pytest.skip('nvcc not found')
  out = tmp_path_factory.mktemp('ard_adam_ptxas')
  cmd = [nvcc] + _makefile_flags() + ['-Xptxas', '-v', '-c', os.path.join(CSRC, 'ard_adam.cu'), '-o',
                                      str(out / 'ard_adam.o')]
  res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
  assert res.returncode == 0, res.stderr[-4000:]
  report = {}
  for m in re.finditer(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads\s*\n[^\n]*Used (\d+) registers([^\n]*)", res.stderr):
    smem = re.search(r'(\d+) bytes smem', m.group(6))
    report[m.group(1)] = {'stack': int(m.group(2)), 'spills': int(m.group(3)) + int(m.group(4)),
                          'registers': int(m.group(5)), 'static_smem': int(smem.group(1)) if smem else 0}
  return report


@pytest.mark.parametrize('wide', [0, 1])
def test_k_ard_adam_small_has_no_static_shared_memory_spills_or_stack(ptxas_report, wide):
  names = [n for n in ptxas_report if n.startswith(f'_ZN4vzgp16k_ard_adam_smallILb{wide}E')]
  assert len(names) == 1, sorted(ptxas_report)
  r = ptxas_report[names[0]]
  print(names[0], r)
  assert r['static_smem'] == 0 and r['spills'] == 0 and r['stack'] == 0, r


def _supported():
  from vizier_b200 import _lib
  if not os.path.exists(_lib.LIB_PATH):
    import __graft_entry__ as g
    g.build()
  return _lib.load().vzgp_ard_adam_small_supported


def _smem_bytes(dc, dk):
  """The launch's dynamic shared memory (ard_adam_small_smem_bytes over nll_small_smem_bytes), restated."""
  p = dc + dk + 2
  zk = 32 if dk > 32 else dk
  evaluation = 8 * (4 * 64 * 66 + 32 * 34 + dc * 66 + 6 * 64 + 8 * p) + 4 * zk * 66
  kernel_params = 8 + 8 + 2 * 64 * 8 + 32 * 8 + 8 + 8 + 16   # dc dk, sf2, inv_ls2_c, inv_ls_c, inv_ls2_k, wide, linear
  return evaluation + 8 * (4 + 10 * p + (dk if dk > 32 else 0) + 1) + kernel_params + 8


def test_supported_counts_the_whole_launch():
  supported = _supported()
  assert not supported(64, 0, 500) and not supported(64, 55, 256)   # past the limit: the host-stepped route
  assert supported(64, 64, 33) and supported(64, 20, 64) and supported(64, 1, 200)
  assert not supported(65, 3, 2) and not supported(0, 3, 2)
  for dc in (0, 1, 20, 55, 64):
    for dk in range(0, 1025, 7):
      if dc + dk == 0:
        continue
      assert bool(supported(64, dc, dk)) == (_smem_bytes(dc, dk) <= MAX_CTA_SMEM), (dc, dk, _smem_bytes(dc, dk))
