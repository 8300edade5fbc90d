"""k_score fits its register budget: every instance compiles for sm_90a without spills or a stack frame.

k_score runs 9 warps per SM (8 math warps and the TMA producer, __launch_bounds__(288, 1)).  The SM's
four sub-partitions hold 16 K registers each and one of them hosts 3 of the 9 warps, so ptxas caps the
kernel at 168 registers per thread.  A spill there puts local-memory traffic in the phase-1 or slab loop,
so this test compiles score.cu with the Makefile's flags plus -Xptxas -v and reads the ptxas report."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'vizier_b200', 'csrc')
INSTANCES = [f'_ZN4vzgp7k_scoreILb{linf}ELb{generic}EEEvNS_9ScoreArgsE' for linf in (0, 1) for generic in (0, 1)]
MAX_REGISTERS = 65536 // 4 // (3 * 32) // 8 * 8   # 168: 16 K registers per sub-partition, 3 warps on one of them


def _nvcc():
  for c in (os.environ.get('NVCC'), shutil.which('nvcc'),
            os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc')):
    if c and os.path.isfile(c) and os.access(c, os.X_OK):
      return c
  return None


def _makefile_flags():
  """NVFLAGS of vizier_b200/csrc/Makefile with $(ARCH) expanded and $(EXTRA) empty."""
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
  out = tmp_path_factory.mktemp('score_ptxas')
  cmd = [nvcc] + _makefile_flags() + ['-Xptxas', '-v', '-c', os.path.join(CSRC, 'score.cu'), '-o', str(out / 'score.o')]
  res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
  assert res.returncode == 0, res.stderr[-4000:]
  report = {}
  # ptxas info : Compiling entry function '<name>' for 'sm_90a'
  # ptxas info : Function properties for <name>
  #     N bytes stack frame, N bytes spill stores, N bytes spill loads
  # ptxas info : Used N registers, ...
  for m in re.finditer(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads\s*\n[^\n]*Used (\d+) registers", res.stderr):
    report[m.group(1)] = {'stack': int(m.group(2)), 'spill_stores': int(m.group(3)), 'spill_loads': int(m.group(4)),
                          'registers': int(m.group(5))}
  return report


@pytest.mark.parametrize('name', INSTANCES)
def test_k_score_has_no_spills_and_no_stack_frame(ptxas_report, name):
  assert name in ptxas_report, sorted(ptxas_report)
  r = ptxas_report[name]
  print(name, r)
  assert r['spill_stores'] == 0 and r['spill_loads'] == 0, r
  assert r['stack'] == 0, r
  assert r['registers'] <= MAX_REGISTERS, r
