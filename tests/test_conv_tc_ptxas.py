"""What ptxas makes of the tensor-core convolution kernels (csrc/conv_tc.cu) for sm_90a, compiled with the library's own
nvcc flags.  Two properties the kernels' speed rests on and no functional test sees:

  * no C7511 ("wgmma.mma_async instructions are serialized due to insufficient register resources"): ptxas then makes
    every wgmma wait for the previous one, and no group stays in flight whatever the kernel's wait<N> says;
  * no spill in any conv_tc_kernel, conv_halo_kernel or wgrad_tc_kernel instantiation (the accumulators are
    registers; a spilled fragment costs local-memory traffic on every k-block).

Skipped where nvcc is not installed.  The compile takes about a minute."""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, 'fewshot_detection_b200', 'csrc', 'conv_tc.cu')
KERNELS = ('conv_tc_kernel', 'conv_halo_kernel', 'wgrad_tc_kernel')


def _nvcc():
    p = shutil.which('nvcc')
    if p is None and os.path.exists('/usr/local/cuda/bin/nvcc'):
        p = '/usr/local/cuda/bin/nvcc'
    return p


def _build_flags():
    spec = importlib.util.spec_from_file_location('_graft_entry_flags', os.path.join(ROOT, '__graft_entry__.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return list(mod.NVCC_FLAGS)


def test_wgmma_not_serialized_and_no_spills(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc not found')
    cmd = [nvcc] + _build_flags() + ['-Xptxas', '-v', '-c', SRC, '-o', str(tmp_path / 'conv_tc.o')]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    serialized = [l.strip() for l in r.stdout.splitlines() if 'C7511' in l]
    assert not serialized, '%d wgmma functions serialized by ptxas:\n%s' % (len(serialized), '\n'.join(serialized))
    spills, func, checked = [], None, 0
    for line in r.stdout.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            func = m.group(1)
            continue
        m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if m and func and any(k in func for k in KERNELS):
            checked += 1
            if int(m.group(1)) or int(m.group(2)):
                spills.append('%s: %s' % (func, line.strip()))
    assert checked >= len(KERNELS), 'ptxas reported no kernel of %s' % (KERNELS,)
    assert not spills, 'register spills:\n' + '\n'.join(spills)
