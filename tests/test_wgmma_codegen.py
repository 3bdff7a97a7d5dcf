"""CPU: what ptxas makes of the two wgmma kernels.  No GPU is needed, only nvcc.

* A call anywhere in a kernel (printf, the IEEE fp32 / fp64 division slow paths, ...) makes ptxas serialise every
  wgmma.mma_async of that kernel (warning C7510): each MMA then waits for the previous one to finish and the commit-group
  pipelining of conv_umma_kernel / wgrad_umma_kernel never takes effect.
* conv_umma_kernel's consumer warpgroups hold the accumulators in registers (setmaxnreg budget); a spill store there
  puts local-memory traffic next to the MMAs.
"""
import os
import re
import shutil
import subprocess

import pytest

from vid2vid_b200 import build as B

KERNELS = {'conv_umma.cu': 'conv_umma_kernel', 'wgrad_umma.cu': 'wgrad_umma_kernel'}


def _nvcc():
    return B.NVCC if os.path.exists(B.NVCC) else shutil.which('nvcc')


def _ptxas_report(src, tmp_path):
    out = subprocess.run([_nvcc()] + B.FLAGS + ['-Xptxas', '-v', '-c', os.path.join(B.CSRC, src), '-o', str(tmp_path / 'k.o')],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout
    return out.stdout


def _spill_stores(report):
    """{mangled function name: spill-store bytes} from ptxas -v output."""
    res, fn = {}, None
    for line in report.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            fn = m.group(1)
        m = re.search(r'(\d+) bytes spill stores', line)
        if m and fn:
            res[fn] = int(m.group(1))
            fn = None
    return res


@pytest.mark.skipif(_nvcc() is None, reason='nvcc not found')
@pytest.mark.parametrize('src', sorted(KERNELS))
def test_wgmma_kernels_are_call_free_and_do_not_spill(src, tmp_path):
    report = _ptxas_report(src, tmp_path)
    serialised = [line for line in report.splitlines() if 'C7510' in line]
    assert not serialised, 'ptxas serialises the wgmmas:\n' + '\n'.join(serialised)
    spills = {fn: n for fn, n in _spill_stores(report).items() if KERNELS[src] in fn}
    assert spills, 'no %s instantiation in the ptxas report:\n%s' % (KERNELS[src], report)
    assert all(n == 0 for n in spills.values()), spills
