"""No GPU: csrc/targets.cu compiles for sm_90a with the library's flags (and its own, no FMA contraction) and ptxas
reports no register spills for any of its kernels."""
import os
import re
import shutil
import subprocess

from horizonnet_b200 import build as B


def test_targets_kernels_build_without_spills(tmp_path):
    nvcc = shutil.which(B._nvcc())
    assert nvcc, 'nvcc not found'
    assert 'targets.cu' in B.SOURCES
    assert '--fmad=false' in B.FILE_FLAGS['targets.cu']
    r = subprocess.run([nvcc] + B.NVCC_FLAGS + B.FILE_FLAGS['targets.cu'] +
                       ['-Xptxas', '-v', '-c', os.path.join(B.CSRC, 'targets.cu'), '-o', str(tmp_path / 't.o')],
                       capture_output=True, text=True)
    log = r.stdout + r.stderr
    assert r.returncode == 0, log
    for k in ('occ_kernel', 'bon_kernel', 'final_kernel'):
        assert k in log, log
    assert 'sm_90a' in log, log
    spills = re.findall(r'(\d+) bytes spill stores, (\d+) bytes spill loads', log)
    assert spills, log
    assert all(s == ('0', '0') for s in spills), log
