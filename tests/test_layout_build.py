"""No GPU: csrc/layout.cu compiles for sm_90a with the library's flags (and its own, no FMA contraction) and ptxas reports
no register spills for the layout kernel."""
import os
import re
import shutil
import subprocess

from horizonnet_b200 import build as B


def test_layout_kernel_builds_without_spills(tmp_path):
    nvcc = shutil.which(B._nvcc())
    assert nvcc, 'nvcc not found'
    assert 'layout.cu' in B.SOURCES
    r = subprocess.run([nvcc] + B.NVCC_FLAGS + B.FILE_FLAGS.get('layout.cu', []) +
                       ['-Xptxas', '-v', '-c', os.path.join(B.CSRC, 'layout.cu'), '-o', str(tmp_path / 'layout.o')],
                       capture_output=True, text=True)
    log = r.stdout + r.stderr
    assert r.returncode == 0, log
    assert 'layout_kernel' in log, log
    spills = re.findall(r'(\d+) bytes spill stores, (\d+) bytes spill loads', log)
    assert spills, log
    assert all(s == ('0', '0') for s in spills), log
