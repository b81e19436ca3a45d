"""No GPU: csrc/layout_cuboid.cu compiles for sm_90a with the library's flags (and its own, no FMA contraction) and
ptxas reports no register spills for any of its kernels."""
import os
import re
import shutil
import subprocess

from horizonnet_b200 import build as B


def test_layout_cuboid_kernels_build_without_spills(tmp_path):
    nvcc = shutil.which(B._nvcc())
    assert nvcc, 'nvcc not found'
    assert 'layout_cuboid.cu' in B.SOURCES
    assert '--fmad=false' in B.FILE_FLAGS['layout_cuboid.cu']
    r = subprocess.run([nvcc] + B.NVCC_FLAGS + B.FILE_FLAGS['layout_cuboid.cu'] +
                       ['-Xptxas', '-v', '-c', os.path.join(B.CSRC, 'layout_cuboid.cu'), '-o', str(tmp_path / 'c.o')],
                       capture_output=True, text=True)
    log = r.stdout + r.stderr
    assert r.returncode == 0, log
    for k in ('bound_kernel', 'pe_kernel', 'iou_kernel'):
        assert k in log, log
    assert 'sm_90a' in log, log
    spills = re.findall(r'(\d+) bytes spill stores, (\d+) bytes spill loads', log)
    assert spills, log
    assert all(s == ('0', '0') for s in spills), log
