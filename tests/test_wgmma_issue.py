"""How the wgmma kernels issue their MMAs, and bott_tc_kernel at conv3 widths other than layer1's.

No GPU: every csrc/*.cu that issues wgmma is compiled with the library's flags.  ptxas must not report C7518 ("wgmma.mma_async
instructions are serialized"): that warning means the compiler waits for each wgmma to finish before the next one
issues, in every path of the kernel.  The SASS of conv_tc_kernel<BN> and bott_tc_kernel must issue each K chunk's 12
wgmma (3 products x 4 K-steps) behind one WARPGROUP.ARRIVE.
-m gpu: hn_bott_tc against fp64 for 1, 3 and 8 conv3 n-tiles (C3 = 64, 192, 512), with an identity and with the
downsample folded in, with the bound of test_downsample_fold.test_bott_tc_vs_fp64."""
import os
import re
import shutil
import subprocess

import pytest

from horizonnet_b200 import build as B

WGMMA_SOURCES = sorted(f for f in os.listdir(B.CSRC)
                       if f.endswith('.cu') and 'wgmma_f16' in open(os.path.join(B.CSRC, f)).read())
# mangled-name fragments of the conv_tc.cu kernels whose mainloops keep a wgmma group in flight
CHECKED = ['conv_tc_kernelILi32E', 'conv_tc_kernelILi64E', 'conv_tc_kernelILi128E', 'bott_tc_kernel']


def test_the_wgmma_sources_are_found():
    assert {'conv_tc.cu', 'wgrad_tc.cu'} <= set(WGMMA_SOURCES)


@pytest.fixture(scope='module')
def compiled(tmp_path_factory):
    nvcc = shutil.which(B._nvcc())
    assert nvcc, 'nvcc not found'
    out = {}
    tmp = tmp_path_factory.mktemp('wgmma')
    for src in WGMMA_SOURCES:
        obj = str(tmp / src.replace('.cu', '.o'))
        r = subprocess.run([nvcc] + B.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(B.CSRC, src), '-o', obj],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        sass = subprocess.run([os.path.join(os.path.dirname(nvcc), 'cuobjdump'), '-sass', obj], capture_output=True,
                              text=True, check=True).stdout
        out[src] = (r.stdout + r.stderr, sass)
    return out


@pytest.mark.parametrize('src', WGMMA_SOURCES)
def test_ptxas_does_not_serialise_wgmma(compiled, src):
    log, _ = compiled[src]
    bad = [l for l in log.splitlines() if 'C7518' in l or 'wgmma.mma_async instructions are serialized' in l]
    assert not bad, '\n'.join(bad)


def _functions(sass):
    """{mangled name: SASS text} of every function in a cuobjdump -sass listing"""
    parts = re.split(r'\n\s*Function : (\S+)\n', sass)
    return dict(zip(parts[1::2], parts[2::2]))


@pytest.mark.parametrize('kernel', CHECKED)
def test_each_chunk_issues_behind_one_arrive(compiled, kernel):
    fns = {n: t for n, t in _functions(compiled['conv_tc.cu'][1]).items() if kernel in n}
    assert len(fns) == 1, sorted(fns)
    text = next(iter(fns.values()))
    hgmma, arrive = text.count('HGMMA.'), text.count('WARPGROUP.ARRIVE')
    assert arrive > 0 and hgmma >= 12 * arrive, (kernel, hgmma, arrive)


# ---------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize('C3', [64, 192, 512])
@pytest.mark.parametrize('variant', ['fold', 'identity'])
def test_bott_tc_n_tiles_vs_fp64(variant, C3):
    """Several tiles per CTA, so that the weight ring's phases run across tiles with odd and even n-tile counts."""
    import torch
    import gpu_utils as gu
    import test_downsample_fold as F
    B_, H, W, dev = 2, 128, 256, 'cuda:0'
    g = torch.Generator().manual_seed(1000 + C3)
    t1 = torch.relu(torch.randn(B_, 64, H, W, generator=g)).to(dev)
    w2 = (torch.randn(64, 64, 3, 3, generator=g) / 24.0).to(dev)
    s2, f2 = (torch.rand(64, generator=g) + 0.5).to(dev), (torch.randn(64, generator=g) * 0.1).to(dev)
    if variant == 'fold':
        x, _, w3, f3 = F._gpu_inputs(g, B_, H, W, 64, 64, C3, 1, dev)
        s3 = res = None
    else:
        w3 = (torch.randn(C3, 64, generator=g) / 8.0).to(dev)
        s3, f3 = (torch.rand(C3, generator=g) + 0.5).to(dev), (torch.randn(C3, generator=g) * 0.1).to(dev)
        res = torch.randn(B_, C3, H, W, generator=g).to(dev)
        x = None
    buf, out, n = F._run_out((B_, H, W, C3), dev)
    t1h = gu.to_halo_nhwc(t1, 1)
    resh, xh = (gu.to_halo_nhwc(t, 1) if t is not None else None for t in (res, x))
    ptr = lambda t: t.data_ptr() if t is not None else None
    rc = F._lib.lib().hn_bott_tc(t1h.data_ptr(), ptr(resh), ptr(xh), B_, H, W, w2.data_ptr(), s2.data_ptr(),
                                 f2.data_ptr(), w3.data_ptr(), ptr(s3), f3.data_ptr(), C3, out.data_ptr(),
                                 torch.cuda.current_stream().cuda_stream)
    F._lib.check(rc, 'hn_bott_tc')
    torch.cuda.synchronize()
    F._check_out(buf, out, n)
    t2 = gu.conv2d_reference(t1.double(), w2.double(), s2, f2, (1, 1), 1, 1, True)
    acc2 = gu._conv_abs(t1.double().abs(), w2.double().abs(), (1, 1), 1, 1)
    ones2 = gu._conv_abs(torch.ones_like(t1[:1].double()), w2.double().abs(), (1, 1), 1, 1)
    b2 = s2.double().abs().view(1, -1, 1, 1) * (gu.C_OPERAND * gu.EPS21 * acc2 + gu.EPS20 * ones2) + \
        gu.EPS21 * t2.abs() + gu.EPS21
    if variant == 'fold':
        ref, acc, ones = F._fold_reference(x, t2, w3, f3, 64, 1)
        w3t = w3.double()[:, :64]
        bound = gu.C_OPERAND * gu.EPS21 * acc + gu.EPS20 * ones
    else:
        w4 = w3.double().view(C3, 64, 1, 1)
        ref = gu.conv2d_reference(t2, w4, s3, f3, (1, 1), 0, 0, True, res.double())
        acc = gu._conv_abs(t2.abs(), w4.abs(), (1, 1), 0, 0)
        ones = gu._conv_abs(torch.ones_like(t2[:1]), w4.abs(), (1, 1), 0, 0)
        w3t = s3.double().view(-1, 1) * w3.double()
        bound = s3.double().abs().view(1, -1, 1, 1) * (gu.C_OPERAND * gu.EPS21 * acc + gu.EPS20 * ones) + \
            gu.EPS21 * (res.double().abs() + 1.0)
    bound = bound + gu.EPS21 * ref.abs() + gu.EPS21 + torch.einsum('bchw,nc->bnhw', b2, w3t.abs())
    ratio = gu._worst_ratio(gu.from_halo_nhwc(out, 1).double() - ref, bound)
    assert ratio <= 1.0, ratio
