"""Host logic of the tensor-core weight-gradient kernel (horizonnet_b200/csrc/wgrad_tc.cu), no GPU needed:
* hn_wgrad_tc_plan -- the tile / slice / CTA plan conv_wgrad_tc launches with -- covers every output pixel exactly once
  for every convolution of HorizonNet('resnet50') (reference model.py:73-81, 129) at several batch sizes;
* a numpy walk over that plan (TMA boxes with out-of-bounds zero fill, traversal stride 2 along H, the parity view for
  stride 2 along W, several images per tile) reproduces torch.autograd's weight gradient, i.e. the coordinates the
  kernel hands to TMA are the right ones.  (What the tensor cores do with the tiles is covered by the -m gpu tests.)"""
import ctypes
import itertools

import numpy as np
import pytest
import torch

import __graft_entry__ as entry
from horizonnet_b200 import _lib
from tc_cases import resnet50_rnn_convs
from wgrad_cases import check_plan, launch

KT = 64


@pytest.fixture(scope='module', autouse=True)
def _built():
    entry.build()


def plan(B, H, W, Ci, Co, k, stride, sms=132):
    out = (ctypes.c_int * 10)()
    p = k // 2
    rc = _lib.lib().hn_wgrad_tc_plan(B, H, W, Ci, Co, k, k, stride[0], stride[1], p, p, sms, out)
    if rc != 0:
        return None
    return dict(zip(('tw', 'rpt', 'wsegs', 'box_rows', 'imgs', 'num_kt', 'kt_per_slice', 'slices', 'items', 'ctas'), out))


@pytest.mark.parametrize('B', [1, 2, 3, 8])
def test_plan_covers_every_pixel_of_every_conv_unit(B):
    _check_plan_covers_every_conv_unit(B, 132)                       # H100 SXM


@pytest.mark.parametrize('sms', [114, 148])                         # H100 PCIe, and a part with more SMs
@pytest.mark.parametrize('B', [1, 8])
def test_plan_covers_every_conv_unit_at_other_sm_counts(B, sms):
    _check_plan_covers_every_conv_unit(B, sms)


def _check_plan_covers_every_conv_unit(B, sms):
    convs = resnet50_rnn_convs()
    assert len(convs) == 68
    on_tc = 0
    for name, H, W, Ci, Co, k, st in convs:
        p = plan(B, H, W, Ci, Co, k, st, sms)
        if Ci % 64 or Co % 64:
            assert p is None, name                                   # ghc0.3 (Cout = 32) stays on the fp32 kernel
            continue
        assert p is not None, (name, _lib.lib().hn_last_error())
        on_tc += 1
        check_plan(launch(name, B, H, W, Ci, Co, k, st), p)
    assert on_tc == 67


def test_plan_rejects_what_the_kernel_does_not_take():
    assert plan(2, 16, 32, 48, 64, 3, (1, 1)) is None                # Cin % 64
    assert plan(2, 512, 1024, 3, 64, 7, (2, 2)) is None              # the stem (Cin = 3): its weight gradient stays fp32
    assert plan(2, 16, 24, 64, 64, 3, (1, 1)) is None                # W = 24: not a power-of-two tile width
    assert plan(2, 6, 16, 64, 64, 3, (1, 1)) is None                 # 4 rows per tile, 6 rows per image
    assert plan(2, 16, 32, 64, 64, 3, (3, 1)) is None                # stride 3
    assert b'unsupported' in _lib.lib().hn_last_error()


def _tma_box(t, start, box, estride=None):
    """cuTensorMapEncodeTiled semantics on a numpy array indexed outermost-first; start / box innermost-first;
    out-of-bounds elements read as zero; estride = traversal stride per dimension."""
    n = t.ndim
    estride = estride or [1] * n
    idx = [[start[i] + j for j in range(0, box[i], estride[i])] for i in range(n)]
    out = np.zeros([len(idx[n - 1 - k]) for k in range(n)], t.dtype)
    for pos in itertools.product(*[range(len(idx[n - 1 - k])) for k in range(n)]):
        src = [idx[n - 1 - k][pos[k]] for k in range(n)]
        if all(0 <= src[k] < t.shape[k] for k in range(n)):
            out[pos] = t[tuple(src)]
    return out


def _walk(x, dz, k, stride, pl):
    """dW[Cout][kh][kw][Cin] by the kernel's tile walk (wgrad_tc.cu: producer warp coordinates, host-side boxes)."""
    B, Ci, H, W = x.shape
    Co, Ho = dz.shape[1], dz.shape[2]
    sh, sw = stride
    p = k // 2
    halo = lambda t: np.concatenate([t[:, :, -1:], t, t[:, :, :1]], axis=2)
    xin, dzh = halo(x.permute(0, 2, 3, 1).numpy()), halo(dz.permute(0, 2, 3, 1).numpy())      # halo-1 NHWC
    tw, rpt, wsegs, box_rows, imgs = (pl[q] for q in ('tw', 'rpt', 'wsegs', 'box_rows', 'imgs'))
    woff, parity = 1 - p, sw == 2
    strided_rows = sh == 2 and box_rows * imgs > 1
    boxrows = box_rows * 2 if strided_rows else box_rows
    rs = 2 if strided_rows else 1
    xv = xin.reshape(B, H, xin.shape[2] // 2, 2, Ci) if parity else None
    dw = np.zeros((Co, k, k, Ci))
    for dy, dx, kt in itertools.product(range(k), range(k), range(pl['num_kt'])):
        rg = kt // wsegs
        wo0, row0 = (kt - rg * wsegs) * tw, rg * rpt
        b, ho = row0 // Ho, row0 % Ho
        hin = ho * sh + dy - p
        zt = _tma_box(dzh, [0, wo0 + 1, ho, b], [Co, tw, box_rows, imgs]).reshape(-1, Co)
        if parity:
            q = dx + woff
            it = _tma_box(xv, [0, q & 1, wo0 + (q >> 1), hin, b], [Ci, 1, tw, boxrows, imgs], [1, 1, 1, rs, 1]).reshape(-1, Ci)
        else:
            it = _tma_box(xin, [0, wo0 + dx + woff, hin, b], [Ci, tw, boxrows, imgs], [1, 1, rs, 1]).reshape(-1, Ci)
        assert zt.shape[0] == KT and it.shape[0] == KT
        dw[:, dy, dx, :] += zt.T @ it
    return dw


@pytest.mark.parametrize('case', [
    (2, 8, 16, 1, (1, 1)), (1, 8, 16, 3, (2, 2)), (2, 4, 16, 1, (2, 2)), (2, 8, 16, 3, (2, 1)), (3, 2, 32, 3, (2, 1)),
    (2, 4, 128, 3, (1, 1)), (3, 4, 64, 3, (1, 1)), (3, 2, 8, 3, (1, 1)), (5, 2, 16, 3, (2, 1)), (1, 2, 32, 3, (2, 1)),
])
def test_tile_walk_reproduces_autograd(case):
    """Channel counts do not enter the pixel tiling, so the plan is taken for 64 channels and walked with 4."""
    B, H, W, k, stride = case
    C = 4
    pl = plan(B, H, W, 64, 64, k, stride)
    assert pl is not None, _lib.lib().hn_last_error()
    g = torch.Generator().manual_seed(B * 1000 + H * 10 + k)
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(C, C, k, k, generator=g, dtype=torch.float64).requires_grad_()
    p = k // 2
    xp = torch.cat([x[..., -p:], x, x[..., :p]], dim=3) if p else x
    y = torch.nn.functional.conv2d(xp, w, None, stride=stride, padding=(p, 0))
    dz = torch.randn(y.shape, generator=g, dtype=torch.float64)
    y.backward(dz)
    got = _walk(x, dz, k, stride, pl)
    assert np.abs(got - w.grad.permute(0, 2, 3, 1).numpy()).max() < 1e-10
