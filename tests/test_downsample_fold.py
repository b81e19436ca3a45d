"""The downsample of each ResNet stage's block 0 folded into its conv3 (eval forward, tensor cores): one GEMM over
[t2 | x at every stride-th pixel] against [s3 W3 ; sd Wd], shift f3 + fd, no identity tensor.

No GPU: the plan of the two-source conv_tc_kernel launch (hn_conv_tc_fold_plan) covers the output once at every block-0
shape of the model, and the committed per-launch table of the folded forward matches profiles/conv_launches.py.
-m gpu: the two-source conv_tc_kernel and bott_tc_kernel, with its downsample chunk and with an identity, against fp64,
elementwise, and the whole batch-32 forward with the option fold_downsample on and off."""
import ctypes
import json
import os
import sys
import zlib

import pytest

import __graft_entry__ as entry
from horizonnet_b200 import _lib
import tc_cases as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'profiles'))
import conv_launches as C  # noqa: E402

BM = 128
# (name, B, x H, x W, Cin, Cmid, Cout, stride): the four block-0 shapes of the model, and small ones
BLOCK0 = [('layer1.0', 128, 256, 64, 64, 256, 1), ('layer2.0', 128, 256, 256, 128, 512, 2),
          ('layer3.0', 64, 128, 512, 256, 1024, 2), ('layer4.0', 32, 64, 1024, 512, 2048, 2)]
SMALL = [('images_ragged', 3, 4, 64, 128, 64, 256, 2),       # 2 output rows per image, 4 per tile: whole images, last tile half
         ('rows_s1', 2, 16, 128, 64, 64, 256, 1)]


@pytest.fixture(scope='module', autouse=True)
def _built():
    entry.build()


def fold_plan(B, H, W, Cin, Cmid, Cout, stride, sms=T.SMS):
    out = (ctypes.c_int * len(T.PLAN_FIELDS))()
    rc = _lib.lib().hn_conv_tc_fold_plan(B, H, W, Cin, Cmid, Cout, stride, sms, out)
    return dict(zip(T.PLAN_FIELDS, out)) if rc == 0 else None


def _cases():
    for name, H, W, Ci, Cm, Co, s in BLOCK0:
        for B in (1, 2, 3, 8, 32):
            yield (f'{name}_b{B}', B, H, W, Ci, Cm, Co, s)
    yield from SMALL


@pytest.mark.parametrize('sms', [132, 114])
def test_fold_plans_cover_the_output_once(sms):
    for name, B, H, W, Ci, Cm, Co, s in _cases():
        p = fold_plan(B, H, W, Ci, Cm, Co, s, sms)
        assert p is not None, (name, _lib.lib().hn_last_error())
        Ho, Wo = H // s, W // s
        assert not p['gemm_kernel'] and p['mode'] == 1 and not p['dxr'], name
        assert p['num_kc'] == (Cm + Ci) // 64 and p['parity'] == (s == 2), name
        assert p['n_tiles'] * p['BN'] == Co and p['BN'] in (64, 128), name
        assert p['M'] == B * Ho and p['tw'] * p['rows_per_tile'] == BM and p['wsegs'] * p['tw'] == Wo, name
        assert p['box_rows'] * p['box_imgs'] == p['rows_per_tile'], name
        assert (p['box_imgs'] == 1 and Ho % p['rows_per_tile'] == 0) or p['box_rows'] == Ho, name
        m_tiles = -(-p['M'] // p['rows_per_tile']) * p['wsegs']
        assert p['num_tiles'] == m_tiles * p['n_tiles'] and p['grid'] == min(p['num_tiles'], sms), name


def test_fold_plan_rejects_what_the_kernel_does_not_take():
    assert fold_plan(2, 16, 128, 64, 64, 256, 3) is None                  # stride 3
    assert fold_plan(2, 16, 48, 64, 64, 256, 2) is None                   # output W = 24: no power-of-two tile width
    assert fold_plan(2, 16, 128, 96, 64, 256, 2) is None                  # Cin % 64
    assert fold_plan(2, 16, 128, 64, 64, 96, 2) is None                   # Cout > 64, not a multiple of 128
    assert fold_plan(2, 16, 128, 64, 64, 256, 2) is not None


def test_folded_forward_drops_the_four_downsample_launches():
    plain, fold = C.expected_launches(), C.expected_launches(fold=True)
    assert len(plain) - len(fold) == 4
    assert not [n for n, _ in fold if n.endswith('.downsample')]
    folded = [(n, c) for n, c in fold if n.endswith('+downsample')]
    assert [n for n, _ in folded] == [f'layer{l}.0.conv3+downsample' for l in (2, 3, 4)]
    for _, c in folded:
        assert C.plan_of(c)['num_kc'] * 64 == c['Cin'] + c['Cmid']


def test_committed_fold_table_matches_the_plans():
    d = json.load(open(os.path.join(ROOT, 'profiles', 'h100_conv_launches_b32_pdl0_fold.json')))
    exp = C.expected_launches(fold=True)
    assert d['options'] == {'fold_downsample': 1} and d['env'].get('HN_TC_PDL') == '0' and 'H100' in d['card']
    assert [r['name'] for r in d['launches']] == [n for n, _ in exp]
    for r, (name, c) in zip(d['launches'], exp):
        if c is None:
            assert r['kernel'] == 'bott_tc_kernel'
            continue
        p = C.plan_of(c)
        assert r['kernel'] == ('gemm_tc_kernel' if p['gemm_kernel'] else f'conv_tc_kernel<{p["BN"]}>')
        assert r['num_tiles'] == p['num_tiles'] and r['grid'] == p['grid']


# ---------------------------------------------------------------------------------------------------------- GPU
def _gpu_inputs(g, B, H, W, Ci, Cm, Co, s, dev):
    import torch
    Ho, Wo = H // s, W // s
    x = torch.randn(B, Ci, H, W, generator=g)
    t2 = torch.relu(torch.randn(B, Cm, Ho, Wo, generator=g))
    w = torch.randn(Co, Cm + Ci, generator=g) / (Cm + Ci) ** 0.5
    w[:, Cm:] *= torch.rand(Co, 1, generator=g) * 2         # downsample scales unlike conv3's
    shift = torch.randn(Co, generator=g) * 0.1
    return [t.to(dev) for t in (x, t2, w, shift)]


def _fold_reference(x, t2, w, shift, Cm, s):
    """relu(t2 . W3' + x[::s, ::s] . Wd' + shift) in fp64, and |t2| . |W3'| + |x| . |Wd'|, sum |W| per output channel."""
    import torch
    xs = x.double()[:, :, ::s, ::s]
    w3, wd = w.double()[:, :Cm], w.double()[:, Cm:]
    mm = lambda a, b: torch.einsum('bchw,nc->bnhw', a, b)
    ref = torch.relu(mm(t2.double(), w3) + mm(xs, wd) + shift.double().view(1, -1, 1, 1))
    acc = mm(t2.double().abs(), w3.abs()) + mm(xs.abs(), wd.abs())
    return ref, acc, w.double().abs().sum(1).view(1, -1, 1, 1)


def _run_out(shape, dev):
    import torch
    B, Ho, Wo, Co = shape
    n = B * Ho * (Wo + 2) * Co
    buf = torch.full((n + 4096,), float('nan'), device=dev)
    buf[n:] = 12345.5
    return buf, buf[:n].view(B, Ho, Wo + 2, Co), n


def _check_out(buf, out, n):
    import torch
    assert not torch.isnan(out).any(), 'output elements left unwritten'
    assert bool((buf[n:] == 12345.5).all()), 'write past the end of the output'
    assert torch.equal(out[:, :, 0], out[:, :, -2]) and torch.equal(out[:, :, -1], out[:, :, 1]), \
        'halo columns are not the circular wrap'


GPU_FOLD = [(n, 2, H, W, Ci, Cm, Co, s) for n, H, W, Ci, Cm, Co, s in BLOCK0[1:]] + SMALL


@pytest.mark.gpu
@pytest.mark.parametrize('case', GPU_FOLD, ids=lambda c: c[0])
def test_fold_conv_vs_fp64(case):
    import torch
    import gpu_utils as gu
    name, B, H, W, Ci, Cm, Co, s = case
    dev = 'cuda:0'
    x, t2, w, shift = _gpu_inputs(torch.Generator().manual_seed(zlib.crc32(name.encode())), B, H, W, Ci, Cm, Co, s, dev)
    buf, out, n = _run_out((B, H // s, W // s, Co), dev)
    t2h, xh = gu.to_halo_nhwc(t2, 1), gu.to_halo_nhwc(x, 1)
    rc = _lib.lib().hn_conv_tc_fold(t2h.data_ptr(), xh.data_ptr(), B, H, W, Ci, Cm, Co, s, w.data_ptr(), shift.data_ptr(),
                                    out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, 'hn_conv_tc_fold')
    torch.cuda.synchronize()
    _check_out(buf, out, n)
    ref, acc, ones = _fold_reference(x, t2, w, shift, Cm, s)
    bound = gu.C_OPERAND * gu.EPS21 * acc + gu.EPS20 * ones + gu.EPS21 * ref.abs() + gu.EPS21
    ratio = gu._worst_ratio(gu.from_halo_nhwc(out, 1).double() - ref, bound)
    gu.record('tc_errors.jsonl', {'test': 'fold', 'case': name, 'ratio': ratio})
    assert ratio <= 1.0, ratio


# (name, conv3 variant, B, H, W): layer1.0 runs bott_tc_kernel with its downsample folded in, layer1.1 and 1.2 with the
# block's identity as the residual
BOTT = [('layer1.0_b1', 'fold', 1, 128, 256), ('layer1.0_b3', 'fold', 3, 128, 256), ('small', 'fold', 2, 4, 128),
        ('layer1.1_b1', 'identity', 1, 128, 256), ('layer1.1_b3', 'identity', 3, 128, 256),
        ('small_identity', 'identity', 2, 4, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize('case', BOTT, ids=lambda c: c[0])
def test_bott_tc_vs_fp64(case):
    """hn_bott_tc, both variants of the fused layer1 conv2 + conv3 kernel, against fp64 elementwise."""
    import torch
    import gpu_utils as gu
    name, variant, B, H, W = case
    C3, dev = 256, 'cuda:0'
    g = torch.Generator().manual_seed(17)
    t1 = torch.relu(torch.randn(B, 64, H, W, generator=g)).to(dev)
    w2 = (torch.randn(64, 64, 3, 3, generator=g) / 24.0).to(dev)
    s2, f2 = (torch.rand(64, generator=g) + 0.5).to(dev), (torch.randn(64, generator=g) * 0.1).to(dev)
    if variant == 'fold':
        x, _, w3, f3 = _gpu_inputs(g, B, H, W, 64, 64, C3, 1, dev)
        s3 = res = None
    else:
        w3 = (torch.randn(C3, 64, generator=g) / 8.0).to(dev)
        s3, f3 = (torch.rand(C3, generator=g) + 0.5).to(dev), (torch.randn(C3, generator=g) * 0.1).to(dev)
        res = torch.randn(B, C3, H, W, generator=g).to(dev)
        x = None
    buf, out, n = _run_out((B, H, W, C3), dev)
    t1h = gu.to_halo_nhwc(t1, 1)
    resh, xh = (gu.to_halo_nhwc(t, 1) if t is not None else None for t in (res, x))
    ptr = lambda t: t.data_ptr() if t is not None else None
    rc = _lib.lib().hn_bott_tc(t1h.data_ptr(), ptr(resh), ptr(xh), B, H, W, w2.data_ptr(), s2.data_ptr(), f2.data_ptr(),
                               w3.data_ptr(), ptr(s3), f3.data_ptr(), C3, out.data_ptr(),
                               torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, 'hn_bott_tc')
    torch.cuda.synchronize()
    _check_out(buf, out, n)
    # conv2 in fp64 with its own error bound, which conv3 carries through |W3'| (its weights on t2 in output units)
    t2 = gu.conv2d_reference(t1.double(), w2.double(), s2, f2, (1, 1), 1, 1, True)
    acc2 = gu._conv_abs(t1.double().abs(), w2.double().abs(), (1, 1), 1, 1)
    ones2 = gu._conv_abs(torch.ones_like(t1[:1].double()), w2.double().abs(), (1, 1), 1, 1)
    b2 = s2.double().abs().view(1, -1, 1, 1) * (gu.C_OPERAND * gu.EPS21 * acc2 + gu.EPS20 * ones2) + \
        gu.EPS21 * t2.abs() + gu.EPS21
    if variant == 'fold':
        ref, acc, ones = _fold_reference(x, t2, w3, f3, 64, 1)
        w3t = w3.double()[:, :64]
        bound = gu.C_OPERAND * gu.EPS21 * acc + gu.EPS20 * ones
    else:
        w4 = w3.double().view(C3, 64, 1, 1)
        ref = gu.conv2d_reference(t2, w4, s3, f3, (1, 1), 0, 0, True, res.double())
        acc = gu._conv_abs(t2.abs(), w4.abs(), (1, 1), 0, 0)
        ones = gu._conv_abs(torch.ones_like(t2[:1]), w4.abs(), (1, 1), 0, 0)
        w3t = s3.double().view(-1, 1) * w3.double()
        # accumulator terms through the BN scale, and the identity's own plane rounding (gpu_utils.run_tc_case)
        bound = s3.double().abs().view(1, -1, 1, 1) * (gu.C_OPERAND * gu.EPS21 * acc + gu.EPS20 * ones) + \
            gu.EPS21 * (res.double().abs() + 1.0)
    carried = torch.einsum('bchw,nc->bnhw', b2, w3t.abs())
    bound = bound + gu.EPS21 * ref.abs() + gu.EPS21 + carried
    ratio = gu._worst_ratio(gu.from_halo_nhwc(out, 1).double() - ref, bound)
    gu.record('tc_errors.jsonl', {'test': 'bott_' + variant, 'case': name, 'ratio': ratio})
    assert ratio <= 1.0, ratio


@pytest.mark.gpu
def test_forward_fold_on_vs_off_batch32():
    """The bench's weights and first batch.  Folding changes how the sums are rounded: the BN scales go into the fp32
    weights before the hi/lo split, and the identity is no longer rounded to planes.  Both paths stay within 1e-4 of the
    fp32 reference (test_gpu_parity.py); they differ from each other by about 5e-6 (H100), well inside that."""
    import torch
    from horizonnet_b200.model import HorizonNet
    from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas
    net = HorizonNet('resnet50', True).eval()
    net.load_state_dict(synthetic_state_dict(0, 'random'), strict=True)
    net = net.to('cuda:0')
    x = synthetic_panoramas(32, seed=1000).to('cuda:0')
    got = {}
    with torch.no_grad():
        net(x)                                      # creates the handle for batch 32
        for mode in (0, 1):
            net.set_option('fold_downsample', mode)
            bon, cor = net(x)
            got[mode] = (bon.clone(), cor.clone())
    net.check()
    for i in range(2):
        assert torch.isfinite(got[1][i]).all()
        err = (got[1][i] - got[0][i]).abs().max().item()
        print('fold on vs off max-abs', ('bon', 'cor')[i], err)
        assert err <= 1e-5, err
