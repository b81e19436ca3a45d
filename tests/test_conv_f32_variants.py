"""Every launch of the fp32 CUDA-core convolution kernels (conv_f32.cu: conv_igemm_f32; bwd_kernels.cu: conv_wgrad_f32 and
conv_dgrad_f32), by variant key, and the BatchNorm kernels at the model's channel counts.

CPU (no GPU needed):
* coverage guard: every variant key (f32_cases.variant_key) that resnet50 or resnet18, with the bi-LSTM or the MLP head,
  with option tensor_cores on or off, reaches at any batch the library accepts (tc_cases.ACCEPTED_BATCHES, 1 .. 1024) on a
  132-SM H100 SXM or a 114-SM H100 PCIe is reached by a unit case of f32_cases.CASES planned for the same SM count.  A
  failure names the missing key and the first model launch and batch that reach it;
* every plan of a unit case and of a model launch covers its output once.
-m gpu:
* each unit case through hn_conv2d impl 0 (conv) or hn_conv2d_backward (wgrad, dgrad; dgrad also accumulated in place
  through hn_conv2d) against fp64, elementwise, with the bound of gpu_utils.run_f32_conv; outputs start NaN-filled with a
  canary behind them and halo columns must equal the circular wrap bit for bit.  Worst err / bound per case and key go to
  $HN_TEST_RECORD_DIR/f32_errors.jsonl when that variable is set;
* an all-zero dz gives exactly zero weight and data gradients;
* hn_bn_forward_backward (bn_batch_stats, bn_apply_fwd, bn_bwd) against fp64, elementwise, at C = 8 .. 2048, a ragged
  channel block, a row split equal to the rows and one capped below them, train and frozen, with ReLU and with a
  residual."""
import pytest
import torch

import __graft_entry__ as entry
from horizonnet_b200 import _lib
import f32_cases as F
import gpu_utils as gu
import tc_cases as T

BACKBONES = ('resnet50', 'resnet18')
DEV = 'cuda:0'


@pytest.fixture(scope='module', autouse=True)
def _built():
    entry.build()


def _model_launches():
    for B in T.ACCEPTED_BATCHES:                          # batch outermost: a failure names the first batch of a key
        for backbone in BACKBONES:
            for use_rnn in (True, False):
                for tc in (True, False):
                    for c in F.model_launches(backbone, use_rnn, B, tc):
                        yield f"{backbone} {'rnn' if use_rnn else 'mlp'} tensor_cores={int(tc)} {c['name']} @ B={B}", c


def _model_keys(sms):
    keys = {}
    for where, c in _model_launches():
        p = F.plan(c, sms)
        assert p is not None, (where, _lib.lib().hn_last_error())
        keys.setdefault(F.variant_key(c, p), where)
    return keys


@pytest.mark.parametrize('sms', T.SM_COUNTS)
def test_unit_cases_reach_every_variant_key_of_the_model(sms):
    model = _model_keys(sms)
    cases = {F.variant_key(c, F.plan(c, sms)) for c in F.CASES}
    missing = {k: v for k, v in model.items() if k not in cases}
    assert not missing, f'{len(missing)} variant key(s) at {sms} SMs without a unit case:\n' + \
        '\n'.join(f'{F.key_dict(k)}  (e.g. {v})' for k, v in missing.items())
    print(f'fp32 kernels: {len(model)} variant keys of the model at {sms} SMs, all reached by the {len(F.CASES)} unit cases')


@pytest.mark.parametrize('sms', T.SM_COUNTS)
def test_every_plan_covers_its_output_once(sms):
    assert len({c['name'] for c in F.CASES}) == len(F.CASES)
    for c in F.CASES:
        p = F.plan(c, sms)
        assert p is not None, (c['name'], _lib.lib().hn_last_error())
        F.check_plan(c, p)
    for where, c in _model_launches():
        F.check_plan(c, F.plan(c, sms))


def test_the_census_reaches_the_large_tiles_and_the_in_place_launches():
    """The launches the model runs on 128-row tiles and in place are in the census (at 132 SMs): the LSTM input projections
    switch to 128 x 128 at B = 3, the gate recompute at B = 5 and the in-place dx accumulation at B = 9."""
    def tile(name, B):
        c = next(c for c in F.model_launches('resnet50', True, B, True) if c['name'] == name)
        return F.conv_plan(c, 132)['BM'], c['residual']
    assert tile('bi_rnn.xproj_l1', 2)[0] == 64 and tile('bi_rnn.xproj_l1', 3)[0] == 128
    assert tile('bi_rnn.gates_l1', 4) == (64, 'inplace') and tile('bi_rnn.gates_l1', 5) == (128, 'inplace')
    assert tile('bi_rnn.dx_l1_dir1', 8) == (64, 'inplace') and tile('bi_rnn.dx_l1_dir1', 9) == (128, 'inplace')
    keys = {F.variant_key(c, F.plan(c, 132)) for c in F.CASES}
    assert any(k[1] == '128x128' and k[8] == 'inplace' for k in keys)
    assert any(k[1] == '128x64' for k in keys)
    assert any(k[1] == 'wgrad64_scalar' and k[2] for k in keys)       # the stem's weight gradient over several slices


def test_unplannable_shapes_are_rejected():
    import ctypes
    out = (ctypes.c_int * 5)()
    lib = _lib.lib()
    assert lib.hn_conv_f32_plan(1, 8, 16, 24, 1, 64, 3, 3, 1, 1, 1, 1, 1, 132, out) != 0         # Cin % 16
    assert lib.hn_conv_f32_plan(1, 8, 16, 64, 0, 64, 3, 3, 1, 1, 1, 1, 1, 132, out) != 0         # pad wider than the halo
    assert lib.hn_wgrad_f32_plan(1, 8, 16, 64, 1, 62, 3, 3, 1, 1, 1, 1, 1, 132, out) != 0        # Cout % 4


# ------------------------------------------------------------------------------------------------------------------ GPU
def _record(test, c, ratio):
    key = F.key_dict(F.variant_key(c, F.plan(c, gu.device_sms())))
    gu.record('f32_errors.jsonl', {'test': test, 'case': c['name'], 'sms': gu.device_sms(), 'ratio': ratio,
                                   'key': {k: list(v) if isinstance(v, tuple) else v for k, v in key.items()}})


@pytest.mark.gpu
@pytest.mark.parametrize('c', F.CASES, ids=lambda c: c['name'])
def test_f32_variant_vs_fp64(c):
    ratio = gu.run_f32_conv(c) if c['op'] == 'conv' else gu.run_f32_backward(c)
    _record('f32', c, ratio)
    assert ratio <= 1.0, ratio


ZERO_DZ_CASES = ('r50.stem:wgrad_b1_tc', 'r50.layer1.0.conv2:wgrad_b1_f32', 'r50.layer4.0.conv2:dgrad_b3_f32',
                 'r18.ghc0.3:dgrad_b8_tc')


@pytest.mark.gpu
@pytest.mark.parametrize('name', ZERO_DZ_CASES)
def test_f32_gradients_of_a_zero_dz_are_exactly_zero(name):
    assert gu.run_f32_backward(next(c for c in F.CASES if c['name'] == name), zero_dz=True) == 0.0


# ---- BatchNorm2d (+ identity, ReLU), train-mode statistics or frozen, forward and backward: bn_batch_stats / bn_bwd run
# CL4 channel quads per block (the largest power of two <= C/4, at most 64) and split the B*H rows over
# ceil(8 * SMs / channel blocks) blocks, at most the row count.
BN_SHAPES = [
    # B, C, H, W
    (2, 8, 8, 256),         # resnet18 ghc0.3 output: CL4 = 2, one channel block, split = rows
    (2, 16, 16, 256),       # resnet18 ghc0.2 / ghc1.3
    (5, 64, 256, 16),       # stem-like C = 64 (CL4 = 16), 1280 rows: the split is capped below the rows
    (2, 512, 16, 32),       # layer4 conv2 / ghc: two channel blocks of 64 quads, split = rows
    (3, 2048, 64, 8),       # layer4 conv3 / ghc3.0 input: 8 channel blocks, 192 rows > split 132 (114 SMs: 114)
    (2, 320, 8, 16),        # ragged channel block: 80 quads = 64 + 16
]


def _bn_reference(z, gamma, beta, rm, rv, train, relu, res, dy, y_dev, factor):
    """fp64 BatchNorm forward and backward with the ReLU mask of the device's y (its own forward is checked separately)."""
    C = z.shape[1]
    v = lambda t: t.view(1, C, 1, 1)
    if train:
        mean, var = z.mean(dim=(0, 2, 3)), z.var(dim=(0, 2, 3), unbiased=False)
    else:
        mean, var = rm, rv
    invstd = 1.0 / torch.sqrt(var + 1e-5)
    s = gamma * invstd
    xhat = (z - v(mean)) * v(invstd)
    y = xhat * v(gamma) + v(beta) + (res if res is not None else 0.0)
    if relu:
        y = torch.relu(y)
    g = dy * (y_dev > 0) if relu else dy
    n = z.numel() // C
    s1, s2 = g.sum(dim=(0, 2, 3)), (g * xhat).sum(dim=(0, 2, 3))
    dz = v(s) * (g - v(s1) / n - xhat * v(s2) / n) if train else v(s) * g
    out = dict(y=y, dz=dz, dres=g, dgamma=s2, dbeta=s1, mean=mean, invstd=invstd, xhat=xhat, g=g, s=s)
    if train:
        out['rm'] = (1 - factor) * rm + factor * mean
        out['rv'] = (1 - factor) * rv + factor * var * n / (n - 1)
    return out


# bound constant of the BatchNorm checks, in units of 2^-24 of the magnitudes of each formula's terms: 3x the worst measured
# on an H100 SXM (2.6, y = relu(z * scale + shift + res); dz 2.4)
BN_C = 8.0


@pytest.mark.gpu
@pytest.mark.parametrize('shape', BN_SHAPES, ids=lambda s: 'x'.join(map(str, s)))
@pytest.mark.parametrize('train', [1, 0], ids=['train', 'frozen'])
@pytest.mark.parametrize('relu,res', [(1, False), (0, True), (1, True)], ids=['relu', 'res', 'relu_res'])
def test_batchnorm_at_model_shapes_vs_fp64(shape, train, relu, res):
    B, C, H, W = shape
    g = torch.Generator().manual_seed(B * 100000 + C * 10 + train * 2 + relu + 4 * res)
    z = torch.randn(B, C, H, W, generator=g) * (torch.rand(C, generator=g) * 3 + 0.1).view(1, C, 1, 1) + \
        torch.randn(C, generator=g).view(1, C, 1, 1)
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.1
    rm, rv = torch.randn(C, generator=g) * 0.1, torch.rand(C, generator=g) + 0.5
    r = torch.randn(B, C, H, W, generator=g) if res else None
    dy = torch.randn(B, C, H, W, generator=g) * 1e-3
    factor = 0.1
    dev = lambda t: gu.to_halo_nhwc(t, 1).to(DEV)
    zt, dyt, rt = dev(z), dev(dy), (dev(r) if res else None)
    n = zt.numel()

    def nan_buf():
        b = gu._nan_buffer(n, DEV)
        return b, b[:n].view(zt.shape)
    yb, yt = nan_buf()
    dzb, dzt = nan_buf()
    drt = torch.zeros_like(zt) if res else None
    gam, bet, rmt, rvt = gamma.to(DEV), beta.to(DEV), rm.to(DEV), rv.to(DEV)
    dgam, dbet = torch.full((C,), float('nan'), device=DEV), torch.full((C,), float('nan'), device=DEV)
    scratch, sums = torch.empty(4 * C, device=DEV), torch.zeros(3 * C, device=DEV, dtype=torch.float64)
    _lib.check(_lib.lib().hn_bn_forward_backward(
        zt.data_ptr(), B, H, W, C, gam.data_ptr(), bet.data_ptr(), rmt.data_ptr(), rvt.data_ptr(), factor, train, relu,
        rt.data_ptr() if res else None, yt.data_ptr(), dyt.data_ptr(), dzt.data_ptr(), drt.data_ptr() if res else None,
        dgam.data_ptr(), dbet.data_ptr(), scratch.data_ptr(), sums.data_ptr(), torch.cuda.current_stream().cuda_stream),
        'hn_bn_forward_backward')
    torch.cuda.synchronize()
    for name, b, t in (('y', yb, yt), ('dz', dzb, dzt)):
        gu._check_output(f'bn {shape} {name}', b, n, t, 1)
    y_dev = gu.from_halo_nhwc(yt, 1).double().cpu()
    ref = _bn_reference(z.double(), gamma.double(), beta.double(), rm.double(), rv.double(), train, relu,
                        r.double() if res else None, dy.double(), y_dev, factor)
    u, v = gu.EPS24, (lambda t: t.view(1, C, 1, 1))
    zd = z.double()
    ratios = {}
    # y = relu(z * s + (beta - mean * s) (+ res)): roundings of s, shift, the fma and the add
    ymag = (zd * v(ref['s'])).abs() + v((ref['mean'] * ref['s']).abs() + beta.double().abs()) + \
        (r.double().abs() if res else 0.0)
    ratios['y'] = gu._worst_ratio(y_dev - ref['y'], BN_C * u * ymag)
    # dz = s * (g - s1/N - xhat * s2/N)   (frozen: s * g): xhat in fp32 carries 2^-23 of (|z| + |mean|) * invstd
    xerr = (zd.abs() + v(ref['mean'].abs())) * v(ref['invstd'])
    N = zd.numel() // C
    if train:
        # the two means carry their sums' errors: 2^-24 of sum|g| and of sum|g| (|xhat| + xerr), over N
        gx = (ref['g'].abs() * (ref['xhat'].abs() + xerr)).sum(dim=(0, 2, 3)) / N
        dzmag = v(ref['s'].abs()) * (ref['g'].abs() + v(ref['g'].abs().sum(dim=(0, 2, 3))) / N +
                                     (ref['xhat'].abs() + xerr) * v(ref['dgamma'].abs() / N + gx))
    else:
        dzmag = v(ref['s'].abs()) * ref['g'].abs()
    ratios['dz'] = gu._worst_ratio(gu.from_halo_nhwc(dzt, 1).double().cpu() - ref['dz'], BN_C * u * dzmag)
    # dgamma = sum g * xhat, dbeta = sum g (fp64 sums of fp32 terms, rounded once)
    gmag = ref['g'].abs()
    ratios['dgamma'] = gu._worst_ratio(dgam.double().cpu() - ref['dgamma'],
                                       BN_C * u * (gmag * (ref['xhat'].abs() + xerr)).sum(dim=(0, 2, 3)))
    ratios['dbeta'] = gu._worst_ratio(dbet.double().cpu() - ref['dbeta'], BN_C * u * gmag.sum(dim=(0, 2, 3)))
    if res:
        assert torch.equal(gu.from_halo_nhwc(drt, 1).double().cpu(), ref['dres']), 'the identity gradient is dy masked'
    if train:
        for k, t, old in (('rm', rmt, rm), ('rv', rvt, rv)):
            mag = old.double().abs() + ref[k].abs()
            ratios[k] = gu._worst_ratio(t.double().cpu() - ref[k], BN_C * u * mag)
    else:
        assert torch.equal(rmt.cpu(), rm) and torch.equal(rvt.cpu(), rv)
    worst = max(ratios.values())
    gu.record('f32_errors.jsonl', {'test': 'bn', 'shape': list(shape), 'train': train, 'relu': relu, 'res': res,
                                   'sms': gu.device_sms(), 'ratio': worst, 'ratios': ratios})
    assert worst <= 1.0, ratios
