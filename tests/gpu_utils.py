"""Helpers for the -m gpu tests: torch is used only to build inputs in the library's halo-NHWC
layout and to hold device memory; every computation under test goes through the C ABI."""
import ctypes
import hashlib
import json
import math
import os

import torch
import torch.nn.functional as F

from horizonnet_b200 import _lib


def to_halo_nhwc(x_nchw, halo):
    """NCHW -> [B, H, W+2*halo, C] with circular wrap columns."""
    x = x_nchw.permute(0, 2, 3, 1)
    if halo:
        x = torch.cat([x[:, :, -halo:], x, x[:, :, :halo]], dim=2)
    return x.contiguous()


def from_halo_nhwc(y, halo):
    if halo:
        y = y[:, :, halo:-halo]
    return y.permute(0, 3, 1, 2).contiguous()


def pack_weight(w_oihw):
    co, ci, kh, kw = w_oihw.shape
    return w_oihw.permute(2, 3, 1, 0).reshape(kh * kw * ci, co).contiguous()


def conv2d(x_nchw, w_oihw, scale, shift, stride, ph, pw, relu, residual_nchw=None, impl=0, in_halo=1, out_halo=1):
    """Runs hn_conv2d on cuda tensors, returns (NCHW interior, raw halo-NHWC output)."""
    lib = _lib.lib()
    dev = x_nchw.device
    B, Ci, H, W = x_nchw.shape
    Co, _, kh, kw = w_oihw.shape
    sh, sw = stride
    Ho = (H + 2 * ph - kh) // sh + 1
    Wo = (W + 2 * pw - kw) // sw + 1
    xin = to_halo_nhwc(x_nchw.float(), in_halo)
    wp = pack_weight(w_oihw.float())
    out = torch.full((B, Ho, Wo + 2 * out_halo, Co), float('nan'), device=dev)
    res = to_halo_nhwc(residual_nchw.float(), out_halo) if residual_nchw is not None else None
    stream = torch.cuda.current_stream(dev).cuda_stream
    rc = lib.hn_conv2d(xin.data_ptr(), B, H, W, Ci, in_halo, wp.data_ptr(), scale.contiguous().data_ptr(),
                       shift.contiguous().data_ptr(), res.data_ptr() if res is not None else None, Co, kh, kw, sh, sw,
                       ph, pw, int(relu), out.data_ptr(), out_halo, impl, stream)
    _lib.check(rc, 'hn_conv2d')
    torch.cuda.synchronize()
    return from_halo_nhwc(out, out_halo), out


def conv2d_reference(x, w, scale, shift, stride, ph, pw, relu, residual=None):
    """Plain PyTorch fp64 reference of the same op (circular W pad, zero H pad)."""
    x = x.double()
    if pw:
        x = torch.cat([x[..., -pw:], x, x[..., :pw]], dim=3)
    y = F.conv2d(x, w.double(), None, stride=stride, padding=(ph, 0))
    y = y * scale.double().view(1, -1, 1, 1) + shift.double().view(1, -1, 1, 1)
    if residual is not None:
        y = y + residual.double()
    if relu:
        y = F.relu(y)
    return y


def record(name, payload):
    """Appends one JSON line of measured errors to $HN_TEST_RECORD_DIR/<name> when that variable names a directory (kept
    outside the source tree, which may be read-only); without it nothing is written."""
    d = os.environ.get('HN_TEST_RECORD_DIR')
    if d and os.path.isdir(d):
        with open(os.path.join(d, name), 'a') as f:
            f.write(json.dumps(payload) + '\n')


# ---- elementwise error bound of the split-fp16 tensor-core convolution (conv_tc.cuh plane format)
# An operand v is carried as fp16 hi = fp16(v/16) and lo = fp16(v/16 - hi); the MMAs take hi*hi, hi*lo and lo*hi.
#  * operands: a normal lo leaves |v| * 2^-22 of each operand, and the dropped lo*lo is |x||w| * 2^-22 at most: 3 * 2^-22 per
#    product; fp32 accumulation in the tensor cores (256-deep segments) and in the register sum adds a few 2^-24 of the
#    magnitude sum.  C_OPERAND = 8 covers both with margin:  C_OPERAND * 2^-21 * (|x| conv |w|);
#  * activations below 2 in magnitude have a subnormal lo, i.e. an absolute resolution of 16 * 2^-25 = 2^-21 per element
#    (2^-20 with margin):  2^-20 * (1 conv |w|);
#  * both terms are in accumulator units and pass through the epilogue scale |scale|;
#  * the output: fp32 rounding, or for plane outputs the re-split (2^-22 |y|, and 2^-21 absolute below 2): 2^-21 |y|
#    (+ 2^-21 for planes); a plane residual adds its own representation error, 2^-21 (|r| + 1).
C_OPERAND = 8.0
EPS21, EPS20 = 2.0 ** -21, 2.0 ** -20


def _conv_abs(x, w, stride, ph, pw):
    if pw:
        x = torch.cat([x[..., -pw:], x, x[..., :pw]], dim=3)
    return F.conv2d(x, w, None, stride=stride, padding=(ph, 0))


def tc_case_inputs(c, dev, seed=None):
    g = torch.Generator().manual_seed(seed if seed is not None else
                                      int(hashlib.sha1(c['name'].encode()).hexdigest()[:8], 16))
    B, Ci, H, W, Co, k = c['B'], c['Cin'], c['H'], c['W'], c['Cout'], c['k']
    x = torch.randn(B, Ci, H, W, generator=g)
    w = torch.randn(Co, Ci, k, k, generator=g) / (Ci * k * k) ** 0.5
    scale = torch.rand(Co, generator=g) + 0.5
    shift = torch.randn(Co, generator=g) * 0.1
    Ho = (H + 2 * c['ph'] - k) // c['stride'][0] + 1
    Wo = (W + 2 * c['pw'] - k) // c['stride'][1] + 1
    res = torch.randn(B, Co, Ho, Wo, generator=g) if c['residual'] else None
    return [t.to(dev) if t is not None else None for t in (x, w, scale, shift, res)]


CANARY = 12345.5


def run_tc_case(c, dev='cuda:0'):
    """Runs one case of tests/tc_cases.py through hn_conv2d (impl 1, or 2 for fp32 output) and checks it against the fp64
    reference elementwise.  Returns worst err / bound; raises AssertionError on a violation."""
    lib = _lib.lib()
    x, w, scale, shift, res = tc_case_inputs(c, dev)
    B, Ci, H, W, Co, k = c['B'], c['Cin'], c['H'], c['W'], c['Cout'], c['k']
    sh, sw = c['stride']
    ph, pw, hi, ho = c['ph'], c['pw'], c['in_halo'], c['out_halo']
    Ho, Wo = (H + 2 * ph - k) // sh + 1, (W + 2 * pw - k) // sw + 1
    xin = to_halo_nhwc(x, hi)
    wp = pack_weight(w)
    n_out = B * Ho * (Wo + 2 * ho) * Co
    buf = torch.full((n_out + 4096,), float('nan'), device=dev)
    buf[n_out:] = CANARY
    out = buf[:n_out].view(B, Ho, Wo + 2 * ho, Co)
    resin = to_halo_nhwc(res, ho) if res is not None else None
    impl = 2 if c['out_f32'] else 1
    rc = lib.hn_conv2d(xin.data_ptr(), B, H, W, Ci, hi, wp.data_ptr(), scale.data_ptr(), shift.data_ptr(),
                       resin.data_ptr() if resin is not None else None, Co, k, k, sh, sw, ph, pw, int(c['relu']),
                       out.data_ptr(), ho, impl, torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(rc, 'hn_conv2d')
    torch.cuda.synchronize(dev)
    assert not torch.isnan(out).any(), f"{c['name']}: output elements left unwritten"
    assert bool((buf[n_out:] == CANARY).all()), f"{c['name']}: write past the end of the output"
    if ho:
        assert torch.equal(out[:, :, 0], out[:, :, -2]) and torch.equal(out[:, :, -1], out[:, :, 1]), \
            f"{c['name']}: halo columns are not the circular wrap"
    y = from_halo_nhwc(out, ho).double()
    xd, wd = x.double(), w.double()
    ref = conv2d_reference(xd, wd, scale, shift, (sh, sw), ph, pw, c['relu'], res.double() if res is not None else None)
    acc = _conv_abs(xd.abs(), wd.abs(), (sh, sw), ph, pw)
    ones = _conv_abs(torch.ones_like(xd[:1]), wd.abs(), (sh, sw), ph, pw)
    sc = scale.double().abs().view(1, -1, 1, 1)
    bound = sc * (C_OPERAND * EPS21 * acc + EPS20 * ones) + EPS21 * ref.abs()
    if not c['out_f32']:
        bound = bound + EPS21
    if res is not None:
        bound = bound + EPS21 * (res.double().abs() + 1.0)
    return _worst_ratio(y - ref, bound)


def _worst_ratio(diff, bound):
    """max |diff| / bound; an exact element counts 0 even where the bound is 0 (a pixel no output depends on)."""
    err = diff.abs()
    return torch.where(err == 0, torch.zeros_like(err), err / bound).max().item()


def pow2_factor(absmax):
    """conv_tc.cuh: the power of two that brings the largest magnitude of a gradient to [2^11, 2^12) before the split."""
    if not absmax > 0 or math.isinf(absmax):
        return 1.0
    e = math.frexp(absmax)[1]
    return 2.0 ** max(-100, min(100, 12 - e))


def run_dgrad_case(B, Ci, H, W, Co, k, stride, dz_scale=1.0, prefill=False, zero=False, seed=0, dev='cuda:0'):
    """hn_conv2d_dgrad_tc (the training step's tensor-core data gradient) against torch.autograd in fp64.  din starts as
    the prefill (zeros or random, circular halo) and must come back as prefill + gradient within the bound of run_tc_case
    applied to the power-of-two scaled planes of dz.  Returns worst err / bound."""
    g = torch.Generator().manual_seed(seed)
    p = k // 2
    sh, sw = stride
    Ho, Wo = (H + 2 * p - k) // sh + 1, (W + 2 * p - k) // sw + 1
    w = (torch.randn(Co, Ci, k, k, generator=g) / (Ci * k * k) ** 0.5).to(dev)
    dz = (torch.randn(B, Co, Ho, Wo, generator=g) * dz_scale).to(dev)
    if zero:
        dz.zero_()
    pre = (torch.randn(B, Ci, H, W, generator=g) if prefill else torch.zeros(B, Ci, H, W)).to(dev)
    dzin = to_halo_nhwc(dz, 1)
    n = B * H * (W + 2) * Ci
    buf = torch.full((n + 4096,), CANARY, device=dev)
    din = buf[:n].view(B, H, W + 2, Ci)
    din.copy_(to_halo_nhwc(pre, 1))
    rc = _lib.lib().hn_conv2d_dgrad_tc(B, H, W, Ci, w.data_ptr(), dzin.data_ptr(), Co, k, k, sh, sw, p, p, din.data_ptr(),
                                       torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(rc, 'hn_conv2d_dgrad_tc')
    torch.cuda.synchronize(dev)
    assert torch.isfinite(din).all(), 'non-finite data gradient'
    assert bool((buf[n:] == CANARY).all()), 'write past the end of din'
    assert torch.equal(din[:, :, 0], din[:, :, -2]) and torch.equal(din[:, :, -1], din[:, :, 1]), 'halo is not the wrap'
    got = from_halo_nhwc(din, 1).double()
    if zero:
        assert torch.equal(got, pre.double()), 'an all-zero dz must leave din exactly as it was'
        return 0.0

    def grad(wt, d):
        xv = torch.zeros(B, Ci, H, W, dtype=torch.float64, device=dev, requires_grad=True)
        _conv_abs(xv, wt, stride, p, p).backward(d)
        return xv.grad

    wd = w.double()
    ref = grad(wd, dz.double())
    acc = grad(wd.abs(), dz.double().abs())
    ones = grad(wd.abs(), torch.ones_like(dz.double()))
    f = pow2_factor(dz.abs().max().item())
    bound = C_OPERAND * EPS21 * acc + EPS20 / f * ones + EPS21 * (ref.abs() + pre.double().abs())
    return _worst_ratio(got - (pre.double() + ref), bound)


# ---- elementwise error bound of the tensor-core weight gradient (wgrad_tc.cu): dW = dz^T x over the pixel axis, both operands
# as split planes (x: fp16 hi / lo of x/16; dz: of dz * f/16 with f = pow2_factor(max|dz|)), products hi*hi + hi*lo + lo*hi
# accumulated in fp32:
#  * operands with normal lo planes leave 2^-22 |v| each, the dropped lo*lo is 2^-22 |dz||x| at most: 1.5 * 2^-21 per
#    product.  The fp32 sums -- wgmma accumulation over a slice of up to 4096 pixels in 16-pixel steps, the reduction of
#    the pixel slices with red.global.add and the final rounding -- add 2^-24 of a partial sum per step; with BN-backward
#    dz (zero mean over the pixels of each channel) the partial sums stay far below sum |dz||x|, and 6.5 * 2^-21 of it
#    leaves them 200 steps of worst-case growth.  C_WGRAD = 8 in all: C_WGRAD * 2^-21 * (|dz|^T |x|);
#  * activations below 2 in magnitude (every LSTM state) have a subnormal lo plane: 2^-25 * 16 = 2^-21 absolute per
#    element (2^-20 with margin):  2^-20 * (|dz|^T 1);
#  * small dz (a channel 2^-20 below the largest) has a subnormal lo plane too: 2^-21 / f absolute per element (2^-20 / f
#    with margin):  2^-20 / f * (1^T |x|).
# A lost cross product (hi*lo or lo*hi) leaves an error of about 2^-12 |dz||x| per pixel, i.e. 2^-12 sqrt(N) against the
# bound's 2^-18 N over N pixels of similar terms: the bound notices it below about 4000 pixels per weight, which every
# unit case has.
C_WGRAD = 8.0


def wgrad_case_inputs(c, dev, seed=None):
    """Inputs that look like the training step's: x post-ReLU (about half zeros) or an LSTM state inside (-1, 1); dz of
    zero mean with per-output-channel scales spread over 2^-20 .. 1, like BatchNorm-backward output."""
    g = torch.Generator().manual_seed(seed if seed is not None else
                                      int(hashlib.sha1(c['name'].encode()).hexdigest()[:8], 16))
    B, Ci, H, W, Co, k = c['B'], c['Cin'], c['H'], c['W'], c['Cout'], c['k']
    sh, sw = c['stride']
    Ho, Wo = (H + 2 * (k // 2) - k) // sh + 1, (W + 2 * (k // 2) - k) // sw + 1
    if c['kind'] == 'lstm':
        x = torch.rand(B, Ci, H, W, generator=g) * 2 - 1
    else:
        x = torch.relu(torch.randn(B, Ci, H, W, generator=g))
    scale = 2.0 ** (-20 * torch.rand(Co, generator=g))
    scale[torch.randint(Co, (1,), generator=g)] = 1.0
    dz = torch.randn(B, Co, Ho, Wo, generator=g) * scale.view(1, -1, 1, 1)
    return x.to(dev), dz.to(dev)


def wgrad_reference(x, dz, k, stride):
    """dW (OIHW) of the circular-W, zero-H-padded convolution, by autograd in the dtype of the inputs."""
    w = torch.zeros(dz.shape[1], x.shape[1], k, k, dtype=x.dtype, device=x.device, requires_grad=True)
    _conv_abs(x, w, stride, k // 2, k // 2).backward(dz)
    return w.grad


def run_wgrad_case(c, zero_dz=False, with_fp32=False, dev='cuda:0'):
    """Runs one case of tests/wgrad_cases.py through hn_conv2d_wgrad_tc (the training step's wgrad: plane splits, then
    wgrad_tc_kernel) and checks dW against fp64 elementwise with the bound above.  dW starts NaN-filled with a canary behind
    it.  zero_dz: dz = 0, for which dW must be exactly 0.  with_fp32: also runs hn_conv2d_backward (the fp32 CUDA-core
    weight gradient) on the same inputs under the same bound.  Returns worst err / bound (and the fp32 kernel's)."""
    lib = _lib.lib()
    x, dz = wgrad_case_inputs(c, dev)
    if zero_dz:
        dz.zero_()
    B, Ci, H, W, Co, k = c['B'], c['Cin'], c['H'], c['W'], c['Cout'], c['k']
    sh, sw = c['stride']
    p = k // 2
    xin, dzin = to_halo_nhwc(x, 1), to_halo_nhwc(dz, 1)
    st = torch.cuda.current_stream(dev).cuda_stream

    def run(fn, *args):
        n = Co * Ci * k * k
        buf = torch.full((n + 4096,), float('nan'), device=dev)
        buf[n:] = CANARY
        _lib.check(fn(*args[:-1], buf.data_ptr(), st), fn.__name__)
        torch.cuda.synchronize(dev)
        dw = buf[:n].view(Co, Ci, k, k)
        assert not torch.isnan(dw).any(), f"{c['name']}: dW elements left unwritten"
        assert bool((buf[n:] == CANARY).all()), f"{c['name']}: write past the end of dW"
        return dw.double()

    got = run(lib.hn_conv2d_wgrad_tc, xin.data_ptr(), B, H, W, Ci, dzin.data_ptr(), Co, k, k, sh, sw, p, p, None)
    if zero_dz:
        assert torch.equal(got, torch.zeros_like(got)), f"{c['name']}: an all-zero dz must give dW = 0 exactly"
        return 0.0
    xd, dzd = x.double(), dz.double()
    ref = wgrad_reference(xd, dzd, k, (sh, sw))
    acc = wgrad_reference(xd.abs(), dzd.abs(), k, (sh, sw))
    ones_x = wgrad_reference(torch.ones_like(xd[:, :1]), dzd.abs(), k, (sh, sw)).expand_as(ref)
    ones_z = wgrad_reference(xd.abs(), torch.ones_like(dzd[:, :1]), k, (sh, sw)).expand_as(ref)
    f = pow2_factor(dz.abs().max().item())
    bound = C_WGRAD * EPS21 * acc + EPS20 * ones_x + EPS20 / f * ones_z
    ratio = _worst_ratio(got - ref, bound)
    if not with_fp32:
        return ratio
    wdev = torch.zeros(Co, Ci, k, k, device=dev)
    got32 = run(lib.hn_conv2d_backward, xin.data_ptr(), B, H, W, Ci, 1, wdev.data_ptr(), dzin.data_ptr(), Co, k, k, sh, sw,
                p, p, None, None)
    return ratio, _worst_ratio(got32 - ref, bound)


# ---- elementwise error bound of the fp32 CUDA-core kernels (conv_f32.cu, conv_wgrad_f32): every product a*w is exact to
# 2^-24 and the fp32 sums add 2^-24 of a partial sum per step, so the error of an output is a multiple of 2^-24 of the
# magnitude sum sum|a*w| of its terms, times |scale|, plus the epilogue's roundings of shift, residual and the result:
#   C32 * 2^-24 * (sum|a*w| * |scale| + |shift| + |res|) + 2^-24 * |ref|.
# C32 = 48 is 3x the worst err / (2^-24 * magnitude sum) measured over the unit cases of tests/f32_cases.py on an H100 SXM
# (132 SMs, 700 W): 16, a data gradient on 128 x 128 tiles, where one dz channel at scale 1 dominates K = 1152 terms and
# each later step rounds at that magnitude (sqrt(K) growth, far below the K of the worst case); the forward convolutions
# reach 10, the weight gradients 4.  A term left out, or added twice, is worth about 2^24 / C32 bounds.
C32 = 48.0
EPS24 = 2.0 ** -24


def f32_case_inputs(shape, kind, g):
    """An input operand like the model's: 'act' post-ReLU (about half zeros), 'lstm' an LSTM state in (-1, 1), 'grad' a
    signed gradient with per-channel scales spread over 2^-20 .. 1 (dim 1 = channels)."""
    if kind == 'act':
        return torch.relu(torch.randn(*shape, generator=g))
    if kind == 'lstm':
        return torch.rand(*shape, generator=g) * 2 - 1
    s = 2.0 ** (-20 * torch.rand(shape[1], generator=g))
    s[0] = 1.0
    return torch.randn(*shape, generator=g) * s.view(1, -1, *([1] * (len(shape) - 2)))


def _seed(name):
    return int(hashlib.sha1(name.encode()).hexdigest()[:8], 16)


def _nan_buffer(n, dev):
    buf = torch.full((n + 4096,), float('nan'), device=dev)
    buf[n:] = CANARY
    return buf


def _check_output(name, buf, n, out, halo):
    assert not torch.isnan(out).any(), f'{name}: output elements left unwritten'
    assert bool((buf[n:] == CANARY).all()), f'{name}: write past the end of the output'
    if halo:
        assert torch.equal(out[:, :, 0], out[:, :, -2]) and torch.equal(out[:, :, -1], out[:, :, 1]), \
            f'{name}: halo columns are not the circular wrap'


def run_f32_conv(c, dev='cuda:0'):
    """One 'conv' case of tests/f32_cases.py through hn_conv2d impl 0 (conv_f32) against fp64, elementwise.  The output
    starts NaN-filled with a canary behind it; residual 'inplace' passes the output buffer itself as the residual, filled
    with a random tensor first (halo columns wrapped).  Returns worst err / bound."""
    g = torch.Generator().manual_seed(_seed(c['name']))
    B, Ci, H, W, Co, k = c['B'], c['Cin'], c['H'], c['W'], c['Cout'], c['k']
    (sh, sw), ph, pw, hi, ho = c['stride'], c['ph'], c['pw'], c['in_halo'], c['out_halo']
    Ho, Wo = (H + 2 * ph - k) // sh + 1, (W + 2 * pw - k) // sw + 1
    x = f32_case_inputs((B, Ci, H, W), c['kind'], g)
    w = torch.randn(Co, Ci, k, k, generator=g) / (Ci * k * k) ** 0.5
    scale, shift = torch.rand(Co, generator=g) + 0.5, torch.randn(Co, generator=g) * 0.1
    res = torch.randn(B, Co, Ho, Wo, generator=g) if c['residual'] != 'none' else None
    x, w, scale, shift = x.to(dev), w.to(dev), scale.to(dev), shift.to(dev)
    res = res.to(dev) if res is not None else None
    n = B * Ho * (Wo + 2 * ho) * Co
    buf = _nan_buffer(n, dev)
    out = buf[:n].view(B, Ho, Wo + 2 * ho, Co)
    resin = None
    if c['residual'] == 'separate':
        resin = to_halo_nhwc(res, ho)
    elif c['residual'] == 'inplace':
        out.copy_(to_halo_nhwc(res, ho))
        resin = out
    xin, wp = to_halo_nhwc(x, hi), pack_weight(w)
    rc = _lib.lib().hn_conv2d(xin.data_ptr(), B, H, W, Ci, hi, wp.data_ptr(), scale.data_ptr(), shift.data_ptr(),
                              resin.data_ptr() if resin is not None else None, Co, k, k, sh, sw, ph, pw, int(c['relu']),
                              out.data_ptr(), ho, 0, torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(rc, 'hn_conv2d')
    torch.cuda.synchronize(dev)
    _check_output(c['name'], buf, n, out, ho)
    y = from_halo_nhwc(out, ho).double()
    xd, wd = x.double(), w.double()
    rd = res.double() if res is not None else None
    ref = conv2d_reference(xd, wd, scale, shift, (sh, sw), ph, pw, c['relu'], rd)
    acc = _conv_abs(xd.abs(), wd.abs(), (sh, sw), ph, pw)
    bound = C32 * EPS24 * (acc * scale.double().abs().view(1, -1, 1, 1) + shift.double().abs().view(1, -1, 1, 1)) + \
        EPS24 * ref.abs()
    if rd is not None:
        bound = bound + C32 * EPS24 * rd.abs()
    return _worst_ratio(y - ref, bound)


def _grad_inputs(x, w, dz, stride, ph, pw):
    """(din, dW) of the circular-W, zero-H-padded convolution by autograd in the inputs' dtype."""
    xv, wv = x.clone().requires_grad_(), w.clone().requires_grad_()
    if pw:
        xp = torch.cat([xv[..., -pw:], xv, xv[..., :pw]], dim=3)
    else:
        xp = xv
    F.conv2d(xp, wv, None, stride=stride, padding=(ph, 0)).backward(dz)
    return xv.grad, wv.grad


def run_f32_backward(c, zero_dz=False, dev='cuda:0'):
    """One 'wgrad' or 'dgrad' case of tests/f32_cases.py against fp64, elementwise, under the bound of run_f32_conv with
    scale 1 and no shift.
    * wgrad: hn_conv2d_backward's weight gradient (conv_wgrad_f32) with the input in the case's halo;
    * dgrad: hn_conv2d_backward's data gradient (pack_dgrad_weight, the zero dilation of dz, conv_f32 over it into a fresh
      din), and the same transposed conv through hn_conv2d impl 0 accumulated in place into a prefilled din, as the
      training step runs it (the dilated dz and flipped weights built here).  A unit whose Cout is not a multiple of 16
      runs as the training step pads it: Cout rounded up to 16 with zero weight rows and zero dz channels, against the
      unpadded conv's gradient.
    The outputs start NaN-filled with a canary behind them.  zero_dz: dz = 0 must give exactly 0 (dgrad: exactly the
    prefill).  Returns worst err / bound."""
    g = torch.Generator().manual_seed(_seed(c['name']))
    B, Ci, H, W, Co, k = c['B'], c['Cin'], c['H'], c['W'], c['Cout'], c['k']
    (sh, sw), ph, pw = c['stride'], c['ph'], c['pw']
    Ho, Wo = (H + 2 * ph - k) // sh + 1, (W + 2 * pw - k) // sw + 1
    lib, st = _lib.lib(), torch.cuda.current_stream(dev).cuda_stream
    x = f32_case_inputs((B, Ci, H, W), c['kind'] if c['op'] == 'wgrad' else 'act', g).to(dev)
    w = (torch.randn(Co, Ci, k, k, generator=g) / (Ci * k * k) ** 0.5).to(dev)
    dz = f32_case_inputs((B, Co, Ho, Wo), 'grad', g).to(dev)
    if zero_dz:
        dz.zero_()
    xd, wd, dzd = x.double(), w.double(), dz.double()
    if c['op'] == 'wgrad':
        hi = c['in_halo']
        n = Co * Ci * k * k
        buf = _nan_buffer(n, dev)
        xin, dzin = to_halo_nhwc(x, hi), to_halo_nhwc(dz, 1)          # (kept alive until the kernels have run)
        rc = lib.hn_conv2d_backward(xin.data_ptr(), B, H, W, Ci, hi, w.data_ptr(), dzin.data_ptr(), Co, k, k, sh, sw, ph,
                                    pw, None, buf.data_ptr(), st)
        _lib.check(rc, 'hn_conv2d_backward')
        torch.cuda.synchronize(dev)
        dw = buf[:n].view(Co, Ci, k, k)
        _check_output(c['name'], buf, n, dw, 0)
        if zero_dz:
            assert torch.equal(dw, torch.zeros_like(dw)), f"{c['name']}: an all-zero dz must give dW = 0 exactly"
            return 0.0
        ref = _grad_inputs(xd, wd, dzd, (sh, sw), ph, pw)[1]
        acc = _grad_inputs(xd.abs(), wd, dzd.abs(), (sh, sw), ph, pw)[1]
        return _worst_ratio(dw.double() - ref, C32 * EPS24 * acc + EPS24 * ref.abs())
    # data gradient: Cout padded to 16 as walk_backward does
    cp = -(-Co // 16) * 16
    wpd = torch.cat([w, torch.zeros(cp - Co, Ci, k, k, device=dev)]) if cp != Co else w
    dzp = torch.cat([dz, torch.zeros(B, cp - Co, Ho, Wo, device=dev)], dim=1) if cp != Co else dz
    dzin = to_halo_nhwc(dzp, 1)
    n = B * H * (W + 2) * Ci
    buf = _nan_buffer(n, dev)
    dwbuf = torch.empty(cp * Ci * k * k, device=dev)
    xin = to_halo_nhwc(x, 1)
    rc = lib.hn_conv2d_backward(xin.data_ptr(), B, H, W, Ci, 1, wpd.data_ptr(), dzin.data_ptr(), cp, k, k,
                                sh, sw, ph, pw, buf.data_ptr(), dwbuf.data_ptr(), st)
    _lib.check(rc, 'hn_conv2d_backward')
    torch.cuda.synchronize(dev)
    din = buf[:n].view(B, H, W + 2, Ci)
    _check_output(c['name'], buf, n, din, 1)
    # in place: din += conv(dilate(dz), flip(W)) on conv_f32 with the output as its residual
    pre = torch.randn(B, Ci, H, W, generator=g).to(dev)
    buf2 = _nan_buffer(n, dev)
    acc_out = buf2[:n].view(B, H, W + 2, Ci)
    acc_out.copy_(to_halo_nhwc(pre, 1))
    dil = torch.zeros(B, cp, H, W, device=dev)
    dil[:, :, ::sh, ::sw] = dzp
    wt = wpd.transpose(0, 1).flip(2, 3)
    ones, zeros = torch.ones(Ci, device=dev), torch.zeros(Ci, device=dev)
    tph, tpw = k - 1 - ph, k - 1 - pw
    dilin, wtp = to_halo_nhwc(dil, 1), pack_weight(wt)
    rc = lib.hn_conv2d(dilin.data_ptr(), B, H, W, cp, 1, wtp.data_ptr(), ones.data_ptr(),
                       zeros.data_ptr(), acc_out.data_ptr(), Ci, k, k, 1, 1, tph, tpw, 0, acc_out.data_ptr(), 1, 0, st)
    _lib.check(rc, 'hn_conv2d')
    torch.cuda.synchronize(dev)
    _check_output(c['name'], buf2, n, acc_out, 1)
    got, got_acc = from_halo_nhwc(din, 1).double(), from_halo_nhwc(acc_out, 1).double()
    pred = pre.double()
    if zero_dz:
        assert torch.equal(got, torch.zeros_like(got)), f"{c['name']}: an all-zero dz must give din = 0 exactly"
        assert torch.equal(got_acc, pred), f"{c['name']}: an all-zero dz must leave din exactly as it was"
        return 0.0
    ref = _grad_inputs(xd, wd, dzd, (sh, sw), ph, pw)[0]
    acc = _grad_inputs(xd, wd.abs(), dzd.abs(), (sh, sw), ph, pw)[0]
    bound = C32 * EPS24 * acc + EPS24 * ref.abs()
    return max(_worst_ratio(got - ref, bound),
               _worst_ratio(got_acc - (pred + ref), bound + C32 * EPS24 * pred.abs() + EPS24 * (pred + ref).abs()))


def device_sms(dev=0):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def lstm_error(T, B, dev='cuda:0'):
    """hn_lstm_layer against an fp64 recurrence of the same inputs (test_gpu_parity.py: test_lstm_layer_vs_oracle)."""
    g = torch.Generator().manual_seed(T * 100 + B)
    xproj = torch.randn(T, B, 4096, generator=g) * 0.5
    whh = [torch.rand(2048, 512, generator=g) * 0.08 - 0.04 for _ in range(2)]
    ref = lstm_reference(xproj, whh)
    out = torch.full((T, B, 1024), float('nan'), device=dev)
    xd, w0, w1 = xproj.to(dev), whh[0].to(dev), whh[1].to(dev)
    _lib.check(_lib.lib().hn_lstm_layer(xd.data_ptr(), w0.data_ptr(), w1.data_ptr(), out.data_ptr(), T, B,
                                        torch.cuda.current_stream().cuda_stream), 'hn_lstm_layer')
    torch.cuda.synchronize()
    return (out.cpu().double() - ref).abs().max().item()


def lstm_reference(xproj, whh):
    """Both directions of one LSTM layer in fp64 from the input projection [T][B][4096]."""
    T, B = xproj.shape[:2]
    out = []
    for d in range(2):
        xp = xproj[:, :, d * 2048:(d + 1) * 2048].double()
        w = whh[d].double()
        h = torch.zeros(B, 512, dtype=torch.float64)
        c = torch.zeros(B, 512, dtype=torch.float64)
        o = torch.empty(T, B, 512, dtype=torch.float64)
        for t in (range(T - 1, -1, -1) if d else range(T)):
            i, f, gg, og = (xp[t] + h @ w.t()).chunk(4, dim=1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
            h = torch.sigmoid(og) * torch.tanh(c)
            o[t] = h
        out.append(o)
    return torch.cat(out, dim=2)


# ---- elementwise error bound of the bi-LSTM recurrence (lstm_cluster.cu), by a teacher-forced fp64 replay.
# A bound on the free-running recurrence would have to grow through W_hh exponentially.  Instead every step is replayed in
# fp64 from the kernel's own h_{t-1}: pre_t = xp_t + W h^kernel_{t-1} (all steps in one matmul), the gates and the cell scan
# from c = 0 in fp64.  The reference is driven by the kernel's h, so an error never feeds back through W; the gap between
# kernel and reference c only carries each step's local error forward, multiplied by sigma(f) <= 1.
#  * pre-activations.  W is carried as fp16 hi / lo of W * s (s = a per-row power of two that puts max|w| of the row into
#    (2^13, 2^14]), h as fp16 hi / lo of 256 h; the MMAs take hi*hi + hi*lo + lo*hi (lo*lo dropped) and the partial sums
#    (k = 16 per MMA, 4 MMAs per warp, 3 products, 8 warps) are added in fp32.  A normal lo leaves 2^-22 |v| of each operand
#    and the dropped lo*lo is 2^-22 |w h|: 1.5 * 2^-21 per product; the ~14 fp32 additions of the sum (tensor-core adds may
#    truncate) add up to about 2^-21 of the magnitude sum.  C_LSTM = 8 covers both with margin:  C_LSTM * 2^-21 * |W| |h|.
#    A subnormal lo plane has an absolute resolution of 2^-25: 2^-33 of h (256 h) and 2^-25 / s <= 2^-38 max|w_row| of w
#    (2x margin each):  2^-32 * sum|w_row| + 2^-37 * max|w_row| * sum|h|  (none at step 0, which has no product).  The
#    unscale is a power of two; fmaf(sum, unscale, xp) rounds once:  2^-23 (|xp| + |pre|) with margin.
#  * gates: each passes e_pre through its derivative at the fp64 value, plus 2^-21 relative for expf / tanhf and the
#    division of sigmoid = 1 / (1 + expf(-x)) in fp32.
#  * cell: e_c <- sigma(f) e_c + |c| e_sf + |tanh g| e_si + sigma(i) e_tg + 2^-23 (|sigma(f) c| + |sigma(i) tanh g| + |c'|)
#    (two products and a sum, or an fma, in fp32; 2x margin).
#  * output: e_h = sigma(o) (1 - tanh^2 c) e_c + |tanh c| e_so + 2^-21 sigma(o) |tanh c| + 2^-23 |h|.
# A dropped cross product (hi*lo or lo*hi) leaves about 2^-12 of |W| |h| per step, 2^9 bounds; an h_{t-2} fed in where
# h_{t-1} belongs is off by |W| |h_{t-1} - h_{t-2}|.  test_lstm_variants.py checks both against a CPU emulation of the
# kernel's arithmetic.  On an H100 SXM (80 GB HBM3, 700 W limit, 7 co-resident clusters) the worst err / bound over every
# unit case and input kind is 0.20; most worst elements sit at step 0, where pre = xp and only the fp32 gates and cell count.
C_LSTM = 8.0
LSTM_KINDS = ('init', 'trained', 'saturated', 'small')


def lstm_inputs(kind, T, B, seed):
    """xproj [T][B][4096] and W_hh [2048][512] of both directions, on the CPU:
    * init: today's distribution: W uniform in +-0.04 (PyTorch's nn.LSTM init range is 1/sqrt(512) ~ 0.044), xproj ~ N(0, 0.5);
    * trained: rows scaled by 2^-6 .. 2 (each row its own power-of-two row scale in the kernel), a few all-zero rows, rows
      with one dominant entry (the rest 2^-16 below it: subnormal lo planes), xproj ~ N(0, 3);
    * saturated: i and f pre-activations around +20 and g of either sign (fixed per column and unit), so |c| grows toward T
      and its error is carried through sigma(f) ~ 1 at every step; o around +20 in half of the columns, so h ~ +-1;
    * small: o around -9, so sigma(o) ~ 1e-4 and h ~ 1e-4, where the lo plane of 256 h is subnormal."""
    g = torch.Generator().manual_seed(seed)
    xp = torch.randn(T, B, 4096, generator=g)
    W = [torch.rand(2048, 512, generator=g) * 0.08 - 0.04 for _ in range(2)]
    if kind == 'init':
        return xp * 0.5, W
    if kind == 'trained':
        for w in W:
            w.mul_(2.0 ** (torch.rand(2048, 1, generator=g) * 7 - 6))
            rows = torch.randperm(2048, generator=g)[:16]
            w[rows[:6]] = 0.0
            for r in rows[6:]:
                w[r].mul_(2.0 ** -16)
                w[r, torch.randint(512, (1,), generator=g)] = 0.5
        return xp * 3.0, W
    xv = xp.view(T, B, 2, 4, 512)
    xv.mul_(0.5)
    if kind == 'saturated':
        xv[:, :, :, 0:2] += 20.0
        sign = torch.where(torch.rand(B, 2, 512, generator=g) < 0.5, -1.0, 1.0)
        xv[:, :, :, 2] += 1.5 * sign
        xv[:, 1::2, :, 3] += 20.0
    elif kind == 'small':
        xv[:, :, :, 3] -= 9.0
    else:
        raise ValueError(kind)
    return xp, W


def lstm_bound(h, xp, W):
    """One direction in step order: h [T][B][512] the kernel's outputs, xp [T][B][2048], W [2048][512] (any device).
    Returns (reference h, bound), fp64, of the teacher-forced replay above."""
    h, xp, W = h.double(), xp.double(), W.double()
    hprev = torch.cat([torch.zeros_like(h[:1]), h[:-1]])
    pre = xp + hprev @ W.t()
    Wa = W.abs()
    step = (torch.arange(h.shape[0], device=h.device) > 0).double().view(-1, 1, 1)
    e_pre = C_LSTM * EPS21 * (hprev.abs() @ Wa.t()) + 2.0 ** -23 * (xp.abs() + pre.abs()) + \
        step * (2.0 ** -32 * Wa.sum(1) + 2.0 ** -37 * Wa.amax(1) * hprev.abs().sum(2, keepdim=True))
    i, f, g, o = pre.chunk(4, 2)
    ei, ef, eg, eo = e_pre.chunk(4, 2)
    si, sf, tg, so = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
    esi, esf = si * (1 - si) * ei + EPS21 * si, sf * (1 - sf) * ef + EPS21 * sf
    etg, eso = (1 - tg * tg) * eg + EPS21 * tg.abs(), so * (1 - so) * eo + EPS21 * so
    c = torch.zeros_like(h[0])
    ec = torch.zeros_like(c)
    ref, bound = torch.empty_like(h), torch.empty_like(h)
    for t in range(h.shape[0]):
        fc, ig = sf[t] * c, si[t] * tg[t]
        cn = fc + ig
        ec = sf[t] * ec + c.abs() * esf[t] + tg[t].abs() * esi[t] + si[t] * etg[t] + \
            2.0 ** -23 * (fc.abs() + ig.abs() + cn.abs())
        c = cn
        tc = torch.tanh(c)
        ref[t] = so[t] * tc
        bound[t] = so[t] * (1 - tc * tc) * ec + tc.abs() * eso[t] + EPS21 * so[t] * tc.abs() + 2.0 ** -23 * ref[t].abs()
    return ref, bound


def lstm_ratio(out, xproj, W):
    """Worst err / bound of hn_lstm_layer's output [T][B][1024] over both directions (the backward one replayed from
    t = T-1 down), and the element where it occurs."""
    worst, where = 0.0, None
    for d in range(2):
        h, xp = out[..., d * 512:(d + 1) * 512], xproj[..., d * 2048:(d + 1) * 2048]
        if d:
            h, xp = h.flip(0), xp.flip(0)
        ref, bound = lstm_bound(h, xp, W[d])
        err = (h.double() - ref).abs()
        r = torch.where(err == 0, torch.zeros_like(err), err / bound)
        m = r.max().item()
        if m >= worst:
            t, b, u = (int(v) for v in torch.nonzero(r == r.max())[0])
            worst, where = m, dict(dir=d, t=(h.shape[0] - 1 - t) if d else t, col=b, unit=u)
    return worst, where


def lstm_run(xproj, W, dev='cuda:0'):
    """hn_lstm_layer on device tensors into a NaN-filled output with a canary behind it; checks that every element is
    written and finite and nothing past the end.  Returns out [T][B][1024]."""
    T, B = xproj.shape[:2]
    n = T * B * 1024
    buf = torch.full((n + 4096,), float('nan'), device=dev)
    buf[n:] = CANARY
    _lib.check(_lib.lib().hn_lstm_layer(xproj.data_ptr(), W[0].data_ptr(), W[1].data_ptr(), buf.data_ptr(), T, B,
                                        torch.cuda.current_stream(dev).cuda_stream), 'hn_lstm_layer')
    torch.cuda.synchronize(dev)
    out = buf[:n].view(T, B, 1024)
    assert not torch.isnan(out).any(), 'output elements left unwritten'
    assert torch.isfinite(out).all(), 'non-finite output'
    assert bool((buf[n:] == CANARY).all()), 'write past the end of the output'
    return out


# ---- split planes (conv_tc.cuh split_scaled / merge_scaled) emulated in torch: s = v * 2^-4 clamped to the fp16 range,
# hi = fp16(s) and lo = fp16(s - hi), both rounded to nearest even.  Returns the two int16 bit patterns.
def split_planes_torch(v):
    s = (v.float() * 0.0625).clamp(-65504.0, 65504.0)
    hi = s.half()
    lo = (s - hi.float()).half()
    return hi.view(torch.int16), lo.view(torch.int16)


def merge_planes_torch(hi, lo):
    return (hi.view(torch.float16).float() + lo.view(torch.float16).float()) * 16.0


# ---- the stem (conv_f32.cu: stem_kernel; conv_tc.cu: stem_pack_kernel + stem_tc_kernel): normalise, 7x7 stride-2 conv
# with circular W / zero H padding 3, y = conv * scale + shift (ReLU in eval, none in the training step's raw pass).
# The kernels normalise in fp32 with fp32 constants; the fp64 reference normalises the same fp32 constants in fp64, and the
# fp32 rounding of (x - mean) / std is 2^-23 |x^| at most:  2^-23 * (|x^| conv |w|) * |scale|.
# Tensor-core stem, in the terms of run_tc_case:
#  * the input plane is 16 x^ (exact), its lo plane normal above |x^| = 2^-7: 2^-22 |x^|; below, the lo plane rounds to
#    half its subnormal spacing, 2^-25 / 16 = 2^-29 of x^ (2^-27 with a 4x margin):  2^-27 * (1 conv |w|) per output;
#  * the weights are split at the per-tensor power of two 2^t of pack_weight_tc (max|w| 2^t in (2^13, 2^14]): 2^-22 |w|
#    for a normal lo, else 2^-25 2^-t < 2^-38 max|w| absolute (2^-36 with a 4x margin):  2^-36 max|w| * (|x^| conv 1);
#  * the dropped lo*lo (2^-22 |x^ w|) and the fp32 accumulation of 42 MMAs (14 K-steps x 3 products) in the tensor
#    cores, which is not round-to-nearest: with the operand terms, C_STEM_TC * 2^-21 * (|x^| conv |w|);
#  * the epilogue is one fmaf with the exact power-of-two rescale, after the accumulator's own last rounding: 2^-24 |y|
#    each.  Where the products are exact (8-bit inputs, power-of-two-scaled filters) or the scale is small and the shift
#    large, these roundings are all of the error, so the term carries the 3x margin itself:  2^-22 |y|.
# The fp32 stem (147 fmaf per output in fp32, then the epilogue fmaf): the terms of run_f32_conv's bound with its own
# constant, C_STEM_F32 * 2^-24 * (sum|a*w| * |scale| + |shift|), and the same 2^-22 |y| output term.
# Worst err / bound on an H100 80GB HBM3 at a 700 W power limit, over every stem case of tests/test_stem_pool_tail.py
# (B = 1, 2, 3 and images 0, 31, 63 of B = 64): 0.30 for the tensor cores and 0.28 for stem_kernel, both on 8-bit panoramas
# with checkpoint-like weights; 0.24 and 0.19 on the smallest-output channel of a case.  How the constants were set there:
#  * with C = 8 of the other tensor-core convolutions and the subnormal terms at 2x (2^-28, 2^-37) the tensor-core stem
#    reached 0.50 of its bound; C = 12 gave 0.35 and C = 14 0.33, both at uniform inputs near the mean, i.e. the
#    subnormal lo-plane term was the limit.  With that term at 4x the uniform cases fell to 0.21;
#  * stem_kernel reached 0.37 of the shared C32 = 48 bound, its accumulation term dominant; C_STEM_F32 = 64 gives 0.28.
X_MEAN32 = torch.tensor([0.485, 0.456, 0.406], dtype=torch.float32)
X_STD32 = torch.tensor([0.229, 0.224, 0.225], dtype=torch.float32)
EPS22, EPS23, EPS27, EPS36 = 2.0 ** -22, 2.0 ** -23, 2.0 ** -27, 2.0 ** -36
C_STEM_TC, C_STEM_F32 = 14.0, 64.0


def normalise_f32(x):
    """The kernels' normalisation (x - mean) / std in fp32 with fp32 constants, on the first 3 channels (NCHW)."""
    m, s = X_MEAN32.to(x.device).view(1, 3, 1, 1), X_STD32.to(x.device).view(1, 3, 1, 1)
    return (x[:, :3] - m) / s


def normalise_f64(x):
    m, s = X_MEAN32.to(x.device).double().view(1, 3, 1, 1), X_STD32.to(x.device).double().view(1, 3, 1, 1)
    return (x[:, :3].double() - m) / s


def stem_reference(x, w, scale, shift, relu):
    """fp64 stem of x (NCHW fp32, >= 3 channels, any H, W) with folded BN scale / shift: (ref, acc = |x^| conv |w|,
    ones = 1 conv |w| with the zero H padding, xsum = |x^| conv 1)."""
    xn, wd = normalise_f64(x), w.double()
    y = _conv_abs(xn, wd, (2, 2), 3, 3) * scale.double().view(1, -1, 1, 1) + shift.double().view(1, -1, 1, 1)
    if relu:
        y = F.relu(y)
    acc = _conv_abs(xn.abs(), wd.abs(), (2, 2), 3, 3)
    ones = _conv_abs(torch.ones_like(xn[:1]), wd.abs(), (2, 2), 3, 3)
    xsum = _conv_abs(xn.abs(), torch.ones_like(wd[:1]), (2, 2), 3, 3)
    return y, acc, ones, xsum


def stem_bound(impl, w, scale, shift, ref, acc, ones, xsum):
    sc = scale.double().abs().view(1, -1, 1, 1)
    if impl == 1:
        wmax = w.abs().max().item()
        return sc * (C_STEM_TC * EPS21 * acc + EPS23 * acc + EPS27 * ones + EPS36 * wmax * xsum) + EPS22 * ref.abs()
    return C_STEM_F32 * EPS24 * (acc * sc + shift.double().abs().view(1, -1, 1, 1)) + sc * EPS23 * acc + EPS22 * ref.abs()


def run_stem(x, w, scale, shift, relu, impl):
    """hn_stem into [B][256][514][64] whose interior starts NaN and whose halo columns hold the canary, with the canary
    behind it; checks that every interior element is written, nothing past the end, and the halo columns: the circular
    wrap (impl 0) or untouched (impl 1).  Returns the output (halo-NHWC)."""
    B, Cx = x.shape[:2]
    dev = x.device
    n = B * 256 * 514 * 64
    buf = torch.full((n + 4096,), CANARY, device=dev)
    out = buf[:n].view(B, 256, 514, 64)
    out[:, :, 1:-1] = float('nan')
    _lib.check(_lib.lib().hn_stem(x.data_ptr(), B, Cx, w.data_ptr(), scale.data_ptr(), shift.data_ptr(), int(relu), impl,
                                  out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream), 'hn_stem')
    torch.cuda.synchronize(dev)
    assert not torch.isnan(out[:, :, 1:-1]).any(), f'stem impl {impl}: output elements left unwritten'
    assert bool((buf[n:] == CANARY).all()), f'stem impl {impl}: write past the end of the output'
    if impl == 0:
        assert torch.equal(out[:, :, 0], out[:, :, -2]) and torch.equal(out[:, :, -1], out[:, :, 1]), \
            'stem impl 0: halo columns are not the circular wrap'
    else:
        assert bool((out[:, :, 0] == CANARY).all()) and bool((out[:, :, -1] == CANARY).all()), \
            'stem impl 1: a halo column was written'
    return out


def stem_ratio(out, x, w, scale, shift, relu, impl):
    """Worst err / bound of a stem output against fp64, elementwise (so each channel against its own bound), and the
    worst ratio of the channel whose outputs are smallest."""
    ref, acc, ones, xsum = stem_reference(x, w, scale, shift, relu)
    bound = stem_bound(impl, w, scale, shift, ref, acc, ones, xsum)
    err = (from_halo_nhwc(out, 1).double() - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    per_ch = r.amax(dim=(0, 2, 3))
    small = int(ref.abs().amax(dim=(0, 2, 3)).argmin())
    return r.max().item(), per_ch[small].item()
