"""The kernels at the two ends of the network against fp64, forward and backward, at the batches the model runs: the stem
(conv_f32.cu: stem_kernel; conv_tc.cu: stem_pack_kernel + stem_tc_kernel), the 3x3 max-pool (conv_f32.cu: maxpool_kernel;
bwd_kernels.cu: maxpool_bwd_kernel), the feature sequence (tail.cu: ghc_to_sequence_kernel; bwd_kernels.cu:
ghc_to_sequence_bwd_kernel), the linear heads (tail.cu: head_kernel; bwd_kernels.cu: head_bwd_input_kernel,
head_bwd_weight_kernel, col_sum_kernel) and the stem's weight-gradient operand (bwd_kernels.cu: stem_input_kernel), each
through the C entry point that calls the library function the model calls.

CPU (no GPU needed):
* every fp64 reference below is pinned to the oracle (oracle/horizonnet_ref.py) on a small input: the stem, the max-pool
  and its routing, the feature path and the head;
* a torch emulation of the tensor-core stem's arithmetic (the input planes as stem_pack_kernel builds them, the weight
  planes as pack_weight_tc builds them, the products hi*hi + hi*lo + lo*hi in fp32) on the border rows, a middle row and
  every column (the wrap included) stays below 0.5 of gpu_utils.stem_bound, and exceeds it with either cross product
  dropped;
* the entry points reject bad arguments before any GPU work, and the library's ABI version is 11.
-m gpu (outputs start NaN-filled with the canary of gpu_utils behind them; worst err / bound per case goes to
$HN_TEST_RECORD_DIR/stem_pool_tail.jsonl when that variable is set):
* stem, both impls, eval and raw (the training step's scale 1, shift 0, no ReLU) epilogues, B = 1, 2, 3, inputs uniform,
  8-bit panoramas with saturated and flat mid-grey blocks, and a 4-channel input whose 4th channel is NaN; weights of the
  synthetic init, checkpoint-like filters and folded BN scales over 1e-3 .. 1e2; elementwise against fp64 under
  gpu_utils.stem_bound.  stem_kernel writes the wrap columns bit for bit, stem_tc_kernel leaves them untouched.  At B = 64
  every image equals the same image run alone at B = 1, bit for bit, and images 0, 31 and 63 meet the fp64 bound;
* max-pool at [B][256][512][64], B = 1, 3, 64: the fp32 output equals F.max_pool2d exactly (signed inputs, all-negative
  borders: -inf padding, not zero), the split-plane output is the split of the fp32 output bit for bit; the backward
  routes each gradient to torch's first maximum (exact positive ties included): exact where one window routes to an
  element, within the atomic-add bound where several do, conserved per (image, channel), halo columns untouched;
* feature sequence, both backbones, B in tc_cases.BATCHES: fp32 and plane paths against fp64 (f = 1 columns exact copies),
  the backward against the fp64 adjoint with the bound of its at most 2f atomic contributions;
* heads, K = 1024 and 512, T = 256, B in tc_cases.BATCHES: forward with the [T,B,3,4] -> [B,3,T*4] scatter, drnn, dW and
  db against fp64; col_sum at the model's bias shapes; stem_input bit-identical to the fp32 normalisation at the 3-column
  circular halo."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import __graft_entry__ as entry
from horizonnet_b200 import _lib
from oracle import horizonnet_ref
import gpu_utils as gu
import tc_cases as T

DEV = 'cuda:0'
STEM_INPUTS = ('uniform', 'pano8', 'nan4')
STEM_WEIGHTS = ('init', 'ckpt', 'bnspread')
BACKBONES = {'resnet50': (32, 64, 128, 256), 'resnet18': (8, 16, 32, 64)}    # C of the 4 height-reduction outputs
# dW / db of the heads and col_sum: fp64 partial sums over row slices, each rounded to fp32 and added atomically into the
# zeroed output: one rounding per slice and one per addition, 2^-24 of at most the magnitude sum each.  Worst err / bound
# on an H100 80GB HBM3 (700 W limit): 0.09 (dW, db), 0.02 (col_sum); the forward head 0.02 and drnn 0.09 of the C32 bound.
HEAD_SLICES, COL_SUM_SLICES = 16, 64
# The max-pool backward's atomic adds and the feature sequence's fp32 interpolation, its re-split into planes and its
# atomic backward: each derived bound below counts the roundings one by one, and one rounding of the right size reaches it
# (worst measured on that H100: 1.00 of the derived bound for the max-pool backward and the sequence's plane path, 0.99
# for its fp32 path, 0.67 for its backward).  The tests take MARGIN = 3 times the derived bound.
MARGIN = 3.0


@pytest.fixture(scope='module', autouse=True)
def _built():
    entry.build()


def _record(payload):
    gu.record('stem_pool_tail.jsonl', payload)


# ------------------------------------------------------------------------------------------------------------ inputs
def stem_input(kind, B, seed, H=512, W=1024):
    """NCHW fp32 panoramas: 'uniform' U[0, 1); 'pano8' 8-bit values k / 255 with saturated 0 and 1 blocks (one on the top
    rows, one on the bottom rows across the wrap) and flat blocks at the mean's grey level (|x^| < 2^-7: subnormal lo
    planes) and at 128; 'nan4' uniform with a 4th channel of NaN."""
    g = torch.Generator().manual_seed(seed)
    if kind == 'uniform':
        return torch.rand(B, 3, H, W, generator=g)
    if kind == 'nan4':
        return torch.cat([torch.rand(B, 3, H, W, generator=g), torch.full((B, 1, H, W), float('nan'))], dim=1)
    k = torch.randint(0, 256, (B, 3, H, W), generator=g)
    grey = torch.tensor([124, 116, 104]).view(3, 1, 1)          # round(255 * mean)
    for b in range(B):
        o = int(torch.randint(0, W // 4, (1,), generator=g))
        k[b, :, :H // 12, o:o + W // 10] = 0
        k[b, :, H - H // 12:, -W // 40:] = 255
        k[b, :, H - H // 12:, :W // 40] = 255
        k[b, :, H // 3:H // 3 + H // 5, o + W // 4:o + W // 2] = grey
        k[b, :, H // 2:H // 2 + H // 8, W - W // 4 - o:W - o] = 128
    return k.float() / 255


def stem_weights(kind, seed):
    """(w OIHW [64][3][7][7], scale, shift): 'init' the synthetic kaiming init with BN-like scale / shift; 'ckpt' filters
    scaled by 2^-8 .. 1, one all-zero filter and one with a single dominant tap; 'bnspread' folded BN scales spread
    over 1e-3 .. 1e2."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(64, 3, 7, 7, generator=g) * (2.0 / (64 * 49)) ** 0.5
    scale, shift = torch.rand(64, generator=g) + 0.5, torch.randn(64, generator=g) * 0.1
    if kind == 'ckpt':
        w *= 2.0 ** (-8 * torch.rand(64, 1, 1, 1, generator=g))
        w[5] = 0.0
        w[9] *= 2.0 ** -16
        w[9, 1, 3, 2] = 0.25
    elif kind == 'bnspread':
        scale = 10.0 ** (torch.rand(64, generator=g) * 5 - 3)
        shift = torch.randn(64, generator=g) * 0.5
    return w, scale, shift


def _dev(*ts):
    return [t.to(DEV).contiguous() for t in ts]


# ------------------------------------------------------------------------------------------------------ CPU: references
def test_abi_version_and_argument_checks():
    lib = _lib.lib()
    assert lib.hn_abi_version() == 11
    nul = ctypes.c_void_p(0)
    ptrs = (ctypes.c_void_p * 4)(1, 1, 1, 1)
    assert lib.hn_feature_sequence(b'resnet34', 1, ptrs, 0, ctypes.c_void_p(1), None) == -1
    assert b'unknown backbone' in lib.hn_last_error()
    assert lib.hn_stem(ctypes.c_void_p(1), 1, 3, ctypes.c_void_p(1), ctypes.c_void_p(1), ctypes.c_void_p(1), 1, 2,
                       ctypes.c_void_p(1), None) == -1
    assert lib.hn_stem(ctypes.c_void_p(1), 1, 2, ctypes.c_void_p(1), ctypes.c_void_p(1), ctypes.c_void_p(1), 1, 0,
                       ctypes.c_void_p(1), None) == -1
    assert lib.hn_col_sum(nul, 4, 4, ctypes.c_void_p(1), None) == -1
    assert lib.hn_linear_head(*([ctypes.c_void_p(1)] * 5), 257, 1, 1024, None) == -1


def test_stem_reference_is_the_oracles_stem():
    x = stem_input('pano8', 2, 1, H=24, W=48)
    w, scale, shift = stem_weights('init', 2)
    bn = {'feature_extractor.encoder.bn1.' + k: v for k, v in
          (('weight', torch.rand(64, dtype=torch.float64) + 0.5), ('bias', torch.randn(64, dtype=torch.float64) * 0.1),
           ('running_mean', torch.randn(64, dtype=torch.float64) * 0.1),
           ('running_var', torch.rand(64, dtype=torch.float64) + 0.5))}
    p = 'feature_extractor.encoder.bn1.'
    sc = bn[p + 'weight'] / torch.sqrt(bn[p + 'running_var'] + horizonnet_ref.BN_EPS)
    sh = bn[p + 'bias'] - bn[p + 'running_mean'] * sc
    xn = gu.normalise_f64(x)
    conv = horizonnet_ref._circ_conv(xn, w.double(), None, 2, 3, 3)
    oracle = F.relu(horizonnet_ref._bn(conv, bn, p[:-1]))
    ref = gu.stem_reference(x, w, sc.float(), sh.float(), True)[0]
    # the folded constants are rounded to fp32 here (the kernels take fp32): 2^-24 relative each
    assert torch.allclose(ref, oracle, rtol=2e-7, atol=1e-7)
    assert torch.equal(gu.stem_reference(x, w, torch.ones(64), torch.zeros(64), False)[0], conv)
    # the oracle's fp32 normalisation (forward(): x.new_tensor(X_MEAN) in the input's dtype) is the kernels'
    mean = x.new_tensor(horizonnet_ref.X_MEAN).view(1, 3, 1, 1)
    std = x.new_tensor(horizonnet_ref.X_STD).view(1, 3, 1, 1)
    assert torch.equal(gu.normalise_f32(x), (x[:, :3] - mean) / std)


def _pool_bwd_reference(x, dp):
    """(dx, windows routing to each element, sum of |dp| routed to it), fp64, from torch's own argmax (first maximum)."""
    B, C, H, W = x.shape
    _, idx = F.max_pool2d(x, 3, 2, 1, return_indices=True)
    idx = idx.flatten(2)
    z = torch.zeros(B, C, H * W, dtype=torch.float64, device=x.device)
    dx = z.clone().scatter_add_(2, idx, dp.double().flatten(2))
    cnt = z.clone().scatter_add_(2, idx, torch.ones_like(dp, dtype=torch.float64).flatten(2))
    mag = z.clone().scatter_add_(2, idx, dp.double().abs().flatten(2))
    return dx.view(B, C, H, W), cnt.view(B, C, H, W), mag.view(B, C, H, W)


def pool_input(kind, B, seed, H=256, W=512, C=64, dev='cpu'):
    """'signed' N(0, 1); 'negborder' N(0, 1) with the two outer rows and columns all negative (a window there has a
    negative maximum: zero padding would give 0); 'ties' post-ReLU values on a grid of 0.25 with flat blocks, so windows
    hold exact positive ties."""
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(B, C, H, W, generator=g, device=dev)
    if kind == 'negborder':
        x[:, :, :2] = -x[:, :, :2].abs() - 0.5
        x[:, :, -2:] = -x[:, :, -2:].abs() - 0.5
        x[:, :, :, :2] = -x[:, :, :, :2].abs() - 0.5
        x[:, :, :, -2:] = -x[:, :, :, -2:].abs() - 0.5
    elif kind == 'ties':
        x = (torch.round(x * 4) / 4).clamp_min(0)
        x[:, :, H // 4:H // 2, W // 4:W // 2] = 0.75
        x[:, :, -H // 8:, :W // 8] = 1.5
    return x


def test_pool_references_are_the_oracles_pool():
    """The encoder's F.max_pool2d(x, 3, 2, 1) (model.py:76), whose autograd is the routing reference (ties included)."""
    x = pool_input('ties', 2, 3, H=14, W=22, C=4).double().requires_grad_()
    dp = torch.randn(2, 4, 7, 11, dtype=torch.float64)
    F.max_pool2d(x, 3, 2, 1).backward(dp)
    dx, cnt, mag = _pool_bwd_reference(x.detach(), dp)
    assert torch.equal(dx, x.grad) and cnt.sum() == dp.numel() and torch.allclose(mag.sum(), dp.abs().sum())
    # first maximum: each window of a flat input routes to the top-left element of its in-bounds part
    flat = torch.ones(1, 1, 3, 3, dtype=torch.float64)
    want = torch.tensor([[1.0, 1.0, 0.0], [1.0, 1.0, 0.0], [0.0, 0.0, 0.0]], dtype=torch.float64)
    assert torch.equal(_pool_bwd_reference(flat, torch.ones(1, 1, 2, 2, dtype=torch.float64))[0][0, 0], want)
    xn = pool_input('negborder', 1, 4, H=8, W=8, C=1)
    assert F.max_pool2d(xn, 3, 2, 1)[0, 0, 0, 0] < 0


def sequence_reference(ghc, out_w=256):
    """model.py:152-155 (circular pad 1, bilinear W-upsample to out_w + 2f, crop f) + :175-178 (flatten C, H; concat
    scales) + :263 (permute): ghc = the 4 (or fewer) NCHW inputs -> [out_w][B][sum C*H] in their dtype."""
    red = []
    for x in ghc:
        B, C, H, W = x.shape
        f = out_w // W
        x = torch.cat([x[..., -1:], x, x[..., :1]], 3)
        x = F.interpolate(x, size=(H, out_w + 2 * f), mode='bilinear', align_corners=False)[..., f:-f]
        red.append(x.reshape(B, C * H, out_w))
    return torch.cat(red, 1).permute(2, 0, 1)


def test_sequence_reference_is_the_oracles_feature_path():
    """horizonnet_ref.global_height_conv with four identity convs (the centre tap of channel o to o, BN mean 0, var 1)
    reduces to a row subsample, each BN scaling by (1 + eps)^-1/2, then its own pad / upsample / crop."""
    C, H, W, out_w = 16, 32, 8, 32
    x = torch.rand(2, C, H, W, dtype=torch.float64)
    sd = {}
    for j, (ci, co) in enumerate(((C, C // 2), (C // 2, C // 2), (C // 2, C // 4), (C // 4, C // 8))):
        p = f'reduce_height_module.ghc_lst.0.layer.{j}.layers.'
        w = torch.zeros(co, ci, 3, 3, dtype=torch.float64)
        w[torch.arange(co), torch.arange(co), 1, 1] = 1.0
        sd[p + '0.1.weight'], sd[p + '0.1.bias'] = w, torch.zeros(co, dtype=torch.float64)
        sd[p + '1.weight'], sd[p + '1.bias'] = torch.ones(co, dtype=torch.float64), torch.zeros(co, dtype=torch.float64)
        sd[p + '1.running_mean'], sd[p + '1.running_var'] = (torch.zeros(co, dtype=torch.float64),
                                                             torch.ones(co, dtype=torch.float64))
    oracle = horizonnet_ref.global_height_conv(x, sd, 0, out_w).reshape(2, -1, out_w).permute(2, 0, 1)
    k = (1.0 + horizonnet_ref.BN_EPS) ** -2
    ref = sequence_reference([x[:, :C // 8, ::16]], out_w) * k
    assert torch.allclose(ref, oracle, rtol=1e-13, atol=0)


def head_reference(rnn, w, b):
    """model.py:266-269, 278-279 in rnn's dtype: (bon [B][2][T*4], cor [B][1][T*4])."""
    out = rnn @ w.t() + b
    T_, B = out.shape[:2]
    out = out.view(T_, B, 3, 4).permute(1, 2, 0, 3).reshape(B, 3, T_ * 4)
    return out[:, 1:], out[:, :1]


def head_grad_rows(dbon, dcor):
    """d out [T][B][12] from (dbon, dcor): the adjoint of the scatter, o = 4s + k <- column 4t + k of channel s."""
    d = torch.cat([dcor, dbon], 1)                       # [B][3][T*4]
    B = d.shape[0]
    return d.view(B, 3, -1, 4).permute(2, 0, 1, 3).reshape(-1, B, 12)


def test_head_reference_is_the_oracles_head():
    """The oracle's forward (fp64, B = 1): its bon / cor are its linear head of its own rnn_out, and the gradient rows
    are the adjoint of the head's scatter."""
    from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas
    sd = synthetic_state_dict(7, 'random')
    bon, cor, st = horizonnet_ref.forward(sd, synthetic_panoramas(1, seed=8), dtype=torch.float64, return_stages=True)
    hb, hc = head_reference(st['rnn_out'], sd['linear.weight'].double(), sd['linear.bias'].double())
    assert torch.equal(hb, bon) and torch.equal(hc, cor)
    rnn = torch.randn(256, 2, 64, dtype=torch.float64, requires_grad=True)
    w = torch.randn(12, 64, dtype=torch.float64)
    b_, c_ = head_reference(rnn, w, torch.zeros(12, dtype=torch.float64))
    db_, dc_ = torch.randn_like(b_), torch.randn_like(c_)
    (b_ * db_).sum().add((c_ * dc_).sum()).backward()
    assert torch.allclose(rnn.grad, head_grad_rows(db_, dc_) @ w, rtol=1e-13, atol=1e-13)


# ---- the tensor-core stem's arithmetic, emulated
def _pow2_weight_scale(wmax):
    """conv_tc.cu weight_scale: max|w| * 2^t in (2^13, 2^14]."""
    import math
    return 2.0 ** (math.frexp(16384.0 / wmax)[1] - 1)


def _emulate_stem_tc(x, w, scale, shift, relu, rows, drop=None):
    """Output rows `rows` of stem_tc_kernel for one image, emulated: input planes hi / lo of 16 x^ (fp32 normalisation,
    channels of the zero-padded rows zero), weight planes hi / lo of w 2^t, the fp32 sums of hi*hi + hi*lo + lo*hi (drop:
    'wlo' leaves out x_hi*w_lo, 'xlo' x_lo*w_hi), then fmaf(acc, scale 2^-4 2^-t, shift) once-rounded.  [1][64][rows][512]."""
    v = gu.normalise_f32(x) * 16.0
    xh = v.half().float()
    xl = (v - xh).half().float()
    t = _pow2_weight_scale(w.abs().max().item())
    ws = (w * t).float()
    wh = ws.half().float()
    wl = (ws - wh).half().float()
    out = []
    for yo in rows:
        def slab(p):
            p = torch.cat([p[..., -3:], p, p[..., :3]], 3)
            p = F.pad(p, (0, 0, 3, 3))
            return p[:, :, 2 * yo:2 * yo + 7]
        a = F.conv2d(slab(xh), wh, stride=2)
        if drop != 'wlo':
            a = a + F.conv2d(slab(xh), wl, stride=2)
        if drop != 'xlo':
            a = a + F.conv2d(slab(xl), wh, stride=2)
        sc = (scale.double() * 0.0625 / t).view(1, -1, 1, 1)
        y = (a.double() * sc + shift.double().view(1, -1, 1, 1)).float()
        out.append(F.relu(y) if relu else y)
    return torch.cat(out, 2)


def _emulated_stem_ratio(in_kind, w_kind, relu, drop=None):
    rows = [0, 1, 100, 254, 255]
    x = stem_input(in_kind, 1, 11)
    w, scale, shift = stem_weights(w_kind, 12)
    if not relu:
        scale, shift = torch.ones(64), torch.zeros(64)
    y = _emulate_stem_tc(x, w, scale, shift, relu, rows, drop).double()
    # the fp64 reference and bound terms of gpu_utils.stem_reference on the same rows: 7-row slabs of the zero-H-padded
    # normalised input
    xn = F.pad(gu.normalise_f64(x), (0, 0, 3, 3))
    inside = F.pad(torch.ones_like(xn[:, :, 3:-3]), (0, 0, 3, 3))
    wd = w.double()

    def conv(v, k):
        return torch.cat([gu._conv_abs(v[:, :, 2 * r:2 * r + 7], k, (2, 2), 0, 3) for r in rows], 2)
    ref = conv(xn, wd) * scale.double().view(1, -1, 1, 1) + shift.double().view(1, -1, 1, 1)
    ref = F.relu(ref) if relu else ref
    bound = gu.stem_bound(1, w, scale, shift, ref, conv(xn.abs(), wd.abs()), conv(inside, wd.abs()),
                          conv(xn.abs(), torch.ones_like(wd[:1])))
    return gu._worst_ratio(y - ref, bound)


@pytest.mark.parametrize('relu', [True, False])
@pytest.mark.parametrize('w_kind', STEM_WEIGHTS)
@pytest.mark.parametrize('in_kind', ('uniform', 'pano8'))
def test_stem_bound_holds_for_an_emulation_of_the_tensor_core_stem(in_kind, w_kind, relu):
    r = _emulated_stem_ratio(in_kind, w_kind, relu)
    print(f'{in_kind} {w_kind} relu={relu}: emulated err / bound {r:.3f}')
    assert r < 0.5, r


@pytest.mark.parametrize('drop', ['wlo', 'xlo'])
@pytest.mark.parametrize('w_kind', ('init', 'ckpt'))
@pytest.mark.parametrize('in_kind', ('uniform', 'pano8'))
def test_stem_bound_catches_an_emulation_with_a_lost_cross_product(in_kind, w_kind, drop):
    r = _emulated_stem_ratio(in_kind, w_kind, True, drop)
    print(f'{in_kind} {w_kind} without {drop}: emulated err / bound {r:.1f}')
    assert r > 1.0, r


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize('w_kind', STEM_WEIGHTS)
@pytest.mark.parametrize('in_kind', STEM_INPUTS)
@pytest.mark.parametrize('B', [1, 2, 3])
def test_stem_vs_fp64(B, in_kind, w_kind):
    x = stem_input(in_kind, B, seed=100 * B + STEM_INPUTS.index(in_kind))
    w, scale, shift = stem_weights(w_kind, seed=7 + STEM_WEIGHTS.index(w_kind))
    x, w, scale, shift = _dev(x, w, scale, shift)
    ones, zeros = torch.ones(64, device=DEV), torch.zeros(64, device=DEV)
    worst = {}
    for impl in (0, 1):
        for epi, (sc, sh, relu) in (('eval', (scale, shift, True)), ('raw', (ones, zeros, False))):
            out = gu.run_stem(x, w, sc, sh, relu, impl)
            ratio, small = gu.stem_ratio(out, x, w, sc, sh, relu, impl)
            _record({'test': 'stem', 'impl': impl, 'epilogue': epi, 'B': B, 'input': in_kind, 'weights': w_kind,
                     'ratio': ratio, 'smallest_channel_ratio': small})
            worst[(impl, epi)] = ratio
    bad = {k: v for k, v in worst.items() if not v <= 1.0}
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize('impl', [0, 1])
def test_stem_batch_64_images_equal_batch_1(impl):
    x = stem_input('pano8', 64, seed=64)
    w, scale, shift = stem_weights('ckpt', seed=8)
    x, w, scale, shift = _dev(x, w, scale, shift)
    out = gu.run_stem(x, w, scale, shift, True, impl)
    for b in range(64):
        one = gu.run_stem(x[b:b + 1].contiguous(), w, scale, shift, True, impl)
        assert torch.equal(out[b:b + 1], one), f'stem impl {impl}: image {b} of B = 64 differs from the image alone'
    sel = [0, 31, 63]
    ratio, small = gu.stem_ratio(out[sel], x[sel], w, scale, shift, True, impl)
    _record({'test': 'stem', 'impl': impl, 'epilogue': 'eval', 'B': 64, 'input': 'pano8', 'weights': 'ckpt',
             'images': sel, 'ratio': ratio, 'smallest_channel_ratio': small})
    assert ratio <= 1.0, ratio


def _run_pool(xin, B, H, W, C, planes):
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    n = B * Ho * (Wo + 2) * C
    buf = torch.full((n + 4096,), gu.CANARY, device=DEV)
    if planes:
        buf[:n].view(torch.int16).fill_(-1)            # all-ones fp16 = NaN
    else:
        buf[:n] = float('nan')
    _lib.check(_lib.lib().hn_maxpool(xin.data_ptr(), B, H, W, C, int(planes), buf.data_ptr(),
                                     torch.cuda.current_stream().cuda_stream), 'hn_maxpool')
    torch.cuda.synchronize()
    assert bool((buf[n:] == gu.CANARY).all()), 'max-pool: write past the end of the output'
    return buf[:n]


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['signed', 'negborder', 'ties'])
@pytest.mark.parametrize('B', [1, 3, 64])
def test_maxpool_forward_and_backward(B, kind):
    H, W, C = 256, 512, 64
    Ho, Wo = H // 2, W // 2
    x = pool_input(kind, B, seed=B * 10 + len(kind), dev=DEV)
    xin = gu.to_halo_nhwc(x, 1)
    xin[:, :, 0], xin[:, :, -1] = 1e30, 1e30           # the pool does not wrap: a read of a halo column shows
    # fp32 output
    got = _run_pool(xin, B, H, W, C, False).view(B, Ho, Wo + 2, C)
    assert not torch.isnan(got).any(), 'max-pool: output elements left unwritten'
    assert torch.equal(got[:, :, 0], got[:, :, -2]) and torch.equal(got[:, :, -1], got[:, :, 1]), \
        'max-pool: halo columns are not the circular wrap'
    ref = F.max_pool2d(x, 3, 2, 1)
    assert torch.equal(gu.from_halo_nhwc(got, 1), ref), 'max-pool: fp32 output differs from F.max_pool2d'
    # split-plane output: the split of the fp32 output, bit for bit (wrap columns included)
    pl = _run_pool(xin, B, H, W, C, True).view(torch.int16).view(2, B, Ho, Wo + 2, C)
    hi, lo = gu.split_planes_torch(got)
    assert torch.equal(pl[0], hi) and torch.equal(pl[1], lo), 'max-pool: split-plane output is not the split of the fp32 one'
    del pl, hi, lo, got
    # backward: dp with its halo columns NaN (never read), dx zeroed with canary halo columns
    g = torch.Generator(device=DEV).manual_seed(B + 5)
    dp = torch.randn(B, C, Ho, Wo, generator=g, device=DEV)
    dp[:, :, ::7, ::5] = 0.0
    dpin = gu.to_halo_nhwc(dp, 1)
    dpin[:, :, 0], dpin[:, :, -1] = float('nan'), float('nan')
    n = B * H * (W + 2) * C
    buf = torch.full((n + 4096,), gu.CANARY, device=DEV)
    dx = buf[:n].view(B, H, W + 2, C)
    dx[:, :, 1:-1] = 0.0
    _lib.check(_lib.lib().hn_maxpool_backward(xin.data_ptr(), dpin.data_ptr(), B, H, W, C, dx.data_ptr(),
                                              torch.cuda.current_stream().cuda_stream), 'hn_maxpool_backward')
    torch.cuda.synchronize()
    assert bool((buf[n:] == gu.CANARY).all()), 'max-pool backward: write past the end of dx'
    assert bool((dx[:, :, 0] == gu.CANARY).all()) and bool((dx[:, :, -1] == gu.CANARY).all()), \
        'max-pool backward: a halo column of dx was written'
    del xin, dpin
    ratio = cons_ratio = 0.0
    multi = 0
    for b0 in range(0, B, 8):                          # the fp64 reference in chunks of 8 images
        sl = slice(b0, min(B, b0 + 8))
        gdx = gu.from_halo_nhwc(dx[sl], 1).double()
        rdx, cnt, mag = _pool_bwd_reference(x[sl], dp[sl])
        err = (gdx - rdx).abs()
        assert bool((err[cnt <= 1] == 0).all()), 'max-pool backward: an element one window routes to is not exact'
        # k atomic adds of fp32 values round k - 1 times, at most 2^-24 of the routed magnitude each
        bound = MARGIN * gu.EPS24 * (cnt - 1).clamp_min(0) * mag
        ratio = max(ratio, gu._worst_ratio(err, bound))
        cons = (gdx.sum(dim=(2, 3)) - dp[sl].double().sum(dim=(2, 3))).abs()
        slack = 2.0 ** -40 * dp[sl].double().abs().sum(dim=(2, 3))          # fp64 summation order
        cons_ratio = max(cons_ratio, gu._worst_ratio(cons, bound.sum(dim=(2, 3)) + slack))
        multi += int((cnt > 1).sum())
        del gdx, rdx, cnt, mag, err, bound
    _record({'test': 'maxpool_bwd', 'B': B, 'input': kind, 'ratio': ratio, 'conservation_ratio': cons_ratio,
             'multi_window_elements': multi})
    assert ratio <= 1.0 and cons_ratio <= 1.0, (ratio, cons_ratio)


def _ghc_inputs(backbone, B, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randn(B, c, 8 >> s, 256 >> s, generator=g, device=DEV) for s, c in enumerate(BACKBONES[backbone])]


def _seq_call(backbone, B, ptrs, planes, seq):
    arr = (ctypes.c_void_p * 4)(*ptrs)
    _lib.check(_lib.lib().hn_feature_sequence(backbone.encode(), B, arr, int(planes), seq.data_ptr(),
                                              torch.cuda.current_stream().cuda_stream), 'hn_feature_sequence')
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize('B', T.BATCHES)
@pytest.mark.parametrize('backbone', list(BACKBONES))
def test_feature_sequence_vs_fp64(backbone, B):
    ghc = _ghc_inputs(backbone, B, seed=B)
    CL = sum(c * (8 >> s) for s, c in enumerate(BACKBONES[backbone]))
    n = 256 * B * CL
    # fp32 path
    halo = [gu.to_halo_nhwc(x, 1) for x in ghc]
    buf = gu._nan_buffer(n, DEV)
    _seq_call(backbone, B, [h.data_ptr() for h in halo], False, buf)
    got = buf[:n].view(256, B, CL)
    assert not torch.isnan(got).any() and bool((buf[n:] == gu.CANARY).all())
    xd = [x.double() for x in ghc]
    ref = sequence_reference(xd)
    absref = sequence_reference([x.abs() for x in xd])
    c0 = BACKBONES[backbone][0] * 8                     # scale 0: W = 256, f = 1
    assert torch.equal(got[..., :c0].double(), ref[..., :c0]), 'f = 1 columns are not exact copies'
    r32 = gu._worst_ratio(got.double() - ref, MARGIN * 2 * gu.EPS24 * absref)      # two products and a sum in fp32
    # plane path: inputs as split planes, the reference from the merged input planes
    pls, merged = [], []
    for h in halo:
        hi, lo = gu.split_planes_torch(h)
        pls.append(torch.stack([hi, lo]).contiguous())
        merged.append(gu.from_halo_nhwc(gu.merge_planes_torch(hi, lo), 1).double())
    pbuf = torch.full((n + 4096,), gu.CANARY, device=DEV)
    pbuf[:n].view(torch.int16).fill_(-1)
    _seq_call(backbone, B, [p.data_ptr() for p in pls], True, pbuf)
    assert bool((pbuf[n:] == gu.CANARY).all())
    pv = pbuf[:n].view(torch.int16).view(2, n)
    gotp = gu.merge_planes_torch(pv[0], pv[1]).view(256, B, CL).double()
    assert not torch.isnan(gotp).any()
    refp = sequence_reference(merged)
    # the interpolation, then the re-split: 2^-22 |y| with a normal lo plane, half the subnormal spacing (2^-21) below 2
    rp = gu._worst_ratio(gotp - refp, MARGIN * (2 * gu.EPS24 * sequence_reference([m.abs() for m in merged]) +
                                                gu.EPS21 * (refp.abs() + 1.0)))
    # backward: the adjoint, added into prefilled dghc whose halo columns hold the canary
    dseq = torch.randn(256, B, CL, generator=torch.Generator(device=DEV).manual_seed(B + 1), device=DEV)
    pre = [torch.randn_like(x) for x in ghc]
    dg = []
    for p in pre:
        h = gu.to_halo_nhwc(p, 1)
        h[:, :, 0], h[:, :, -1] = gu.CANARY, gu.CANARY
        dg.append(h)
    arr = (ctypes.c_void_p * 4)(*[d.data_ptr() for d in dg])
    _lib.check(_lib.lib().hn_feature_sequence_backward(backbone.encode(), B, dseq.data_ptr(), arr,
                                                       torch.cuda.current_stream().cuda_stream),
               'hn_feature_sequence_backward')
    torch.cuda.synchronize()
    xv = [x.double().requires_grad_() for x in ghc]
    sequence_reference(xv).backward(dseq.double())
    av = [torch.zeros_like(x, dtype=torch.float64, requires_grad=True) for x in ghc]
    sequence_reference(av).backward(dseq.double().abs())
    rb = 0.0
    for s, (d, p, a, b) in enumerate(zip(dg, pre, xv, av)):
        assert bool((d[:, :, 0] == gu.CANARY).all()) and bool((d[:, :, -1] == gu.CANARY).all()), \
            f'scale {s}: a halo column of dghc was written'
        gd = gu.from_halo_nhwc(d, 1).double()
        want = p.double() + a.grad
        if s == 0:                                     # f = 1: one addition of d, rounded once in fp32
            assert torch.equal(gu.from_halo_nhwc(d, 1), p + a.grad.float()), 'f = 1: the gradient is not a copy of d'
        f = 256 // ghc[s].shape[3]
        bound = MARGIN * (2 * f + 1) * gu.EPS24 * (b.grad + p.double().abs())     # l * d products, <= 2f adds
        rb = max(rb, gu._worst_ratio(gd - want, bound))
    _record({'test': 'feature_sequence', 'backbone': backbone, 'B': B, 'ratio_f32': r32, 'ratio_planes': rp,
             'ratio_bwd': rb})
    assert r32 <= 1.0 and rp <= 1.0 and rb <= 1.0, (r32, rp, rb)


@pytest.mark.gpu
@pytest.mark.parametrize('B', T.BATCHES)
@pytest.mark.parametrize('K', [1024, 512])
def test_linear_head_forward_and_backward_vs_fp64(K, B):
    g = torch.Generator(device=DEV).manual_seed(K + B)
    Tn = 256
    rnn = torch.rand(Tn, B, K, generator=g, device=DEV) * 2 - 1
    if K == 512:
        rnn = rnn.clamp_min(0)                        # the MLP's hidden layer is post-ReLU
    w = (torch.rand(12, K, generator=g, device=DEV) * 2 - 1) / K ** 0.5
    b = torch.randn(12, generator=g, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    nb, nc = B * 2 * 1024, B * 1024
    bb, cb = gu._nan_buffer(nb, DEV), gu._nan_buffer(nc, DEV)
    _lib.check(_lib.lib().hn_linear_head(rnn.data_ptr(), w.data_ptr(), b.data_ptr(), bb.data_ptr(), cb.data_ptr(), Tn, B,
                                         K, st), 'hn_linear_head')
    torch.cuda.synchronize()
    for buf, n in ((bb, nb), (cb, nc)):
        assert not torch.isnan(buf[:n]).any() and bool((buf[n:] == gu.CANARY).all())
    bon, cor = bb[:nb].view(B, 2, 1024), cb[:nc].view(B, 1, 1024)
    rd, wd, bd = rnn.double(), w.double(), b.double()
    rbon, rcor = head_reference(rd, wd, bd)
    abon, acor = head_reference(rd.abs(), wd.abs(), bd.abs())
    rf = max(gu._worst_ratio(bon.double() - rbon, gu.C32 * gu.EPS24 * abon + gu.EPS24 * rbon.abs()),
             gu._worst_ratio(cor.double() - rcor, gu.C32 * gu.EPS24 * acor + gu.EPS24 * rcor.abs()))
    # backward
    dbon = torch.randn(B, 2, 1024, generator=g, device=DEV)
    dcor = torch.randn(B, 1, 1024, generator=g, device=DEV) * 0.01
    nd = Tn * B * K
    drb, dwb, dbb = gu._nan_buffer(nd, DEV), gu._nan_buffer(12 * K, DEV), gu._nan_buffer(12, DEV)
    _lib.check(_lib.lib().hn_linear_head_backward(dbon.data_ptr(), dcor.data_ptr(), rnn.data_ptr(), w.data_ptr(),
                                                  drb.data_ptr(), dwb.data_ptr(), dbb.data_ptr(), Tn, B, K, st),
               'hn_linear_head_backward')
    torch.cuda.synchronize()
    for buf, n in ((drb, nd), (dwb, 12 * K), (dbb, 12)):
        assert not torch.isnan(buf[:n]).any() and bool((buf[n:] == gu.CANARY).all())
    drnn, dw, db = drb[:nd].view(Tn, B, K).double(), dwb[:12 * K].view(12, K).double(), dbb[:12].double()
    d = head_grad_rows(dbon.double(), dcor.double())              # [T][B][12]
    ref_drnn = d @ wd
    rdi = gu._worst_ratio(drnn - ref_drnn, gu.C32 * gu.EPS24 * (d.abs() @ wd.abs()) + gu.EPS24 * ref_drnn.abs())
    d2, r2 = d.reshape(-1, 12), rd.reshape(-1, K)
    ref_dw, ref_db = d2.t() @ r2, d2.sum(0)
    cw = (HEAD_SLICES + 1) * gu.EPS24
    rdw = max(gu._worst_ratio(dw - ref_dw, cw * (d2.abs().t() @ r2.abs()) + gu.EPS24 * ref_dw.abs()),
              gu._worst_ratio(db - ref_db, cw * d2.abs().sum(0) + gu.EPS24 * ref_db.abs()))
    # autograd through the reference head agrees with the rows of d (the scatter's adjoint)
    rv = rd[:, :1].clone().requires_grad_()
    hb, hc = head_reference(rv, wd, bd)
    (hb * dbon.double()[:1]).sum().add((hc * dcor.double()[:1]).sum()).backward()
    assert torch.allclose(rv.grad, ref_drnn[:, :1], rtol=1e-12, atol=1e-12)
    _record({'test': 'linear_head', 'K': K, 'B': B, 'ratio_fwd': rf, 'ratio_drnn': rdi, 'ratio_dw_db': rdw})
    assert rf <= 1.0 and rdi <= 1.0 and rdw <= 1.0, (rf, rdi, rdw)


@pytest.mark.gpu
@pytest.mark.parametrize('B', T.BATCHES)
@pytest.mark.parametrize('cols', [512, 2048])
def test_col_sum_vs_fp64(cols, B):
    g = torch.Generator(device=DEV).manual_seed(cols + B)
    rows = 256 * B
    x = torch.randn(rows, cols, generator=g, device=DEV) * 2.0 ** (-20 * torch.rand(cols, generator=g, device=DEV))
    out = gu._nan_buffer(cols, DEV)
    _lib.check(_lib.lib().hn_col_sum(x.data_ptr(), rows, cols, out.data_ptr(), torch.cuda.current_stream().cuda_stream),
               'hn_col_sum')
    torch.cuda.synchronize()
    assert not torch.isnan(out[:cols]).any() and bool((out[cols:] == gu.CANARY).all())
    ref = x.double().sum(0)
    ratio = gu._worst_ratio(out[:cols].double() - ref,
                            (COL_SUM_SLICES + 1) * gu.EPS24 * x.double().abs().sum(0) + gu.EPS24 * ref.abs())
    _record({'test': 'col_sum', 'cols': cols, 'B': B, 'ratio': ratio})
    assert ratio <= 1.0, ratio


@pytest.mark.gpu
@pytest.mark.parametrize('B', [1, 3, 8])
def test_stem_input_is_the_fp32_normalisation(B):
    x = stem_input('nan4' if B == 3 else 'pano8', B, seed=B).to(DEV)
    n = B * 512 * 1030 * 3
    buf = gu._nan_buffer(n, DEV)
    _lib.check(_lib.lib().hn_stem_input(x.data_ptr(), x.shape[1], B, buf.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream), 'hn_stem_input')
    torch.cuda.synchronize()
    assert bool((buf[n:] == gu.CANARY).all())
    want = gu.to_halo_nhwc(gu.normalise_f32(x), 3)
    assert torch.equal(buf[:n].view(B, 512, 1030, 3), want)
