"""The product's large batches, image by image, bit for bit against the same panorama run at B = 1 (which
test_gpu_parity.py, test_resnet18.py and test_no_rnn_head.py check against the oracle).  -m gpu:

* the eval forward at B = 64 (the forward infer_layout runs for 32 views x 2 panoramas, and validate's chunk): resnet50 +
  bi-LSTM with tensor cores on and off, resnet50 + MLP head and resnet18 + bi-LSTM.  Image 63 lies across byte 2^31 of the
  largest activation buffers, image 62 just below it;
* the eval forward at the first batch past 64 that sends a height-reduction conv into a conv_tc_kernel variant no batch
  up to 64 takes (B = 67 on a 132-SM H100 SXM, 113 on a 114-SM H100 PCIe);
* the eval forward at B = 128: every lo plane of layer1's output past byte 2^31, image 126's lo plane past element 2^31
  of the u16 planes, image 127's hi plane across byte 2^31;
* infer_layout with 32 views of 2 panoramas (one forward of 64) and validate on 65 panoramas (a chunk of 64 and one of 1):
  every panorama equals the same call on that panorama alone.

Each test first checks, from the unit shapes of tc_cases.conv_units, that its batch puts the rows it compares where it
says, so that a layout change cannot quietly remove the crossing.  The device workspace follows the allocation list of
hn_model_create_arch (about 270 MB per image for resnet50 + bi-LSTM); a test skips only when the device has less free
memory than that, and says how much it needed.  The host side of both (the batch past 64 and the workspace estimate)
runs without a GPU."""
import gc

import numpy as np
import pytest
import torch

import __graft_entry__ as entry
from horizonnet_b200 import _lib
from horizonnet_b200 import evaluate as EV
from horizonnet_b200._spec import c_last
from horizonnet_b200.inference import infer_layout
from horizonnet_b200.model import HorizonNet
from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas
import gpu_utils as gu
import tc_cases as T

DEV = 'cuda:0'
TWO_GB = 2 ** 31


@pytest.fixture(scope='module', autouse=True)
def _built():
    entry.build()
    _lib.lib()


# ---- where the images lie (no GPU needed for the arithmetic)
def _px(h, w, c):
    return h * (w + 2) * c                         # halo-NHWC elements of one image


def _out_px(unit):
    name, H, W, Ci, Co, k, (sh, sw) = unit
    return _px(H // sh, W // sw, Co)


def _layer1_img():
    """Elements of one image of resnet50's layer1 output, the largest activation of X[0], X[1], IDN and F[0]."""
    return _out_px(next(u for u in T.conv_units('resnet50') if u[0] == 'layer1.2.conv3'))


STEM_IMG = _px(256, 512, 64)                       # S0, the stem output: fp32 on both paths


def _plane_bytes(B, b, img, lo):
    """(first, last) byte of image b's hi or lo plane in a split-plane activation of B images: the u16 hi planes of all B
    images, then their lo planes (conv_tc.cu: out_plane = the activation's numel)."""
    first = ((B if lo else 0) + b) * img * 2
    return first, first + img * 2 - 1


def _f32_bytes(b, img):
    return b * img * 4, (b + 1) * img * 4 - 1


def _crosses(span, at=TWO_GB):
    return span[0] < at <= span[1]


def _past(span, at=TWO_GB):
    return span[0] >= at


def workspace_bytes(backbone, use_rnn, B):
    """Device bytes hn_model_create_arch allocates for max_batch B, from its allocation list (the stem's packed-input
    scratch and the per-model constants left out)."""
    x_img = t1 = t2 = idn = g_img = 0
    f_img, go_img = {}, {}
    units = T.conv_units(backbone)
    for i, u in enumerate(units):
        name = u[0]
        if name.startswith('ghc'):
            s, j = (int(v) for v in name[3:].split('.'))
            if j == 3:
                go_img[s] = _out_px(u)
            else:
                g_img = max(g_img, _out_px(u))
            continue
        layer, blk, conv = name.split('.')
        if conv == 'conv1':
            t1 = max(t1, _out_px(u))
        elif conv == 'downsample':
            idn = max(idn, _out_px(u))
        elif conv == 'conv2' and T.BACKBONES[backbone][0] == 'bottleneck':
            t2 = max(t2, _out_px(u))
        if T.has_residual(backbone, name):         # the block's output
            nxt = units[i + 1][0]
            if nxt.startswith(layer + '.'):
                x_img = max(x_img, _out_px(u))
            else:
                f_img[layer] = _out_px(u)
    cl = c_last(backbone)
    per_img = (STEM_IMG + _px(128, 256, 64) + max([x_img] + list(f_img.values())) + x_img + idn + t1 + t2 +
               sum(f_img.values()) + 2 * g_img + sum(go_img.values()) + 256 * cl + 2 * (3 * 512 * 1024 + 3 * 1024))
    per_img += 256 * 4096 + 3 * 256 * 1024 if use_rnn else 256 * cl + 256 * 512
    return 4 * per_img * B


def _need(backbone, use_rnn, B):
    """Skips unless the device has the workspace of batch B, its input and 2 GiB for everything else free."""
    need = workspace_bytes(backbone, use_rnn, B) + B * 3 * 512 * 1024 * 4 + TWO_GB
    free, _ = torch.cuda.mem_get_info(DEV)
    print(f'{backbone} use_rnn={use_rnn} B={B}: needs {need / 2 ** 30:.1f} GiB of device memory, {free / 2 ** 30:.1f} GiB free')
    if free < need:
        pytest.skip(f'needs {need / 2 ** 30:.1f} GiB of free device memory, {free / 2 ** 30:.1f} GiB free')


@pytest.fixture
def release():
    """Frees each test's model workspace before the next test measures free memory."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _net(backbone, use_rnn, tensor_cores=True, seed=3):
    net = HorizonNet(backbone, use_rnn).eval()
    net.load_state_dict(synthetic_state_dict(seed, 'random', use_rnn=use_rnn, backbone=backbone), strict=True)
    net.use_tensor_cores(tensor_cores)
    return net.to(DEV)


def _rows_equal_batch_1(net, x, rows):
    with torch.no_grad():
        bon, cor = net(x.to(DEV))
    net.check()
    assert torch.isfinite(bon).all() and torch.isfinite(cor).all()
    B = x.shape[0]
    for r in rows:
        with torch.no_grad():
            b1, c1 = net(x[r:r + 1].to(DEV))
        assert torch.equal(bon[r:r + 1], b1) and torch.equal(cor[r:r + 1], c1), \
            f'row {r} of B = {B} differs from the same panorama at B = 1'


# ---- eval forward
def _first_batch_with_a_new_conv_tc_key(sms):
    """The smallest batch past 64 whose eval forward of resnet50 takes a conv_tc_planes variant no batch 1 .. 64 takes."""
    eval_launches = lambda B: [c for c in T.model_launches('resnet50', B) if ':' not in c['name']]
    seen = {T.variant_key(c, p) for B in range(1, 65) for c in eval_launches(B) for p in [T.plan(c, sms)] if p}
    for B in T.ACCEPTED_BATCHES[64:]:
        if any(p and T.variant_key(c, p) not in seen for c in eval_launches(B) for p in [T.plan(c, sms)]):
            return B
    return None


def test_the_host_side_of_the_tests_below():
    """The batch past 64 the GPU test picks on each H100, and the workspace estimate its skips rest on."""
    assert _first_batch_with_a_new_conv_tc_key(132) == 67
    assert _first_batch_with_a_new_conv_tc_key(114) == 113
    assert 255e6 < workspace_bytes('resnet50', True, 1) < 275e6                    # about 270 MB per image


@pytest.mark.gpu
@pytest.mark.parametrize('backbone,use_rnn,tensor_cores', [('resnet50', True, True), ('resnet50', True, False),
                                                           ('resnet50', False, True), ('resnet18', True, True)],
                         ids=['r50_rnn_tc', 'r50_rnn_f32', 'r50_mlp_tc', 'r18_rnn_tc'])
def test_batch_64_rows_equal_batch_1(backbone, use_rnn, tensor_cores, release):
    B, rows = 64, (0, 62, 63)
    if backbone == 'resnet18':                     # its activations are narrow: the stem's fp32 output crosses
        assert _crosses(_f32_bytes(63, STEM_IMG)) and _f32_bytes(62, STEM_IMG)[1] < TWO_GB
    elif tensor_cores:                             # image 63's lo plane of layer1's output crosses byte 2^31
        img = _layer1_img()
        assert _crosses(_plane_bytes(B, 63, img, lo=True)) and _plane_bytes(B, 62, img, lo=True)[1] < TWO_GB
    else:                                          # fp32 activations: image 63 of layer1's output crosses byte 2^31
        img = _layer1_img()
        assert _crosses(_f32_bytes(63, img)) and _f32_bytes(62, img)[1] < TWO_GB
    _need(backbone, use_rnn, B)
    net = _net(backbone, use_rnn, tensor_cores)
    _rows_equal_batch_1(net, synthetic_panoramas(B, seed=64), rows)


@pytest.mark.gpu
def test_batch_past_64_with_new_conv_tc_variants_rows_equal_batch_1(release):
    sms = gu.device_sms()
    B = _first_batch_with_a_new_conv_tc_key(sms)
    assert B == {132: 67, 114: 113}.get(sms, B), (sms, B)
    img = _layer1_img()
    assert _past(_plane_bytes(B, B - 1, img, lo=True))
    _need('resnet50', True, B)
    net = _net('resnet50', True)
    _rows_equal_batch_1(net, synthetic_panoramas(B, seed=B), (0, B - 1))


@pytest.mark.gpu
def test_batch_128_rows_equal_batch_1(release):
    B, img = 128, _layer1_img()
    assert _past(_plane_bytes(B, 0, img, lo=True))                       # every lo plane past byte 2^31
    assert _crosses(_plane_bytes(B, 126, img, lo=True), 2 * TWO_GB)      # ... image 126's across u16 element 2^31
    assert _crosses(_plane_bytes(B, 127, img, lo=False))                  # image 127's hi plane across byte 2^31
    _need('resnet50', True, B)
    net = _net('resnet50', True)
    _rows_equal_batch_1(net, synthetic_panoramas(B, seed=128), (0, 126, 127))


@pytest.mark.gpu
# ---- the product's batch-64 paths
def test_infer_layout_32_views_of_2_panoramas_equals_each_alone(release):
    rot = [i / 40 for i in range(1, 32)]           # 31 rotations + the view itself: one forward of 64
    assert 2 * (1 + len(rot)) == 64
    _need('resnet50', True, 64)
    net = _net('resnet50', True)
    x = synthetic_panoramas(2, seed=5)
    with torch.no_grad():
        both, st = infer_layout(net, x, rotate=rot, force_raw=True, return_status=True)
        for b in range(2):
            one, st1 = infer_layout(net, x[b:b + 1], rotate=rot, force_raw=True, return_status=True)
            assert st[b] == st1[0], b
            (c, z0, z1), (c1, z01, z11) = both[b], one[0]
            assert (c is None) == (c1 is None), b
            assert c is None or np.array_equal(c, c1), f'panorama {b}: corners differ from the panorama alone'
            assert (z0, np.float32(z1).tobytes()) == (z01, np.float32(z11).tobytes()), b


@pytest.mark.gpu
def test_validate_65_panoramas_equals_each_alone(release):
    from test_layout_eval import _room
    B = 65                                          # a chunk of evaluate.MAX_BATCH and one of 1
    assert EV.MAX_BATCH == 64
    _need('resnet50', True, EV.MAX_BATCH)
    net = _net('resnet50', True)
    x = synthetic_panoramas(B, seed=65)
    gts = [_room(1000 + b) for b in range(B)]
    with torch.no_grad():
        got = EV.validate(net, x, gts, return_status=True)
        for b in range(B):
            one = EV.validate(net, x[b:b + 1], gts[b:b + 1], return_status=True)
            for k in ('status', 'iou2d', 'iou3d', 'rmse', 'delta_1'):
                assert np.array_equal(got[k][b:b + 1], one[k], equal_nan=True), (b, k, got[k][b], one[k][0])
