"""-m gpu: the layout evaluation kernels (csrc/layout_eval.cu, hn_layout_eval_general) and validate() against
oracle/eval_general_ref.py, which tests/test_eval_oracle.py pins to the real reference.

Statuses must be identical; depth maps within 1e-5 relative per pixel; RMSE within 1e-5 relative (the reference sums in
float32); delta_1 within 4e-6 (2 pixels of 524288); iou2d and iou3d within 1e-6.  The depth bound is not 1 ulp because
the per-corner steps of pano_connect_points are float32 sin / cos / tan, which numpy computes with SIMD polynomials up to
about 1.5 ulp from the correctly rounded value (which one depends on the host CPU), and the kernel rounds the float64
result; the boundary amplifies that difference a few times (DESIGN.md section 9)."""
import os

import numpy as np
import pytest
import torch

import __graft_entry__ as entry
from horizonnet_b200 import _lib
from horizonnet_b200 import evaluate as EV
from horizonnet_b200.inference import infer_layout
from horizonnet_b200.model import HorizonNet
from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas
from oracle import eval_general_ref as E

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'eval_general.npz'))
NAMES = [str(n) for n in G['names']]
SCALE = np.array([1024, 512], np.float32)
DEPTH_REL = 1e-5


@pytest.fixture(scope='module', autouse=True)
def _built():
    entry.build()
    _lib.lib()


def _room(seed):
    """A seeded Manhattan room in pixels: a rectangle, optionally notched, rotated, seen from an off-centre camera."""
    rs = np.random.RandomState(seed)
    hx, hy = rs.uniform(1.5, 4.0, 2)
    poly = [(hx, hy), (-hx, hy), (-hx, -hy), (hx, -hy)]
    if rs.rand() < 0.5:
        nx, ny = rs.uniform(0.3, 0.6) * hx, rs.uniform(0.3, 0.6) * hy
        poly = [(hx, hy - ny), (hx - nx, hy - ny), (hx - nx, hy)] + poly[1:]
    p = np.array(poly) - rs.uniform(-0.4, 0.4, 2)
    a = rs.uniform(-np.pi, np.pi)
    p = p @ np.array([[np.cos(a), np.sin(a)], [-np.sin(a), np.cos(a)]])
    u, d = np.arctan2(p[:, 0], -p[:, 1]), np.hypot(p[:, 0], p[:, 1])
    col = (u / (2 * np.pi) + 0.5) * 1024 - 0.5
    ceil_h = rs.uniform(1.0, 1.8)
    order = np.argsort(col)
    cor = np.zeros((2 * len(col), 2), np.float32)
    cor[0::2, 0] = cor[1::2, 0] = col[order]
    cor[0::2, 1] = ((-np.arctan(ceil_h / d) / np.pi + 0.5) * 512 - 0.5)[order]
    cor[1::2, 1] = ((np.arctan(1.6 / d) / np.pi + 0.5) * 512 - 0.5)[order]
    return cor


def _jitter(cor, seed):
    rs = np.random.RandomState(seed)
    d = cor.copy()
    dc = rs.normal(0, 5, len(cor) // 2).astype(np.float32)
    d[0::2, 0] += dc
    d[1::2, 0] += dc
    d[:, 1] += rs.normal(0, 4, len(cor)).astype(np.float32)
    return d


def _fixture_pairs():
    dts, gts, names = [], [], []
    for n in NAMES:
        dt, gt = (G['layout/%s/cor' % str(G['%s/%s_key' % (n, side)])] for side in ('dt', 'gt'))
        dts.append(None if dt.dtype == np.int64 else dt / SCALE)
        gts.append(gt)
        names.append(n)
    return names, dts, gts


def _oracle(dt, gt):
    return E.test_general(E.fallback_box() if dt is None else E.dt_pixels(dt), gt)


def _check(names, dts, gts, depth):
    o, maps = EV._eval(dts, gts, depth=depth)
    res = {k: v.cpu().numpy() for k, v in o.items()}
    maps = maps.cpu().numpy() if depth else None
    for b, name in enumerate(names):
        want = _oracle(dts[b], gts[b])
        st = int(res['status'][b])
        assert st == want['status'], (name, E.STATUS_NAMES[st], E.STATUS_NAMES[want['status']])
        for k, tol in (('iou2d', 1e-6), ('iou3d', 1e-6), ('delta_1', 4e-6)):
            if np.isnan(want[k]):
                assert np.isnan(res[k][b]), (name, k)
            else:
                assert abs(res[k][b] - want[k]) <= tol, (name, k, res[k][b], want[k])
        if np.isnan(want['rmse']):
            assert np.isnan(res['rmse'][b]), name
        else:
            assert abs(res['rmse'][b] - want['rmse']) <= 1e-5 * max(want['rmse'], 1e-3), (name, res['rmse'][b], want['rmse'])
        if depth and st in (E.OK, E.DT_INVALID):
            dt_px = E.fallback_box() if dts[b] is None else E.dt_pixels(dts[b])
            try:
                want_dt = E.layout_2_depth(dt_px)
            except E.DepthAssertion:
                want_dt = np.zeros((512, 1024), np.float32)
            for got, ref in ((maps[b, 0], want_dt), (maps[b, 1], E.layout_2_depth(gts[b]))):
                rel = np.abs(got.astype(np.float64) - ref) / np.maximum(np.abs(ref), 1e-30)
                assert rel.max() <= DEPTH_REL, (name, float(rel.max()))


def test_fixture_pairs_match_the_oracle():
    _check(*_fixture_pairs(), depth=True)


def test_seeded_batch_of_64_matches_the_oracle():
    gts = [_room(s) for s in range(64)]
    dts = [(_jitter(g, 1000 + s) if s % 4 else g.copy()) / SCALE for s, g in enumerate(gts)]
    _check([str(s) for s in range(64)], dts, gts, depth=False)


def test_public_functions():
    names, dts, gts = _fixture_pairs()
    i = names.index('room4_8c_jitter')
    r = EV.eval_general([dts[i]], [gts[i]])
    want = _oracle(dts[i], gts[i])
    assert abs(r['iou3d'][0] - want['iou3d']) <= 1e-6 and r['status'][0] == EV.OK
    d = EV.layout_2_depth(gts[i])
    ref = E.layout_2_depth(gts[i])
    assert (np.abs(d.astype(np.float64) - ref) / ref).max() <= DEPTH_REL
    j = names.index('dt_columns_differ')
    with pytest.raises(AssertionError, match='pair 1'):
        EV.eval_general([dts[i], dts[j]], [gts[i], gts[j]])
    with pytest.raises(NotImplementedError):
        EV.layout_2_depth(gts[i], h=256, w=512)
    losses = EV.summarize(EV.eval_general([dts[i], None], [gts[i], gts[i]]), [gts[i], gts[i]])
    assert len(losses['8']['2DIoU']) == 2 and len(losses['overall']['rmse']) == 2


@pytest.mark.parametrize('backbone,use_rnn', [('resnet50', True), ('resnet50', False), ('resnet18', True),
                                              ('resnet18', False)])
def test_validate_matches_infer_layout_and_the_oracle(backbone, use_rnn):
    net = HorizonNet(backbone, use_rnn).eval()
    net.load_state_dict(synthetic_state_dict(2, 'random', use_rnn=use_rnn, backbone=backbone), strict=True)
    net = net.to('cuda:0')
    x = synthetic_panoramas(3, seed=102)
    gts = [_room(7), _room(8), _room(9)]
    with torch.no_grad():
        got = EV.validate(net, x, gts, return_status=True)
        lay, st = infer_layout(net, x, force_raw=True, return_status=True)
    dts = [lay[b][0] if st[b] in (0, 1) else None for b in range(3)]
    same = EV.eval_general(dts, gts, return_status=True)            # the same kernels on infer_layout's host results
    for k in ('status', 'iou2d', 'iou3d', 'rmse', 'delta_1'):
        np.testing.assert_array_equal(got[k], same[k])
    for b in range(3):
        want = _oracle(dts[b], gts[b])
        assert int(got['status'][b]) == want['status']
        for k, tol in (('iou2d', 1e-6), ('iou3d', 1e-6), ('delta_1', 4e-6)):
            assert abs(got[k][b] - want[k]) <= tol or (np.isnan(got[k][b]) and np.isnan(want[k])), (k, got[k][b], want[k])
        # No RMSE check against numpy here: the random-weight models put the floor boundary within a few thousandths
        # of a pixel of the horizon, where the wall depth (~1e5) follows the last ulp of numpy's float32 sin / cos.
