"""-m gpu: the cuboid evaluation kernels (csrc/layout_cuboid.cu, hn_layout_eval_cuboid / hn_model_eval_cuboid) against
oracle/eval_cuboid_ref.py, which tests/test_eval_cuboid_oracle.py pins to the real reference.

Statuses must be identical and CE within 1e-6 relative.  The count of differing pixels must be exact, except that each
mark whose oracle row lies within 1e-4 of a half-integer may round the other way (one pixel each): the per-corner steps
of pano_connect_points are float32 sin / cos / tan, which numpy computes up to about 1.5 ulp from the correctly rounded
value the kernel uses (DESIGN.md section 9).  3DIoU within 1e-4 percentage points, except where a plane passes within
float32 rounding of the camera (_camera_on_a_plane).  evaluate_cuboid must equal eval_cuboid on
infer_layout(force_cuboid=True)'s results bit for bit."""
import json
import os

import numpy as np
import pytest
import torch

import __graft_entry__ as entry
from horizonnet_b200 import _lib
from horizonnet_b200 import eval_cuboid as EC
from horizonnet_b200.inference import infer_layout
from horizonnet_b200.model import HorizonNet
from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas
from oracle import eval_cuboid_ref as C

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'eval_cuboid.npz'))
NAMES = [str(n) for n in G['names']]
SCALE = np.array([1024, 512], np.float32)
Z1 = -50.0 * 1.6 / 1.4


@pytest.fixture(scope='module', autouse=True)
def _built():
    entry.build()
    _lib.lib()


def _room(seed):
    """A seeded cuboid room in pixels: a jittered rectangle, rotated, seen from an off-centre camera."""
    rs = np.random.RandomState(seed)
    hx, hy = rs.uniform(1.5, 4.0, 2)
    p = np.array([(hx, hy), (-hx, hy), (-hx, -hy), (hx, -hy)]) - rs.uniform(-0.4, 0.4, 2)
    a = rs.uniform(-np.pi, np.pi)
    p = p @ np.array([[np.cos(a), np.sin(a)], [-np.sin(a), np.cos(a)]])
    u, d = np.arctan2(p[:, 0], -p[:, 1]), np.hypot(p[:, 0], p[:, 1])
    col = (u / (2 * np.pi) + 0.5) * 1024 - 0.5
    order = np.argsort(col)
    cor = np.zeros((8, 2), np.float32)
    cor[0::2, 0] = cor[1::2, 0] = col[order]
    cor[0::2, 1] = ((-np.arctan(1.4 / d) / np.pi + 0.5) * 512 - 0.5)[order]
    cor[1::2, 1] = ((np.arctan(1.6 / d) / np.pi + 0.5) * 512 - 0.5)[order]
    return cor


def _jitter(cor, seed):
    rs = np.random.RandomState(seed)
    d = cor.copy()
    dc = rs.normal(0, 5, 4).astype(np.float32)
    d[0::2, 0] += dc
    d[1::2, 0] += dc
    d[:, 1] += rs.normal(0, 4, 8).astype(np.float32)
    return d


def _near_half(bon):
    """Marks of the oracle whose row lies within 1e-4 of a half-integer: each may round the other way."""
    if bon is None:
        return 0
    with np.errstate(invalid='ignore'):
        return int((np.abs(np.abs(bon - np.floor(bon)) - 0.5) < 1e-4).sum())


def _camera_on_a_plane(dt_px, gt):
    """Whether a plane of either room passes within 1e-5 x the rooms' scale of the camera.  Two corners in one column
    give such planes: through the camera up to the float32 rounding of the corners, so which side of the camera they
    keep follows the last ulp of numpy's float32 sin / cos / tan (DESIGN.md section 10)."""
    rooms = [C.room_xyz(c[1::2], c[0::2]) for c in (dt_px, gt)]
    R = C.scale_of(*[p for room in rooms for p in room])
    for fl, ce in rooms:
        h = C.halfspaces(fl, ce)
        n = np.linalg.norm(h[:, :3], axis=1)
        if (np.abs(h[:, 3])[n > 0] < 1e-5 * R * n[n > 0]).any():
            return True
    return False


def _check(names, dts, z0s, z1s, gts):
    got = EC.eval_cuboid(dts, z0s, z1s, gts, return_status=True)
    worst = 0.0
    for b, name in enumerate(names):
        dt_px = None if dts[b] is None else C.dt_pixels(dts[b])
        st = int(got['status'][b])
        if dt_px is None:
            assert st == EC.DT_FAILED, name
            continue
        want = C.test_cuboid(dt_px, z0s[b], z1s[b], gts[b])
        assert st == want['status'], (name, C.STATUS_NAMES[st], C.STATUS_NAMES[want['status']])
        if st != C.OK:
            assert np.isnan(got['ce'][b]) and np.isnan(got['pe'][b]) and np.isnan(got['iou3d'][b]), name
            continue
        assert got['ce'][b] == pytest.approx(want['ce'], rel=1e-6, abs=1e-12), name
        cnt = int(round(got['pe'][b] * 512 * 1024 / 100))
        assert abs(cnt - want['pe_count']) <= _near_half(want['bon']), (name, cnt, want['pe_count'])
        assert got['pe'][b] == 100 * cnt / (512 * 1024)
        if _camera_on_a_plane(dt_px, gts[b]):
            continue
        assert abs(got['iou3d'][b] - want['iou3d']) <= 1e-4, (name, got['iou3d'][b], want['iou3d'])
        worst = max(worst, abs(got['iou3d'][b] - want['iou3d']))
    return got, worst


def test_fixture_pairs_match_the_oracle():
    dts = [G[n + '/dt'] / SCALE for n in NAMES]
    z0s = [float(G[n + '/z0']) for n in NAMES]
    z1s = [float(G[n + '/z1']) for n in NAMES]
    gts = [G[n + '/gt'] for n in NAMES]
    got, worst = _check(NAMES, dts, z0s, z1s, gts)
    print('worst 3DIoU difference: %.3g percentage points' % worst)
    assert {int(s) for s in got['status']} >= {EC.OK, EC.ERR_ROWS, EC.ERR_INDEX, EC.ERR_COLUMNS, EC.ERR_HULL}


def test_seeded_batch_of_64_matches_the_oracle():
    gts = [_room(s) for s in range(64)]
    dts = [(_jitter(g, 1000 + s) if s % 4 else g.copy()) / SCALE for s, g in enumerate(gts)]
    rs = np.random.RandomState(5)
    z1s = [float(Z1 * (1 + rs.normal(0, 0.05))) for _ in range(64)]
    got, worst = _check([str(s) for s in range(64)], dts, [50.0] * 64, z1s, gts)
    print('worst 3DIoU difference: %.3g percentage points' % worst)
    assert (got['status'] == EC.OK).sum() >= 60
    assert (got['iou3d'][::4] == 100).all() or np.allclose(got['iou3d'][::4], 100, atol=1e-9)


def test_public_function_raises_like_the_reference():
    base = G['base_self/dt'] / SCALE
    gt = G['base_self/gt']
    cols = G['dt_columns_differ/dt'] / SCALE
    with pytest.raises(AssertionError, match='pair 1'):
        EC.eval_cuboid([base, cols], [50.0, 50.0], [Z1, Z1], [gt, gt])
    with pytest.raises(ValueError, match='pair 0'):
        EC.eval_cuboid([base[:6]], [50.0], [Z1], [gt])
    with pytest.raises(IndexError, match='pair 0'):
        EC.eval_cuboid([G['dt_nan_row/dt'] / SCALE], [50.0], [Z1], [gt])
    r = EC.eval_cuboid([base, None], [50.0, 50.0], [Z1, Z1], [gt, gt], return_status=True)
    assert list(r['status']) == [EC.OK, EC.DT_FAILED] and r['iou3d'][0] == pytest.approx(100.0, abs=1e-9)


@pytest.mark.parametrize('backbone,use_rnn', [('resnet50', True), ('resnet50', False), ('resnet18', True),
                                              ('resnet18', False)])
@pytest.mark.parametrize('tta', [False, True])
def test_evaluate_cuboid_matches_eval_cuboid_on_infer_layout(backbone, use_rnn, tta):
    net = HorizonNet(backbone, use_rnn).eval()
    net.load_state_dict(synthetic_state_dict(2, 'random', use_rnn=use_rnn, backbone=backbone), strict=True)
    net = net.to('cuda:0')
    x = synthetic_panoramas(3, seed=103)
    gts = [_room(17), _room(18), _room(19)]
    aug = dict(flip=True, rotate=(0.25, 0.5)) if tta else {}
    with torch.no_grad():
        got = EC.evaluate_cuboid(net, x, gts, return_status=True, **aug)
        lay, st = infer_layout(net, x, force_cuboid=True, return_status=True, **aug)
    dts = [lay[b][0] if st[b] in (0, 1) else None for b in range(3)]
    same = EC.eval_cuboid(dts, [lay[b][1] for b in range(3)], [lay[b][2] for b in range(3)], gts, return_status=True)
    for k in ('status', 'ce', 'pe', 'iou3d'):
        np.testing.assert_array_equal(got[k], same[k])
    ok = [b for b in range(3) if dts[b] is not None]
    _check([str(b) for b in ok], [dts[b] for b in ok], [float(lay[b][1]) for b in ok], [float(lay[b][2]) for b in ok],
           [gts[b] for b in ok])


def test_cli_prints_the_reference_summary(tmp_path, capsys):
    names = ['room0_jitter0', 'room3_jitter1', 'wall_across_seam', 'integer_columns']
    (tmp_path / 'gt').mkdir()
    (tmp_path / 'dt').mkdir()
    for i, n in enumerate(names):
        np.savetxt(tmp_path / 'gt' / ('pano%d.txt' % i), G[n + '/gt'], fmt='%.6f')
        uv = (G[n + '/dt'] / SCALE).astype(np.float32)
        with open(tmp_path / 'dt' / ('pano%d.json' % i), 'w') as f:
            json.dump({'z0': float(G[n + '/z0']), 'z1': float(G[n + '/z1']),
                       'uv': [[float(u), float(v)] for u, v in uv]}, f)
    EC.main(['--dt_glob', str(tmp_path / 'dt' / '*'), '--gt_glob', str(tmp_path / 'gt' / '*txt'), '--batch', '3'])
    out = capsys.readouterr().out.splitlines()
    gts = [np.loadtxt(tmp_path / 'gt' / ('pano%d.txt' % i), dtype=np.float32) for i in range(4)]
    dts, z0s, z1s = [], [], []
    for i in range(4):
        with open(tmp_path / 'dt' / ('pano%d.json' % i)) as f:
            d = json.load(f)
        dts.append(np.array(d['uv'], np.float32))
        z0s.append(d['z0'])
        z1s.append(d['z1'])
    r = EC.eval_cuboid(dts, z0s, z1s, gts)
    assert out == [' Testing Result '.center(50, '='),
                   'Corner Error (%): ' + str(np.mean([float(v) for v in r['ce']])),
                   'Pixel  Error (%): ' + str(np.mean([float(v) for v in r['pe']])),
                   '3DIoU        (%): ' + str(np.mean([float(v) for v in r['iou3d']])),
                   '=' * 50]
