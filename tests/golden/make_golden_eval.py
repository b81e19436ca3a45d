"""Mint tests/golden/eval_general.npz by running the REAL reference's evaluation code (read-only, /root/reference) on CPU.

Run in the build container only (the GPU box has no /root/reference):
    python tests/golden/make_golden_eval.py

Pairs (dt, gt), corner lists in pixels as test_general receives them:
  * the synthetic Manhattan rooms of make_golden_layout.py (4 to 12 corners, rotated, camera off-centre) as gt, against
    perturbed copies of themselves as dt;
  * the layout kernel's force_raw output for the random-weight model (tests/golden/layout.npz raw_cor_id), a 1024-corner
    ring that folds over itself, against rooms;
  * train.py's int64 fallback box against rooms;
  * hand-made cases for each status and for the order-dependent steps (vertical walls, columns past 1024).
(cor_2_1d raises ValueError when no wall samples a column; the reference's test_general lets that escape for the gt.)
For each distinct corner list (stored once, under a digest, as layout/<key>/...) the file records the reference's
cor_2_1d and every 128th row of layout_2_depth at the even columns (or what it raised), and the get_z1 heights
(eval_general.py:86-89); for each pair, the keys of its dt and gt and the RMSE and delta_1 of test_general
(eval_general.py:97-105).
The IoUs are not recorded: shapely is not available, and tests/test_eval_oracle.py pins the areas independently.

Shims, for the import only: shapely (not installed) gets a placeholder Polygon -- nothing here calls it -- and
scipy.ndimage.filters is mapped to scipy.ndimage where recent scipy removed it.  The reference's functions are called
unchanged."""
import hashlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import make_golden_layout as mgl     # noqa: E402  (inserts the reference path and the shims)

for _name in ('shapely', 'shapely.geometry'):
    sys.modules.setdefault(_name, types.ModuleType(_name))
sys.modules['shapely.geometry'].Polygon = object

import eval_general as ref_eval      # noqa: E402  reference eval_general.py
import dataset as ref_ds             # noqa: E402  reference dataset.py
from misc import post_proc           # noqa: E402  reference misc/post_proc.py

from oracle import eval_general_ref as E   # noqa: E402  (order_dependent only)

W, H = 1024, 512
ROWS = np.arange(0, H, 128)
COLS = np.arange(0, W, 2)


def perturb(cor, seed, col_sd=4.0, row_sd=3.0):
    rs = np.random.RandomState(seed)
    d = cor.copy()
    dc = rs.normal(0, col_sd, len(cor) // 2).astype(np.float32)
    d[0::2, 0] += dc
    d[1::2, 0] += dc
    d[:, 1] += rs.normal(0, row_sd, len(cor)).astype(np.float32)
    return d


def rect(x0, x1, yc, yf):
    """A hand-made 4-corner layout from its columns and rows (float32 pixels)."""
    c = []
    for x in (x0, x1, x1 + 300, x0 + 700):
        c += [[x, yc], [x, yf]]
    return np.array(c, np.float32)


def pairs():
    out = []
    g = np.load(os.path.join(HERE, 'layout.npz'))
    specs = [(0, 0.0, (0.1, -0.2)), (0, 0.35, (0.3, 0.1)), (1, 0.0, (-0.2, 0.1)), (1, -0.5, (0.0, 0.0)),
             (2, 0.2, (0.1, 0.1)), (2, 0.0, (0.2, -0.1)), (3, 0.6, (-0.1, 0.0)), (3, 0.0, (0.1, 0.2)),
             (4, 0.1, (0.0, 0.1)), (4, -0.3, (0.2, 0.0))]
    rooms = []
    for i, (k, ang, cam) in enumerate(specs):
        gt = mgl.room_corners(k, ang, cam, seed=i)
        rooms.append(gt)
        out.append(('room%d_%dc_self' % (i, len(gt) // 2), gt.copy(), gt))
        out.append(('room%d_%dc_jitter' % (i, len(gt) // 2), perturb(gt, 100 + i), gt))
    out.append(('room0_vs_room5', rooms[5], rooms[0]))
    out.append(('room8_vs_room2', rooms[2], rooms[8]))
    for s in (0, 200):
        raw = g['randombn_roll%d/raw_cor_id' % s]
        out.append(('raw_roll%d_vs_room%d' % (s, s // 100), E.dt_pixels(raw), rooms[s // 100]))
    out.append(('fallback_vs_room0', E.fallback_box(), rooms[0]))
    out.append(('fallback_vs_room9', E.fallback_box(), rooms[9]))
    base = rect(100, 300, 180, 340)
    out.append(('rect_self', base.copy(), base))
    bad_cols = base.copy()
    bad_cols[1, 0] += 1
    out.append(('dt_columns_differ', bad_cols, base))
    out.append(('gt_columns_differ', base.copy(), bad_cols))
    out.append(('dt_odd_rows', base[:7].copy(), base))
    out.append(('dt_two_corners', base[:4].copy(), base))
    bow = base[[0, 1, 4, 5, 2, 3, 6, 7]].copy()              # corners out of order: a self-intersecting floor ring
    out.append(('dt_bowtie', bow, base))
    out.append(('gt_bowtie', base.copy(), bow))
    low = np.array([[100.1, 150], [100.1, 340], [100.3, 200], [100.3, 400], [100.5, 120], [100.5, 380], [100.7, 180],
                    [100.7, 350]], np.float32)              # every wall inside one pixel column: no column sampled
    out.append(('gt_no_column_sampled', base.copy(), low))
    out.append(('dt_no_column_sampled', low, base))
    vert = np.array([[100, 180], [100, 340], [100, 150], [100, 360], [500, 170], [500, 350], [800, 175], [800, 345]],
                    np.float32)                             # two corners in one column: a wall seen edge-on
    out.append(('vertical_wall', vert, rooms[0]))
    wrap = base.copy()
    wrap[4:, 0] = 1030                                      # a wall seen edge-on past the width: its corners keep x = 1030,
    #                                                         which np.interp's period then folds onto column 6
    out.append(('column_past_width', wrap, base))
    return out


def layout_key(cor):
    """Records of one corner list are stored once, under a digest of its dtype and values."""
    return hashlib.sha1(str(cor.dtype).encode() + np.ascontiguousarray(cor).tobytes()).hexdigest()[:16]


def run_layout(cor):
    rec = {'cor': cor}
    try:
        rec['bon'] = ref_ds.cor_2_1d(cor, H, W)[:, COLS]
    except Exception as e:                                  # noqa: BLE001
        rec['bon_exc'] = type(e).__name__
    try:
        rec['depth_rows'] = ref_eval.layout_2_depth(cor, H, W)[ROWS][:, COLS]
        rec['depth_exc'] = ''
    except (AssertionError, ValueError) as e:
        rec['depth_exc'] = type(e).__name__
    try:
        rec['order_dependent'] = np.bool_(len(cor) % 2 == 0 and E.order_dependent(cor))
    except ValueError:                                      # no sample: nothing to order
        rec['order_dependent'] = np.bool_(False)
    if len(cor) % 2 == 0 and len(cor) >= 2:
        rec['z1'] = post_proc.get_z1(cor[1::2, 1], cor[0::2, 1], -1.6, 512)
    return rec


def run_pair(dt, gt):
    """RMSE and delta_1 of test_general (eval_general.py:97-105), when layout_2_depth accepts the gt."""
    try:
        g = ref_eval.layout_2_depth(gt, H, W)
    except (AssertionError, ValueError):
        return {}
    try:
        d = ref_eval.layout_2_depth(dt, H, W)
    except Exception:                                       # noqa: BLE001 -- eval_general.py:100-101
        d = np.zeros_like(g)
    with np.errstate(divide='ignore', invalid='ignore'):
        return {'rmse': np.float64(((g - d) ** 2).mean() ** 0.5),
                'delta_1': np.float64((np.maximum(g / d, d / g) < 1.25).mean())}


def main():
    out = {'depth_rows': ROWS, 'columns': COLS}
    names = []
    for name, dt, gt in pairs():
        names.append(name)
        for side, cor in (('dt', dt), ('gt', gt)):
            key = layout_key(cor)
            out['%s/%s_key' % (name, side)] = np.array(key)
            if 'layout/%s/cor' % key not in out:
                with np.errstate(divide='ignore', invalid='ignore'):
                    for k, v in run_layout(cor).items():
                        out['layout/%s/%s' % (key, k)] = np.asarray(v)
        rec = run_pair(dt, gt)
        for k, v in rec.items():
            out[name + '/' + k] = np.asarray(v)
        print('%-26s rows %4d/%2d  rmse %8s  delta_1 %8s' % (
            name, len(dt), len(gt), '%.4f' % rec['rmse'] if 'rmse' in rec else '-',
            '%.4f' % rec['delta_1'] if 'delta_1' in rec else '-'))
    out['names'] = np.array(names)
    np.savez_compressed(os.path.join(HERE, 'eval_general.npz'), **out)


if __name__ == '__main__':
    main()
