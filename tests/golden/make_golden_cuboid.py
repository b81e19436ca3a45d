"""Mint tests/golden/eval_cuboid.npz by running the REAL reference's eval_cuboid.py (read-only, at
make_golden_layout.REF) on CPU.  Run where that reference checkout exists:
    python tests/golden/make_golden_cuboid.py

Pairs (dt, z0, z1, gt), 8-row corner lists in pixels as eval_cuboid.py's test() receives them, z0 and z1 Python floats
as json.load gives them:
  * the synthetic cuboid rooms of make_golden_layout.py (room_corners with no notch) as gt, against jittered copies;
  * the reference's own force_cuboid outputs (tests/golden/layout.npz */cub_cor_id and z1, the random-weight model
    included) against those rooms;
  * hand-made cases: one per error the reference raises, and one per quirk of its code (a ceiling row that wraps to the
    bottom, a bow-tie dt, two dt corners in one column, corners at integer columns, a wall across the seam, every dt
    ceiling corner below the horizon).
For each pair the file records CE, PE, the raw count of differing pixels and 3DIoU from test(), or the name of the
exception it raised; the four 1024-column boundary rows of eval_cuboid.py:106-127, computed with the reference's
functions where they compute, at every 8th column (`columns`; the dt rows per pair, the gt rows once per gt and z0 under
gt_bon/<gt_key>); and whether
numpy's unstable argsort order can decide a boundary value (`tie`: two points with the same x % 1024 and different
rows).

Shims, for the import only: make_golden_layout.py's (shapely placeholders, scipy.ndimage.filters).  The reference's
functions are called unchanged."""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import make_golden_layout as mgl     # noqa: E402  (inserts the reference path and the shims)
from make_golden_eval import perturb  # noqa: E402

import eval_cuboid as ref_cub        # noqa: E402  reference eval_cuboid.py
from misc import panostretch, post_proc   # noqa: E402

from oracle import eval_cuboid_ref as C   # noqa: E402  (order_dependent only)

W, H = 1024, 512
COLS = np.arange(0, W, 8)                # the columns whose boundary rows are recorded
Z0 = 50.0
Z1 = -50.0 * 1.6 / 1.4


def cuboid(xs, yc, yf):
    """A hand-made 8-row layout from its 4 columns and ceiling / floor rows (float32 pixels)."""
    c = []
    for x, a, b in zip(xs, yc, yf):
        c += [[x, a], [x, b]]
    return np.array(c, np.float32)


def pairs():
    out = []
    g = np.load(os.path.join(HERE, 'layout.npz'))
    specs = [(0.0, (0.1, -0.2)), (0.35, (0.3, 0.1)), (-0.2, (-0.2, 0.1)), (0.6, (0.0, 0.0)), (0.9, (0.2, -0.3)),
             (-0.7, (-0.3, 0.2)), (1.3, (0.1, 0.1)), (0.2, (0.0, -0.4))]
    rooms = []
    for i, (ang, cam) in enumerate(specs):
        gt = mgl.room_corners(0, ang, cam, seed=50 + i)
        rooms.append(gt)
        out.append(('room%d_self' % i, gt.copy(), Z0, Z1, gt))
        rs = np.random.RandomState(300 + i)
        for j, sd in enumerate((2.0, 6.0)):
            out.append(('room%d_jitter%d' % (i, j), perturb(gt, 400 + 10 * i + j, sd, sd * 0.75), Z0,
                        float(Z1 * (1 + rs.normal(0, 0.05))), gt))
    out.append(('room0_vs_room3', rooms[3], Z0, Z1, rooms[0]))
    cases = sorted({k.split('/')[0] for k in g.files if k.endswith('/cub_cor_id')})
    k = 0
    for case in cases:
        if str(g[case + '/cub_exc']) or g[case + '/cub_cor_id'].shape != (8, 2):
            continue
        dt = C.dt_pixels(g[case + '/cub_cor_id'])
        out.append(('%s_cub_vs_room%d' % (case, k % len(rooms)), dt, Z0, float(g[case + '/z1']), rooms[k % len(rooms)]))
        k += 1
    base = cuboid([100.3, 341.7, 600.2, 855.9], [180.2, 190.4, 175.1, 185.6], [340.3, 330.8, 345.2, 335.7])
    out.append(('base_self', base.copy(), Z0, Z1, base))
    wrap = base.copy()
    wrap[2, 1] = -0.7                                        # a ceiling corner above the top row: the marks wrap
    out.append(('dt_ceiling_row_wraps', wrap, Z0, Z1, base))
    edge = base.copy()
    edge[4:6, 0] = base[2, 0]                                # corners 1, 2 in one column: their rows enter the boundary
    edge[2, 1] = edge[4, 1] = -0.7                           # and infer_coory puts the dt floor there past the last row
    out.append(('dt_vertical_wall_above_top', edge, Z0, Z1, base))
    bow = base[[0, 1, 4, 5, 2, 3, 6, 7]].copy()               # corners out of order: a self-intersecting floor
    out.append(('dt_bowtie', bow, Z0, Z1, base))
    same = base.copy()
    same[2:4, 0] = base[0, 0]                                # two dt corners in one column
    out.append(('dt_two_corners_one_column', same, Z0, Z1, base))
    integ = cuboid([100, 342, 600, 856], [180.2, 190.4, 175.1, 185.6], [340.3, 330.8, 345.2, 335.7])
    out.append(('integer_columns', integ, Z0, Z1, base))
    out.append(('integer_columns_gt', base.copy(), Z0, Z1, integ))
    seam = cuboid([700.4, 950.1, 150.8, 420.3], [185.2, 178.9, 190.3, 181.0], [335.1, 341.9, 330.4, 338.8])
    seam_gt = cuboid([702.0, 948.5, 152.2, 418.7], [183.0, 180.1, 188.8, 182.4], [337.0, 340.2, 331.9, 337.5])
    out.append(('wall_across_seam', seam, Z0, Z1, seam_gt))
    below = base.copy()
    below[0::2, 1] = [262.0, 270.5, 265.3, 268.1]             # every dt ceiling corner below the horizon
    out.append(('dt_ceiling_below_horizon', below, Z0, Z1, base))
    out.append(('dt_six_rows', base[:6].copy(), Z0, Z1, base))
    cols = base.copy()
    cols[3, 0] += 1.0                                        # a dt floor column differs from its ceiling column
    out.append(('dt_columns_differ', cols, Z0, Z1, base))
    out.append(('gt_columns_differ', base.copy(), Z0, Z1, cols))
    low = base.copy()
    low[4:6, 0] = base[2, 0]
    low[3, 1] = low[5, 1] = 512.2                            # gt floor rows rounding to 512, past the last image row
    out.append(('gt_floor_past_last_row', base.copy(), Z0, Z1, low))
    nan = base.copy()
    nan[4, 1] = np.nan                                       # a NaN ceiling row
    out.append(('dt_nan_row', nan, Z0, Z1, base))
    out.append(('dt_low_z1', base.copy(), Z0, -20.0, base))
    return out


def bounds(dt, z0, z1, gt):
    """eval_cuboid.py:106-127 with the reference's functions: [4][1024] dt ceiling, dt floor, gt ceiling, gt floor."""
    y0_dt, y0_gt, y1_gt = [], [], []
    for j in range(4):
        y0_dt.append(panostretch.pano_connect_points(dt[j * 2], dt[(j * 2 + 2) % 8], -z0))
        y0_gt.append(panostretch.pano_connect_points(gt[j * 2], gt[(j * 2 + 2) % 8], -z0))
        y1_gt.append(panostretch.pano_connect_points(gt[j * 2 + 1], gt[(j * 2 + 3) % 8], z0))
    y0_dt = ref_cub.gen_reg_from_xy(np.concatenate(y0_dt, 0), W)
    y1_dt = post_proc.infer_coory(y0_dt, z1 - z0, z0)
    y0_gt = ref_cub.gen_reg_from_xy(np.concatenate(y0_gt, 0), W)
    y1_gt = ref_cub.gen_reg_from_xy(np.concatenate(y1_gt, 0), W)
    return np.stack([y0_dt, y1_dt, y0_gt, y1_gt])


def run_pair(dt, z0, z1, gt):
    rec = {'dt': dt, 'gt': gt, 'z0': np.float64(z0), 'z1': np.float64(z1)}
    losses = {'CE': [], 'PE': [], '3DIoU': []}
    with np.errstate(all='ignore'):
        try:
            ref_cub.test(dt, z0, z1, gt, W, H, losses)
            rec['exc'] = ''
            rec['ce'], rec['pe'], rec['iou3d'] = (np.float64(losses[k][0]) for k in ('CE', 'PE', '3DIoU'))
            rec['pe_count'] = np.int64(round(float(losses['PE'][0]) * H * W / 100))
        except Exception as e:                              # noqa: BLE001
            rec['exc'] = type(e).__name__
        if len(dt) == 8 and len(gt) == 8:
            try:
                rec['bon'] = bounds(dt, z0, z1, gt)
            except Exception:                               # noqa: BLE001
                pass
            digest = hashlib.sha1(np.ascontiguousarray(gt).tobytes() + repr(z0).encode()).hexdigest()
            rec['gt_key'] = np.array(digest[:16])
            try:
                rec['tie'] = np.bool_(any(C.order_dependent(c, z) for c, z in
                                          ((dt[0::2], -z0), (gt[0::2], -z0), (gt[1::2], z0))))
            except Exception:                               # noqa: BLE001
                rec['tie'] = np.bool_(False)
    return rec


def main():
    out = {'columns': COLS}
    names = []
    for name, dt, z0, z1, gt in pairs():
        names.append(name)
        rec = run_pair(dt, z0, z1, gt)
        for k, v in rec.items():
            if k == 'bon':                                  # the dt rows per pair, the gt rows once per gt and z0
                out[name + '/bon_dt'] = v[:2, COLS]
                out['gt_bon/%s' % rec['gt_key']] = v[2:, COLS]
            else:
                out[name + '/' + k] = np.asarray(v)
        print('%-34s %-14s ce %9s pe %9s iou %10s tie %s' % (
            name, rec['exc'] or 'ok', '%.4f' % rec['ce'] if 'ce' in rec else '-',
            '%.4f' % rec['pe'] if 'pe' in rec else '-', '%.5f' % rec['iou3d'] if 'iou3d' in rec else '-',
            bool(rec.get('tie', False))))
    out['names'] = np.array(names)
    np.savez_compressed(os.path.join(HERE, 'eval_cuboid.npz'), **out)


if __name__ == '__main__':
    main()
