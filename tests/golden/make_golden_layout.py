"""Mint tests/golden/layout.npz by running the REAL reference's layout post-processing (read-only, /root/reference) on CPU.

Run in the build container only (the GPU box has no /root/reference):
    python tests/golden/make_golden_layout.py

Cases:
  * synthetic Manhattan rooms of 4, 6, 8, 10 and 12 corners (a rectangle with 0-4 of its corners notched), some rotated
    off the image axes, with the camera off-centre: the boundaries come from reference dataset.cor_2_1d, the corner
    signal is 0.96 ** (column distance to the nearest corner) as dataset.py:108-120 builds it, both with seeded noise;
  * the TTA output of the random-weight model (tta_randombn.npz) and rolled copies of it: degenerate signals with many
    peaks that exercise the deferrals and forced insertions of gen_ww_general;
  * a few hand-made corner signals (too few peaks, a flat plateau).
For each case and each of the general (min_v 0.05), cuboid (min_v 0, N 4) and raw modes, the file records the inputs,
z1, the peaks (and whether the top-4 cut falls inside a tie), the column -> wall-group ids, the walls (axis, value, group), the ceiling corners, the general result's
polygon xy2d before any validity check, the packed cor_id, and the exception type where the reference raises.

Shims, for the import only: shapely (not installed) gets placeholder Polygon / LineString classes -- the validity
verdict itself is not taken from the reference here -- and scipy.ndimage.filters is mapped to scipy.ndimage where
recent scipy removed it.  The reference's functions are called unchanged."""
import os
import sys
import traceback
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference'
sys.path.insert(0, REF)

for _name in ('shapely', 'shapely.geometry'):
    sys.modules.setdefault(_name, types.ModuleType(_name))
sys.modules['shapely.geometry'].Polygon = object
sys.modules['shapely.geometry'].LineString = object
try:
    import scipy.ndimage.filters  # noqa: F401
except Exception:
    import scipy.ndimage
    _m = types.ModuleType('scipy.ndimage.filters')
    _m.maximum_filter = scipy.ndimage.maximum_filter
    sys.modules['scipy.ndimage.filters'] = _m

import inference as ref_inf          # noqa: E402  reference inference.py (find_N_peaks)
import dataset as ref_ds             # noqa: E402  reference dataset.py (cor_2_1d)
from misc import post_proc           # noqa: E402  reference misc/post_proc.py

W, H = 1024, 512
R_PX = int(round(W * 0.05 / 2))


def room_corners(n_notch, angle, cam, seed):
    """Pixel corners [2n][2] (ceiling, floor per corner) of a notched rectangle seen from cam, ceiling 1.4 above and
    floor 1.6 below the camera; first corner = smallest column, as the dataset orders them."""
    rs = np.random.RandomState(seed)
    hx, hy = rs.uniform(2.0, 4.0), rs.uniform(2.0, 4.0)
    quads = [(1, 1), (-1, 1), (-1, -1), (1, -1)]
    poly = []
    for k, (sx, sy) in enumerate(quads):                 # counter-clockwise corners, some cut by a notch
        cx, cy = sx * hx, sy * hy
        if k < n_notch:
            nx, ny = rs.uniform(0.3, 0.45) * hx, rs.uniform(0.3, 0.45) * hy
            a, b = (cx, cy - sy * ny), (cx - sx * nx, cy - sy * ny)
            c = (cx - sx * nx, cy)
            pts = [a, b, c] if sx * sy > 0 else [c, b, a]
            poly += pts
        else:
            poly.append((cx, cy))
    poly = np.array(poly) - np.asarray(cam)
    ca, sa = np.cos(angle), np.sin(angle)
    poly = poly @ np.array([[ca, sa], [-sa, ca]])
    u = np.arctan2(poly[:, 0], -poly[:, 1])
    d = np.hypot(poly[:, 0], poly[:, 1])
    col = (u / (2 * np.pi) + 0.5) * W - 0.5
    rows_c = (-np.arctan(1.4 / d) / np.pi + 0.5) * H - 0.5
    rows_f = (np.arctan(1.6 / d) / np.pi + 0.5) * H - 0.5
    order = np.argsort(col)
    cor = np.zeros((2 * len(col), 2), np.float32)
    cor[0::2, 0] = col[order]
    cor[1::2, 0] = col[order]
    cor[0::2, 1] = rows_c[order]
    cor[1::2, 1] = rows_f[order]
    return cor


def room_signals(cor, seed, bon_noise, cor_noise):
    """Network-like outputs of one room: pixel-row boundaries as tta_merge_kernel leaves them, and y_cor."""
    rs = np.random.RandomState(1000 + seed)
    bon = ref_ds.cor_2_1d(cor, H, W) + rs.normal(0, bon_noise, (2, W))
    bon = bon.astype(np.float32)
    y_bon = (bon / np.float32(np.pi) + np.float32(0.5)) * np.float32(H) - np.float32(0.5)
    y_bon[0] = np.clip(y_bon[0], 1, H / 2 - 1)
    y_bon[1] = np.clip(y_bon[1], H / 2 + 1, H - 2)
    x = np.arange(W)[None, :]
    cx = cor[0::2, 0].astype(np.float64)[:, None]
    dist = np.min([np.abs(cx - x), np.abs(cx - x - W), np.abs(cx - x + W)], 0).min(0)
    y_cor = np.clip(0.96 ** dist + rs.normal(0, cor_noise, W), 0, 1).astype(np.float32)
    return y_bon.astype(np.float32), y_cor


def cases():
    out = []
    specs = [(0, 0.0, (0.1, -0.2)), (0, 0.35, (0.3, 0.1)), (1, 0.0, (-0.2, 0.1)), (1, -0.5, (0.0, 0.0)),
             (2, 0.2, (0.1, 0.1)), (2, 0.0, (0.2, -0.1)), (3, 0.6, (-0.1, 0.0)), (3, 0.0, (0.1, 0.2)),
             (4, 0.1, (0.0, 0.1)), (4, -0.3, (0.2, 0.0))]
    for i, (k, ang, cam) in enumerate(specs):
        cor = room_corners(k, ang, cam, seed=i)
        for j, (bn, cn) in enumerate([(0.002, 0.01), (0.01, 0.04)]):
            yb, yc = room_signals(cor, 10 * i + j, bn, cn)
            out.append(('room%d_%dc_%s' % (i, 4 + 2 * k, 'clean' if j == 0 else 'noisy'), yb, yc))
    g = np.load(os.path.join(HERE, 'tta_randombn.npz'))
    for s in (0, 200, 517):
        out.append(('randombn_roll%d' % s, np.roll(g['y_bon'], s, 1).astype(np.float32),
                    np.roll(g['y_cor'], s).astype(np.float32)))
    yb = out[0][1]
    two = np.full(W, 0.01, np.float32)
    two[[100, 600]] = 0.9
    out.append(('two_peaks', yb, two))
    three = np.full(W, 0.01, np.float32)
    three[[100, 400, 800]] = 0.9
    out.append(('three_peaks', yb, three))
    flat = np.full(W, 0.5, np.float32)
    out.append(('plateau', yb, flat))
    out.append(('no_peaks', yb, np.full(W, 0.01, np.float32)))
    low = yb.copy()                                  # floor boundary at the horizon: |z1| and tol below 1
    low[1] = np.float32(H / 2 + 1) + np.float32(0.25) * (np.arange(W) % 3).astype(np.float32)
    pair = out[0][2].copy()
    pair[300:302] = 0.97                             # a two-column plateau: a one-column wall group
    out.append(('low_floor', low, pair))
    return out


def exc_kind(e):
    if isinstance(e, AssertionError):
        fn = traceback.extract_tb(e.__traceback__)[-1].name
        return 'vote' if fn == 'vote' else 'groups'
    return type(e).__name__


def packed(cor, z1):
    """cor_id as inference.py:128-139 builds it, with the reference's infer_coory."""
    full = np.hstack([cor, post_proc.infer_coory(cor[:, 1], z1 - 50, 50)[:, None]])
    cid = np.zeros((2 * len(full), 2), np.float32)
    cid[0::2] = full[:, [0, 1]]
    cid[1::2] = full[:, [0, 2]]
    cid[:, 0] /= W
    cid[:, 1] /= H
    return cid


def run(yb, yc):
    rec = {}
    _, z1 = post_proc.np_refine_by_fix_z(*yb, 50)
    rec['z1'] = np.float32(z1)
    tol = abs(0.16 * z1 / 1.6)
    for mode, min_v, n, cub in (('gen', 0.05, None, False), ('cub', 0, 4, True)):
        pk = ref_inf.find_N_peaks(yc, r=R_PX, min_v=min_v, N=n)[0]
        rec[mode + '_peaks'] = pk.astype(np.int64)
        rec[mode + '_gid'] = post_proc.get_gpid(pk, W).astype(np.int64)
        if n is not None:                  # top-n cut inside a run of equal values: argsort's order is unspecified
            cand = np.sort(yc[np.where(ref_inf.maximum_filter(yc, size=R_PX, mode='wrap') == yc)[0]])[::-1]
            cand = cand[cand > min_v]
            rec[mode + '_tie'] = np.bool_(len(cand) > n and cand[n - 1] == cand[n])
        try:
            cor, xy_cor = post_proc.gen_ww(pk, yb[0], 50, tol=tol, force_cuboid=cub)
        except Exception as e:             # noqa: BLE001 -- the kind is the record
            rec[mode + '_exc'] = exc_kind(e)
            continue
        rec[mode + '_exc'] = ''
        rec[mode + '_axis'] = np.array([w['type'] for w in xy_cor], np.int64)
        rec[mode + '_val'] = np.array([w['val'] for w in xy_cor], np.float64)
        rec[mode + '_group'] = np.array([w.get('gpid', j) for j, w in enumerate(xy_cor)], np.int64)
        rec[mode + '_cor'] = cor
        rec[mode + '_cor_id'] = packed(cor, z1)
        if not cub:
            xy2d = np.zeros((len(xy_cor), 2), np.float32)
            for i in range(len(xy_cor)):
                xy2d[i, xy_cor[i]['type']] = xy_cor[i]['val']
                xy2d[i, xy_cor[i - 1]['type']] = xy_cor[i - 1]['val']
            rec['gen_xy2d'] = xy2d
    raw = np.stack([np.arange(W), yb[0]], 1)
    rec['raw_cor_id'] = packed(raw, z1)
    return rec


def main():
    out = {'r_px': np.int64(R_PX)}
    names = []
    for name, yb, yc in cases():
        rec = run(yb, yc)
        names.append(name)
        out[name + '/y_bon'] = yb
        out[name + '/y_cor'] = yc
        for k, v in rec.items():
            out[name + '/' + k] = np.asarray(v)
        print('%-22s z1 %9.4f  general %2d peaks %-6s cuboid %s' % (
            name, rec['z1'], len(rec['gen_peaks']), rec['gen_exc'] or len(rec.get('gen_axis', [])),
            rec['cub_exc'] or 'ok'))
    out['names'] = np.array(names)
    np.savez_compressed(os.path.join(HERE, 'layout.npz'), **out)


if __name__ == '__main__':
    main()
