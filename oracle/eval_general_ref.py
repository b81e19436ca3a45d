"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the general-layout metrics of reference eval_general.py:14-122.

``test_general(dt_cor_id, gt_cor_id)`` scores one pair of corner lists in pixels (ceiling / floor rows alternating): the
2D IoU of the floor polygons (np_coor2xy with floorW = floorH = 1), the 3D IoU with the get_z1 heights, and the RMSE and
delta_1 of the two depth renders of ``layout_2_depth`` (dataset.cor_2_1d, misc/panostretch.pano_connect_points).  dtypes
follow numpy's at every step: a float32 corner list keeps the per-corner steps in float32 and the per-column ones in
float64; train.py's int64 fallback box is float64 from the first step.

The reference leaves some results to shapely and to unspecified sort orders.  They are fixed here and in
csrc/layout_eval.cu alike (DESIGN.md section 9):
  * validity of a floor ring is ``layout_ref.is_simple_ring`` of its float32 vertices (the layout kernel's definition);
    gt invalid -> SKIP (the reference prints "Skip ground truth invalid"), dt invalid -> iou2d = iou3d = 0 (the except
    branches that catch shapely's refusal to intersect an invalid polygon);
  * the intersection area of two valid rings comes from Green's theorem: each edge split at its crossings with the
    other ring, the pieces inside the other ring kept, a piece on an edge of the other ring kept once when both run the
    same way after orienting both counter-clockwise, and not at all when they run opposite ways;
  * argsort ties of sort_xy_filter_unique and duplicate x % 1024 in np.interp's period sort keep the concatenation
    order (stable sorts).

Pinned by tests/golden/eval_general.npz (minted from the real reference by tests/golden/make_golden_eval.py)."""
import numpy as np

from oracle.layout_ref import is_simple_ring

W, H = 1024, 512
PI = float(np.pi)

# status codes of hn_layout_eval_general (include/horizonnet_b200.h)
OK, DT_INVALID, SKIP, ERR_GT_DEPTH, ERR_COLUMNS, ERR_RING = 0, 1, 2, 3, 4, 5
STATUS_NAMES = {OK: 'ok', DT_INVALID: 'dt_invalid', SKIP: 'skip_gt_invalid', ERR_GT_DEPTH: 'gt_depth',
                ERR_COLUMNS: 'columns', ERR_RING: 'ring'}


def fallback_box():
    """train.py:310-313: what the validation scores when inference() raises (int64, pixels)."""
    return np.array([[k // 2 * 1024, 256 - ((k % 2) * 2 - 1) * 120] for k in range(8)])


# ---------------------------------------------------------------------------------------------- cor_2_1d
def connect(p1, p2, z):
    """pano_connect_points(p1, p2, z, 1024, 512): the wall's boundary sampled at every integer column it spans."""
    if p1[0] == p2[0]:
        return np.array([p1, p2], np.float32)

    def xy(p):
        u = ((p[0] + 0.5) / W - 0.5) * 2 * PI
        v = ((p[1] + 0.5) / H - 0.5) * PI
        c = z / np.tan(v)
        return c * np.cos(u), c * np.sin(u)

    x1, y1 = xy(p1)
    x2, y2 = xy(p2)
    if abs(p1[0] - p2[0]) < W / 2:
        lo, hi = np.ceil(min(p1[0], p2[0])), np.floor(max(p1[0], p2[0]))
    else:
        lo, hi = np.ceil(max(p1[0], p2[0])), np.floor(min(p1[0], p2[0]) + W)
    cols = (np.arange(lo, hi + 1) % W).astype(np.float64)
    t = np.tan(((cols + 0.5) / W - 0.5) * 2 * PI)
    s = (t * x1 - y1) / ((y2 - y1) - t * (x2 - x1))
    dist = np.sqrt((x1 + s * (x2 - x1)) ** 2 + (y1 + s * (y2 - y1)) ** 2)
    rows = (np.arctan2(z, dist) / PI + 0.5) * H - 0.5
    return np.stack([cols, rows], axis=-1)


def boundary_points(cor, floor):
    """The concatenated samples of one boundary's walls, as cor_2_1d collects them (lists of numpy scalars)."""
    n = len(cor)
    xs, ys = [], []
    for i in range(n // 2):
        a, b = (2 * i + 1, (2 * i + 3) % n) if floor else (2 * i, (2 * i + 2) % n)
        p = connect(cor[a], cor[b], 50 if floor else -50)
        xs.extend(p[:, 0])
        ys.extend(p[:, 1])
    return np.array(xs), np.array(ys)


def first_per_x(xs, ys, y_small_first):
    """sort_xy_filter_unique with a stable argsort."""
    order = np.argsort(xs + ys / ys.max() * (int(y_small_first) * 2 - 1), kind='stable')
    xs, ys = xs[order], ys[order]
    _, first = np.unique(xs, return_index=True)
    return xs[first], ys[first]


def periodic_interp(xs, ys):
    """np.interp(arange(W), xs, ys, period=W) with a stable sort of xs % W."""
    xp = xs % W
    order = np.argsort(xp, kind='stable')
    xp, fp = xp[order], ys[order]
    xp = np.concatenate([xp[-1:] - W, xp, xp[0:1] + W])
    fp = np.concatenate([fp[-1:], fp, fp[0:1]])
    return np.interp(np.arange(W), xp, fp)


def cor_2_1d(cor):
    """[2][1024] float64 ceiling / floor boundary angles of a corner list in pixels."""
    bon = np.zeros((2, W))
    for k, floor in enumerate((False, True)):
        xs, ys = first_per_x(*boundary_points(cor, floor), y_small_first=not floor)
        bon[k] = periodic_interp(xs, ys)
    return ((bon + 0.5) / H - 0.5) * np.pi


def order_dependent(cor):
    """Whether cor_2_1d of this corner list depends on a sort order the reference leaves unspecified: two points of one
    boundary with the same x and key but different y, or two kept points with the same x % 1024 but different y."""
    for floor in (False, True):
        xs, ys = boundary_points(cor, floor)
        key = xs + ys / ys.max() * (1 - 2 * int(floor))
        for x in np.unique(xs):
            sel = xs == x
            k = key[sel]
            if len(np.unique(ys[sel][k == k.min()])) > 1:
                return True
        ux, uy = first_per_x(xs, ys, not floor)
        m = ux % W
        for x in np.unique(m):
            if len(np.unique(uy[m == x])) > 1:
                return True
    return False


# ---------------------------------------------------------------------------------------------- depth
class DepthAssertion(Exception):
    pass


def layout_2_depth(cor):
    """[512][1024] float32 depth of a layout (eval_general.py:14-54); raises DepthAssertion where it asserts, and where
    cor_2_1d finds no sample (ys.max() of nothing: ValueError)."""
    xs_ok = all(len(boundary_points(cor, f)[0]) for f in (False, True))
    if not xs_ok:
        raise DepthAssertion('no wall samples a column')
    vc, vf = cor_2_1d(cor)
    if (vc > 0).sum() or (vf < 0).sum():
        raise DepthAssertion('boundary on the wrong side of the horizon')
    vs = ((np.arange(H) + 0.5) / H - 0.5) * np.pi
    vs = np.repeat(vs[:, None], W, axis=1)
    cs = 1.6 / np.tan(vf)
    ceil_h = np.abs(cs * np.tan(vc))
    with np.errstate(divide='ignore', invalid='ignore'):
        depth = np.where(vs < vc, np.abs(ceil_h / np.sin(vs)),
                         np.where(vs > vf, np.abs(1.6 / np.sin(vs)), np.abs(cs / np.cos(vs)))).astype(np.float32)
    if (depth == 0).sum():
        raise DepthAssertion('zero depth')
    return depth


# ---------------------------------------------------------------------------------------------- polygons
def floor_xy(floor):
    """np_coor2xy(floor, -1.6, 1024, 512, floorW=1, floorH=1) in the corners' dtype."""
    u = ((floor[:, 0] + 0.5) / W - 0.5) * 2 * PI
    v = -((floor[:, 1] + 0.5) / H - 0.5) * PI
    c = -1.6 / np.tan(v)
    return np.stack([c * np.sin(u) + 0.0, -c * np.cos(u) + 0.0], -1)


def heights(floor_y, ceil_y):
    """get_z1(floor y, ceiling y, -1.6, 512)."""
    v0 = -((floor_y + 0.5) / H - 0.5) * PI
    v1 = -((ceil_y + 0.5) / H - 0.5) * PI
    return -1.6 / np.tan(v0) * np.tan(v1)


def signed_area(p):
    p = np.asarray(p, np.float64)
    q = np.roll(p, -1, 0)
    return float((p[:, 0] * q[:, 1] - p[:, 1] * q[:, 0]).sum()) / 2


def _cross(ax, ay, bx, by):
    return ax * by - ay * bx


def _inside(q, mx, my):
    inside = False
    n = len(q)
    for j in range(n):
        (cx, cy), (ex, ey) = q[j], q[(j + 1) % n]
        if (cy > my) != (ey > my) and mx < (ex - cx) * (my - cy) / (ey - cy) + cx:
            inside = not inside
    return inside


def _edge_part(p, i, sp, q, sq, own):
    """Twice the area contribution of edge i of ring p to the intersection with ring q (see the module docstring)."""
    (ax, ay), (bx, by) = p[i], p[(i + 1) % len(p)]
    dx, dy = bx - ax, by - ay
    dd = dx * dx + dy * dy
    if dd == 0:
        return 0.0
    nq = len(q)
    total, t0, x0, y0 = 0.0, 0.0, ax, ay
    while t0 < 1:
        t1 = 1.0
        for j in range(nq):
            (qx0, qy0), (qx1, qy1) = q[j], q[(j + 1) % nq]
            cx, cy, fx, fy = qx0 - ax, qy0 - ay, qx1 - qx0, qy1 - qy0
            den = _cross(dx, dy, fx, fy)
            if den == 0:
                if _cross(cx, cy, dx, dy) != 0:
                    continue
                for t in ((cx * dx + cy * dy) / dd, ((qx1 - ax) * dx + (qy1 - ay) * dy) / dd):
                    if t0 < t < t1:
                        t1 = t
            else:
                t, u = _cross(cx, cy, fx, fy) / den, _cross(cx, cy, dx, dy) / den
                if 0 <= u <= 1 and t0 < t < t1:
                    t1 = t
        tm = 0.5 * (t0 + t1)
        shared = 0
        for j in range(nq):
            (qx0, qy0), (qx1, qy1) = q[j], q[(j + 1) % nq]
            cx, cy, fx, fy = qx0 - ax, qy0 - ay, qx1 - qx0, qy1 - qy0
            if _cross(dx, dy, fx, fy) != 0 or _cross(cx, cy, dx, dy) != 0:
                continue
            tc, te = (cx * dx + cy * dy) / dd, ((qx1 - ax) * dx + (qy1 - ay) * dy) / dd
            if min(tc, te) < tm < max(tc, te):
                shared = 1 if (dx * fx + dy * fy) * sp * sq > 0 else -1
                break
        x1, y1 = (bx, by) if t1 >= 1 else (ax + t1 * dx, ay + t1 * dy)
        keep = (own and shared > 0) if shared else _inside(q, ax + tm * dx, ay + tm * dy)
        if keep:
            total += _cross(x0, y0, x1, y1)
        t0, x0, y0 = t1, x1, y1
    return total * sp


def intersection_area(p, q):
    """Area of the intersection of two simple rings (float64 [n][2])."""
    p = [(float(x), float(y)) for x, y in p]
    q = [(float(x), float(y)) for x, y in q]
    sp = -1.0 if signed_area(p) < 0 else 1.0
    sq = -1.0 if signed_area(q) < 0 else 1.0
    t = sum(_edge_part(p, i, sp, q, sq, True) for i in range(len(p)))
    t += sum(_edge_part(q, i, sq, p, sp, False) for i in range(len(q)))
    return t / 2


# ---------------------------------------------------------------------------------------------- test_general
def test_general(dt_cor_id, gt_cor_id):
    """One pair in pixels -> dict(status, iou2d, iou3d, rmse, delta_1, h_dt, h_gt); metrics NaN where not scored."""
    out = dict(status=OK, iou2d=np.nan, iou3d=np.nan, rmse=np.nan, delta_1=np.nan, h_dt=np.nan, h_gt=np.nan)
    dt, gt = np.asarray(dt_cor_id), np.asarray(gt_cor_id)
    for c in (dt, gt):
        if len(c) % 2 or (c[1::2, 0] != c[0::2, 0]).sum():
            out['status'] = ERR_COLUMNS
            return out
    if len(dt) < 6 or len(gt) < 6:
        out['status'] = ERR_RING
        return out
    dt_xy, gt_xy = floor_xy(dt[1::2]), floor_xy(gt[1::2])
    if not is_simple_ring(gt_xy.astype(np.float32)):
        out['status'] = SKIP
        return out
    if not is_simple_ring(dt_xy.astype(np.float32)):
        out['status'] = DT_INVALID
        out['iou2d'] = out['iou3d'] = 0.0
    else:
        a_dt, a_gt = abs(signed_area(dt_xy)), abs(signed_area(gt_xy))
        inter = intersection_area(dt_xy, gt_xy)
        out['iou2d'] = inter / (a_gt + a_dt - inter)
        h_dt = abs(heights(dt[1::2, 1], dt[0::2, 1]).mean() - -1.6)
        h_gt = abs(heights(gt[1::2, 1], gt[0::2, 1]).mean() - -1.6)
        out['h_dt'], out['h_gt'] = h_dt, h_gt
        i3 = inter * min(h_dt, h_gt)
        out['iou3d'] = i3 / (a_dt * h_dt + a_gt * h_gt - i3)
    try:
        g = layout_2_depth(gt)
    except DepthAssertion:
        out.update(status=ERR_GT_DEPTH, iou2d=np.nan, iou3d=np.nan)
        return out
    try:
        d = layout_2_depth(dt)
    except DepthAssertion:
        d = np.zeros_like(g)
    out['rmse'] = float(((g - d) ** 2).mean() ** 0.5)
    with np.errstate(divide='ignore', invalid='ignore'):
        out['delta_1'] = float((np.maximum(g / d, d / g) < 1.25).mean())
    return out


def dt_pixels(dt_normalised):
    """eval_general.py:156-158 / train.py:307-308: a normalised float32 cor_id scaled to pixels in float32."""
    d = np.array(dt_normalised, np.float32)
    d[:, 0] *= W
    d[:, 1] *= H
    return d


def bucket(n_rows):
    """eval_general.py:106-113: the corner-count bucket of a gt with n_rows rows."""
    n = n_rows // 2
    if n % 2 == 1:
        return 'odd'
    return str(n) if n < 10 else '10+'
