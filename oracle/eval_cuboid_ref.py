"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the cuboid metrics of reference eval_cuboid.py:13-145.

``test_cuboid(dt_cor_id, z0, z1, gt_cor_id)`` scores one pair of 8-row corner lists in pixels (ceiling / floor rows
alternating, float32): the corner error, the pixel error of the three-label surfaces and the 3D IoU of the two rooms.
dtypes follow numpy's at every step: the per-corner steps are float32, the per-column ones float64.

Where the reference leaves the result to qhull or to an unspecified sort order, the rules are fixed here and in
csrc/layout_cuboid.cu alike (DESIGN.md section 10):
  * gen_reg_from_xy's two argsorts keep the concatenation order among equal keys (stable sorts);
  * the 3D IoU clips a bounding box by the oriented planes of xyzlst2halfspaces, duplicates included, instead of asking
    qhull (``clip_volume``): a zero normal is a no-op, a plane through the origin is qhull's "feasible point is not
    clearly inside halfspace", a result that still touches the box is the unbounded region qhull refuses, and a result
    of (near) zero volume is qhull's flat initial simplex.  The largest box reaches 65536 times the rooms' scale: a
    region reaching further is refused as unbounded.  Such regions come from planes that are (nearly) parallel, where
    qhull's roundoff decides how far away it closes them and the reference reports a near-zero IoU
    that depends on that roundoff (below 1e-3 % in every such fixture pair).

Pinned by tests/golden/eval_cuboid.npz (minted from the real reference by tests/golden/make_golden_cuboid.py)."""
import numpy as np

from oracle.eval_general_ref import connect

W, H = 1024, 512
PI = float(np.pi)

# status codes of hn_layout_eval_cuboid (include/horizonnet_b200.h)
OK, ERR_ROWS, ERR_INDEX, ERR_COLUMNS, ERR_HULL, DT_FAILED = 0, 1, 2, 3, 4, 5
STATUS_NAMES = {OK: 'ok', ERR_ROWS: 'rows', ERR_INDEX: 'index', ERR_COLUMNS: 'columns', ERR_HULL: 'hull',
                DT_FAILED: 'dt_failed'}
# the exception the reference raises for each error status
EXCEPTIONS = {ERR_ROWS: 'ValueError', ERR_INDEX: 'IndexError', ERR_COLUMNS: 'AssertionError',
              ERR_HULL: ('ValueError', 'QhullError')}

BOX_SCALES = (16.0, 1024.0, 65536.0)   # starting box half-widths, in units of the largest corner coordinate (+ 1)
ON_PLANE = 1e-10            # a vertex closer to a plane than ON_PLANE * (largest coordinate + 1) lies on it
FLAT_VOLUME = 1e-9          # a clipped volume <= FLAT_VOLUME * (largest coordinate + 1) ** 3 is refused as flat


# ---------------------------------------------------------------------------------------------- corner error
def corner_error(dt, gt):
    """eval_cuboid.py:102-103 (float32 up to the mean, float64 after)."""
    mse = np.sqrt(((gt - dt) ** 2).sum(1)).mean()
    return float(100 * mse / np.sqrt(W ** 2 + H ** 2))


# ---------------------------------------------------------------------------------------------- pixel error
def boundary_xy(cor4, z):
    """The concatenated pano_connect_points of the 4 walls of one boundary (eval_cuboid.py:109-123)."""
    return np.concatenate([connect(cor4[j], cor4[(j + 1) % 4], z) for j in range(4)], 0)


def _gen_reg(xy):
    """gen_reg_from_xy(xy, 1024) with stable argsorts (both the one by x and np.interp's by x % period)."""
    xy = xy[np.argsort(xy[:, 0], kind='stable')]
    xp = np.asarray(xy[:, 0], np.float64) % W
    fp = np.asarray(xy[:, 1], np.float64)
    order = np.argsort(xp, kind='stable')
    xp, fp = xp[order], fp[order]
    xp = np.concatenate([xp[-1:] - W, xp, xp[0:1] + W])
    fp = np.concatenate([fp[-1:], fp, fp[0:1]])
    return np.interp(np.arange(W), xp, fp)


def infer_coory(y0, h, z0):
    """post_proc.infer_coory (float64 per column)."""
    v0 = -((y0 + 0.5) / H - 0.5) * PI
    c0 = z0 / np.tan(v0)
    v1 = np.arctan2(z0 + h, c0)
    return (-v1 / PI + 0.5) * H - 0.5


def boundaries(dt, z0, z1, gt):
    """[4][1024] float64: the dt ceiling, dt floor (infer_coory), gt ceiling and gt floor rows (eval_cuboid.py:106-127).
    A boundary that no wall samples (np.interp raises ValueError) is NaN: no row to mark."""
    z0, z1 = float(z0), float(z1)

    def gen_reg(xy):
        return _gen_reg(xy) if len(xy) else np.full(W, np.nan)
    y0_dt = gen_reg(boundary_xy(dt[0::2], -z0))
    y1_dt = infer_coory(y0_dt, z1 - z0, z0)
    y0_gt = gen_reg(boundary_xy(gt[0::2], -z0))
    y1_gt = gen_reg(boundary_xy(gt[1::2], z0))
    return np.stack([y0_dt, y1_dt, y0_gt, y1_gt])


def order_dependent(cor4, z):
    """Whether one boundary's rows depend on the sort order the reference leaves unspecified: two points with the same
    x % 1024 and different rows."""
    xy = boundary_xy(cor4, z)
    xp = np.asarray(xy[:, 0], np.float64) % W
    for x in np.unique(xp):
        if len(np.unique(xy[xp == x, 1])) > 1:
            return True
    return False


def pixel_error_count(bon):
    """eval_cuboid.py:129-138: the number of pixels whose label differs; raises IndexError like the reference."""
    cols = np.arange(W)
    surf = []
    for a, b in ((bon[0], bon[1]), (bon[2], bon[3])):
        s = np.zeros((H, W), np.int32)
        with np.errstate(invalid='ignore'):
            s[np.round(a).astype(int), cols] = 1
            s[np.round(b).astype(int), cols] = 1
        surf.append(np.cumsum(s, axis=0))
    return int((surf[0] != surf[1]).sum())


# ---------------------------------------------------------------------------------------------- 3D IoU
def room_xyz(floor, ceil):
    """eval_3diou.py:58-77 for one room: float64 [4][3] floor and ceiling corners (floorW = floorH = 1, ch = -1.6)."""
    u = ((floor[:, 0] + 0.5) / W - 0.5) * 2 * PI
    v = -((floor[:, 1] + 0.5) / H - 0.5) * PI
    c = -1.6 / np.tan(v)
    xy = np.stack([c * np.sin(u) + 0.5 - 0.5, -c * np.cos(u) + 0.5 - 0.5], -1)   # + floorW / 2 - 0.5, in float32
    fl = np.hstack([xy, np.zeros((len(floor), 1)) + -1.6])
    r = np.sqrt((fl[:, :2] ** 2).sum(1))
    v2 = -((ceil[:, 1] + 0.5) / H - 0.5) * PI
    ce = fl.copy()
    ce[:, 2] = r * np.tan(v2)
    return fl, ce


def halfspaces(fl, ce):
    """xyzlst2halfspaces: 6 planes [nx, ny, nz, d] per corner, oriented so that the origin satisfies n.x + d <= 0."""
    def tri(pa, pb, p):
        vn = np.cross(pa - p, pb - p)
        if -vn @ p > 0:
            vn = -vn
        return [*vn, -vn @ p]

    out = []
    n = len(fl)
    for i in range(n):
        a, b = (i - 1 + n) % n, (i + 1) % n
        out += [tri(fl[a], fl[b], fl[i]), tri(fl[a], ce[i], fl[i]), tri(ce[i], fl[b], fl[i]),
                tri(ce[a], ce[b], ce[i]), tri(ce[a], fl[i], ce[i]), tri(fl[i], ce[b], ce[i])]
    return np.array(out)


def box(L):
    """The faces of [-L, L]^3, counter-clockwise seen from outside, labelled 0..5."""
    m, p = -L, L
    faces = [[(p, m, m), (p, p, m), (p, p, p), (p, m, p)], [(m, m, m), (m, m, p), (m, p, p), (m, p, m)],
             [(m, p, m), (m, p, p), (p, p, p), (p, p, m)], [(m, m, m), (p, m, m), (p, m, p), (m, m, p)],
             [(m, m, p), (p, m, p), (p, p, p), (m, p, p)], [(m, m, m), (m, p, m), (p, p, m), (p, m, m)]]
    return [(k, [tuple(float(c) for c in v) for v in f]) for k, f in enumerate(faces)]


def side(h, v):
    return ((h[0] * v[0] + h[1] * v[1]) + h[2] * v[2]) + h[3]


def cut(a, sa, b, sb):
    """The crossing of the plane on edge a-b, from the inside end, so both faces of the edge get the same point."""
    if sa > 0:
        a, sa, b, sb = b, sb, a, sa
    t = sa / (sa - sb)
    return (a[0] + t * (b[0] - a[0]), a[1] + t * (b[1] - a[1]), a[2] + t * (b[2] - a[2]))


def cap_polygon(pts, h):
    """The points on the cutting plane, ordered counter-clockwise about its outward normal (h[:3]), exact duplicates
    dropped."""
    n = (h[0], h[1], h[2])
    ax = min(range(3), key=lambda k: abs(n[k]))
    e = [0.0, 0.0, 0.0]
    e[ax] = 1.0
    e1 = (n[1] * e[2] - n[2] * e[1], n[2] * e[0] - n[0] * e[2], n[0] * e[1] - n[1] * e[0])   # n x e
    e2 = (n[1] * e1[2] - n[2] * e1[1], n[2] * e1[0] - n[0] * e1[2], n[0] * e1[1] - n[1] * e1[0])   # n x e1
    k = len(pts)
    c = [sum(p[j] for p in pts) / k for j in range(3)]
    ang = []
    for p in pts:
        d = (p[0] - c[0], p[1] - c[1], p[2] - c[2])
        ang.append(np.arctan2(d[0] * e2[0] + d[1] * e2[1] + d[2] * e2[2], d[0] * e1[0] + d[1] * e1[1] + d[2] * e1[2]))
    order = sorted(range(k), key=lambda i: (ang[i], i))
    out = []
    for i in order:                      # each point comes from both faces of its edge: keep one
        if not out or pts[i] != out[-1]:
            out.append(pts[i])
    if len(out) > 1 and out[-1] == out[0]:
        out.pop()
    return out


def clip(faces, h, label, eps):
    """Faces of a convex polyhedron cut by the halfspace h . (x, 1) <= 0: each face clipped (Sutherland-Hodgman), the
    new face on the plane added as the cap.  A vertex within eps of the plane counts as on it, so a plane that repeats
    a face (xyzlst2halfspaces gives each wall several times) changes nothing.  A zero normal is a no-op."""
    if h[0] == 0 and h[1] == 0 and h[2] == 0:
        return faces
    tol = eps * np.sqrt(h[0] * h[0] + h[1] * h[1] + h[2] * h[2])
    if all(side(h, v) <= tol for _, f in faces for v in f):
        return faces
    out, cap = [], []
    for lab, f in faces:
        k = len(f)
        s = [side(h, v) for v in f]
        c = [1 if x > tol else (-1 if x < -tol else 0) for x in s]
        keep, on = [], []
        for i in range(k):
            j = (i + 1) % k
            if c[i] <= 0:
                keep.append(f[i])
                if c[i] == 0:
                    on.append(f[i])
            if c[i] * c[j] < 0:
                p = cut(f[i], s[i], f[j], s[j])
                keep.append(p)
                on.append(p)
        if len(keep) >= 3:
            out.append((lab, keep))
        cap += on
    cap = cap_polygon(cap, h) if len(cap) >= 3 else []
    if len(cap) >= 3:
        out.append((label, cap))
    return out


def volume(faces):
    """Volume of a closed, outward-oriented polyhedron: triangle fans around the origin."""
    t = 0.0
    for _, f in faces:
        v0 = f[0]
        for i in range(1, len(f) - 1):
            a, b = f[i], f[i + 1]
            t += v0[0] * (a[1] * b[2] - a[2] * b[1]) + v0[1] * (a[2] * b[0] - a[0] * b[2]) + \
                v0[2] * (a[0] * b[1] - a[1] * b[0])
    return t / 6


def clip_volume(planes, faces, R):
    """Clip `faces` by every plane in order (R: the corners' scale); returns (faces, touches_box)."""
    for i, h in enumerate(planes):
        faces = clip(faces, [float(x) for x in h], 6 + i, ON_PLANE * R)
    return faces, any(lab < 6 for lab, _ in faces)


def room_volume(planes, R):
    """Volume of the intersection of the halfspaces, clipped from a box of BOX_SCALES[0] * R and, while the result
    touches the box, from the next larger one (a small box keeps the vertices precise).  Returns (volume,
    touches_the_largest_box)."""
    for s in BOX_SCALES:
        faces, touch = clip_volume(planes, box(s * R), R)
        if not touch:
            break
    return volume(faces), touch


def scale_of(*pts):
    return float(np.max(np.abs(np.concatenate([np.ravel(p) for p in pts])))) + 1.0


def iou3d(dt, gt):
    """eval_3diou(dt floor, dt ceiling, gt floor, gt ceiling) by clipping; returns (status, IoU x 100)."""
    if (dt[1::2, 0] != dt[0::2, 0]).sum() or (gt[1::2, 0] != gt[0::2, 0]).sum():
        return ERR_COLUMNS, np.nan
    dfl, dce = room_xyz(dt[1::2], dt[0::2])
    gfl, gce = room_xyz(gt[1::2], gt[0::2])
    if not all(np.isfinite(p).all() for p in (dfl, dce, gfl, gce)):
        return ERR_HULL, np.nan
    hd, hg = halfspaces(dfl, dce), halfspaces(gfl, gce)
    if any(h[3] == 0 and (h[0] != 0 or h[1] != 0 or h[2] != 0) for h in np.concatenate([hd, hg])):
        return ERR_HULL, np.nan                      # the origin lies on a plane
    R = scale_of(dfl, dce, gfl, gce)
    v_dt, t_dt = room_volume(hd, R)
    v_gt, t_gt = room_volume(hg, R)
    if t_dt or t_gt:
        return ERR_HULL, np.nan
    v_in, _ = room_volume(np.concatenate([hd, hg]), R)
    if min(v_dt, v_gt, v_in) <= FLAT_VOLUME * R ** 3:
        return ERR_HULL, np.nan
    return OK, 100 * v_in / (v_dt + v_gt - v_in)


# ---------------------------------------------------------------------------------------------- test
def test_cuboid(dt_cor_id, z0, z1, gt_cor_id):
    """One pair in pixels -> dict(status, ce, pe, pe_count, iou3d, bon); metrics NaN where the reference raises."""
    out = dict(status=OK, ce=np.nan, pe=np.nan, pe_count=-1, iou3d=np.nan, bon=None)
    dt, gt = np.asarray(dt_cor_id, np.float32), np.asarray(gt_cor_id, np.float32)
    if dt.shape != (8, 2) or gt.shape != (8, 2):
        out['status'] = ERR_ROWS
        return out
    ce = corner_error(dt, gt)
    with np.errstate(divide='ignore', invalid='ignore'):
        bon = boundaries(dt, z0, z1, gt)
    out['bon'] = bon
    try:
        cnt = pixel_error_count(bon)
    except IndexError:
        out['status'] = ERR_INDEX
        return out
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        st, iou = iou3d(dt, gt)
    if st != OK:
        out['status'] = st
        return out
    out.update(ce=ce, pe=100 * cnt / (H * W), pe_count=cnt, iou3d=iou)
    return out


def dt_pixels(dt_normalised):
    """eval_cuboid.py:192-194: a normalised float32 cor_id scaled to pixels in float32."""
    d = np.array(dt_normalised, np.float32)
    d[:, 0] *= W
    d[:, 1] *= H
    return d
