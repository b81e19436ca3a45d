"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the label path of reference dataset.py (PanoCorBonDataset.__getitem__
:56-67, 84-120 with cor_2_1d and find_occlusion): the y_bon / y_cor training targets of one sample.

``targets(cor0, cor, flip, dx)`` takes the corners as read (rolled, float32 pixels) and the same corners after the stretch,
and returns the status, y_bon [2][1024] and y_cor [1][1024] float32, the flipped and rolled corners and the occlusion
flags.  dtypes follow numpy's at every step: the corners are float32, so the per-corner steps run in float32 and the
per-column ones in float64.

Where the reference leaves the result to shapely, the rule is fixed here and in csrc/targets.cu alike (DESIGN.md
section 11): ``LineString.intersects`` is an exact predicate on the float32 floor-plane points (closed segments,
touching counts), decided with rational arithmetic.  cor_2_1d is eval_general_ref's (stable sorts, DESIGN.md section 9).

Pinned by tests/golden/dataset_targets.npz (minted from the real reference by tests/golden/make_golden_dataset.py)."""
from fractions import Fraction

import numpy as np

from oracle.eval_general_ref import boundary_points, cor_2_1d

W, H = 1024, 512

# status codes of hn_train_targets (include/horizonnet_b200.h)
OK, ERR_ROWS, ERR_CORNERS, ERR_BOUNDARY, ERR_OCCLUDED = 0, 1, 2, 3, 4
STATUS_NAMES = {OK: 'ok', ERR_ROWS: 'rows', ERR_CORNERS: 'corners', ERR_BOUNDARY: 'boundary', ERR_OCCLUDED: 'occluded'}


# ---------------------------------------------------------------------------------------------- exact segments
def orient(a, b, c):
    """Sign of (b - a) x (c - a), exactly."""
    ax, ay, bx, by, cx, cy = (Fraction(float(v)) for v in (*a, *b, *c))
    d = (bx - ax) * (cy - ay) - (by - ay) * (cx - ax)
    return (d > 0) - (d < 0)


def _in_box(a, b, c):
    return min(a[0], b[0]) <= c[0] <= max(a[0], b[0]) and min(a[1], b[1]) <= c[1] <= max(a[1], b[1])


def segments_meet(p1, p2, q1, q2):
    """Whether the closed segments p1-p2 and q1-q2 share a point (GEOS intersects: touching counts)."""
    d1, d2 = orient(q1, q2, p1), orient(q1, q2, p2)
    d3, d4 = orient(p1, p2, q1), orient(p1, p2, q2)
    if d1 * d2 < 0 and d3 * d4 < 0:
        return True
    return ((d1 == 0 and _in_box(q1, q2, p1)) or (d2 == 0 and _in_box(q1, q2, p2)) or
            (d3 == 0 and _in_box(p1, p2, q1)) or (d4 == 0 and _in_box(p1, p2, q2)))


class LineString:
    """The part of shapely.geometry.LineString that find_occlusion uses, exact: a polyline of >= 2 points (or none)."""

    def __init__(self, pts):
        self.pts = [(float(x), float(y)) for x, y in pts]
        if len(self.pts) == 1:
            raise ValueError('LineStrings must have at least 2 coordinate tuples')

    def intersects(self, other):
        return any(segments_meet(self.pts[i], self.pts[i + 1], other.pts[j], other.pts[j + 1])
                   for i in range(len(self.pts) - 1) for j in range(len(other.pts) - 1))


# ---------------------------------------------------------------------------------------------- occlusion
def _f32_trig(f, v):
    """The device's float32 transcendentals: the float64 result, rounded."""
    return f(v.astype(np.float64)).astype(np.float32)


def floor_plane(coor, trig='numpy'):
    """coorx2u, coory2v, uv2xy(z=-50) of float32 corners, in float32.  trig='numpy': numpy's float32 sin / cos / tan
    (the reference's), 'device': the float64 results rounded (csrc/pano_connect.cuh)."""
    coor = np.asarray(coor, np.float32)
    u = ((coor[:, 0] + 0.5) / W - 0.5) * 2 * np.pi
    v = ((coor[:, 1] + 0.5) / H - 0.5) * np.pi
    if trig == 'numpy':
        c = -50 / np.tan(v)
        return c * np.cos(u), c * np.sin(u)
    c = -50 / _f32_trig(np.tan, v)
    return c * _f32_trig(np.cos, u), c * _f32_trig(np.sin, u)


def find_occlusion(coor, trig='numpy'):
    """dataset.py:172-186 with the exact LineString."""
    x, y = floor_plane(coor, trig)
    occ = []
    for i in range(len(x)):
        ray = LineString([(0, 0), (x[i], y[i])])
        others = [(x[j], y[j]) for j in range(i + 1, len(x))] + [(x[j], y[j]) for j in range(0, i)]
        occ.append(ray.intersects(LineString(others)))
    return np.array(occ, bool)


def near_degenerate(coor, rel=2.0 ** -20):
    """Whether an orientation find_occlusion decides is within a few float32 ulps of zero, or numpy's float32
    trigonometry and the device's give different flags: there the flag follows the last bit of a sine."""
    if (find_occlusion(coor, 'numpy') != find_occlusion(coor, 'device')).any():
        return True
    x, y = floor_plane(coor)
    n = len(x)
    pts = list(zip(x.astype(np.float64), y.astype(np.float64)))
    for i in range(n):
        for k in range(n - 2):
            a, b = pts[(i + 1 + k) % n], pts[(i + 2 + k) % n]
            for p1, p2, q in (((0.0, 0.0), pts[i], a), ((0.0, 0.0), pts[i], b), (a, b, (0.0, 0.0)), (a, b, pts[i])):
                d = (p2[0] - p1[0]) * (q[1] - p1[1]) - (p2[1] - p1[1]) * (q[0] - p1[0])
                scale = (abs(p2[0] - p1[0]) + abs(p2[1] - p1[1])) * (abs(q[0] - p1[0]) + abs(q[1] - p1[1]))
                if d != 0 and abs(d) <= rel * scale:
                    return True
    return False


# ---------------------------------------------------------------------------------------------- targets
def flip_roll_corners(cor, flip, dx):
    """dataset.py:91, 98 in float32; dx < 0: no roll."""
    c = np.array(cor, np.float32, copy=True)
    if flip:
        c[:, 0] = W - 1 - c[:, 0]
    if dx >= 0:
        c[:, 0] = (c[:, 0] + int(dx)) % W
    return c


def flip_roll_bon(bon, flip, dx):
    """dataset.py:90, 97: np.flip, then np.roll of the finished [2][W] array."""
    if flip:
        bon = np.flip(bon, axis=1)
    if dx >= 0:
        bon = np.roll(bon, int(dx), axis=1)
    return bon


def y_cor_of(corx, p_base=0.96):
    """dataset.py:107-120: p_base ** the circular L1 distance of every column to the nearest of corx, float32 [1][W]."""
    corx = np.asarray(corx, np.float64).reshape(-1, 1)
    cols = np.arange(W, dtype=np.float64).reshape(1, -1)
    dist = np.min([np.abs(corx - cols), np.abs(corx - (cols + W)), np.abs(corx - (cols - W))], 0)
    return (p_base ** dist.min(0)).reshape(1, -1).astype(np.float32)


def targets(cor0, cor, flip, dx, p_base=0.96, trig='numpy'):
    """One sample -> dict(status, y_bon [2][W] float32, y_cor [1][W] float32, cor [rows][2] float32, occlusion [rows]
    bool); y_bon / y_cor NaN where the status is not OK, cor / occlusion None where the rows are refused."""
    cor0, cor = np.asarray(cor0, np.float32), np.asarray(cor, np.float32)
    nan = dict(y_bon=np.full((2, W), np.nan, np.float32), y_cor=np.full((1, W), np.nan, np.float32))
    rows = len(cor0)
    if rows == 0 or rows % 2 or len(cor) != rows:
        return dict(status=ERR_ROWS, cor=None, occlusion=None, **nan)
    if rows < 6:
        return dict(status=ERR_CORNERS, cor=None, occlusion=None, **nan)
    occ = find_occlusion(cor0[::2], trig).repeat(2)
    c = flip_roll_corners(cor, flip, dx)
    out = dict(cor=c, occlusion=occ)
    if any(len(boundary_points(cor, f)[0]) == 0 for f in (False, True)):
        return dict(status=ERR_BOUNDARY, **out, **nan)
    if occ.all():
        return dict(status=ERR_OCCLUDED, **out, **nan)
    bon = flip_roll_bon(cor_2_1d(cor), flip, dx)
    return dict(status=OK, y_bon=bon.astype(np.float32), y_cor=y_cor_of(c[~occ, 0], p_base), **out)


# ---------------------------------------------------------------------------------------------- synthetic rooms
ROOM_KINDS = ('cuboid', 'l_shape', 'notch', 'edge_on')


def _polygon(rs, kind):
    """A floor plan around the camera at the origin, counter-clockwise (x right, y forward)."""
    a, b, c, d = rs.uniform(1.0, 5.0, 4)
    if kind == 'cuboid':
        return [(-a, -c), (b, -c), (b, d), (-a, d)]
    if kind == 'l_shape':                              # the corner beyond (f, e) cut away
        f, e = rs.uniform(0.3, 0.9) * b, rs.uniform(0.3, 0.9) * d
        return [(-a, -c), (b, -c), (b, e), (f, e), (f, d), (-a, d)]
    # a rectangular bump into the room from the back wall: its outer corners hide behind its sides
    g1 = rs.uniform(-0.9 * a, 0.5 * b)
    g2 = rs.uniform(g1 + 0.2, b * 0.95) if g1 + 0.2 < b * 0.95 else b * 0.97
    h = rs.uniform(0.2, 0.8) * c
    return [(-a, -c), (g1, -c), (g1, -c + h), (g2, -c + h), (g2, -c), (b, -c), (b, d), (-a, d)]


def synthetic_room(rs, kind):
    """Label corners of a synthetic room, as a label_cor file holds them: float32 [2n][2] integer pixels, ceiling / floor
    rows alternating, camera 1.6 above the floor and 0.5 to 1.5 below the ceiling.  'edge_on' is a notched room whose
    bump side runs along a camera ray: two corners share a column, so their occlusion is decided by float32 rounding."""
    poly = _polygon(rs, 'notch' if kind == 'edge_on' else kind)
    hc = rs.uniform(0.5, 1.5)
    rows = []
    for x, y in poly:
        dist = np.hypot(x, y)
        u = np.arctan2(y, x)
        px = (u / (2 * np.pi) + 0.5) * W - 0.5
        vc, vf = -np.arctan(hc / dist), np.arctan(1.6 / dist)
        rows.append((round(px) % W, round((vc / np.pi + 0.5) * H - 0.5)))
        rows.append((round(px) % W, round((vf / np.pi + 0.5) * H - 0.5)))
    cor = np.array(rows, np.float32)
    if kind == 'edge_on':                              # the bump's outer corner g1 in the column of its inner corner
        cor[2:4, 0] = cor[4, 0]
    return cor


def read_roll(cor):
    """dataset.py:62: the ceiling corner with the smallest x first."""
    cor = np.asarray(cor, np.float32)
    return np.roll(cor[:, :2], -2 * np.argmin(cor[::2, 0]), 0)
