"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the layout post-processing of reference inference.py:95-141.

From the TTA outputs (pixel-row boundaries y_bon_pix [2][1024] and the corner probability y_cor [1024], float32)
to the corner list the reference writes: ceiling height (misc/post_proc.py np_refine_by_fix_z / mean_percentile),
wall-wall peaks (inference.py find_N_peaks), Manhattan wall fitting (post_proc.gen_ww with get_gpid, np_coor2xy, vote,
gen_ww_cuboid / gen_ww_general, np_xy2coor), the polygon-validity fallback to a cuboid, infer_coory and the packing of
cor_id.  dtypes follow numpy's at every step: float32 up to z1 and tol, float64 from the floor-plane projection on
(hstack with an int64 arange promotes), float32 cor_id.

Two rules the reference leaves open are fixed here and in csrc/layout.cu alike (DESIGN.md section 8):
  * top-N peaks: ties in value go to the lower column (the reference's argsort leaves their order unspecified);
  * polygon validity (the reference asks shapely's Polygon.is_valid): see ``is_simple_ring``.

Pinned by tests/golden/layout.npz (minted from the real reference by tests/golden/make_golden_layout.py)."""
import numpy as np

PI = float(np.pi)
W, H = 1024, 512
Z0 = 50

# status codes of hn_layout_postproc (include/horizonnet_b200.h)
OK, FALLBACK, ERR_GROUPS, ERR_VOTE, ERR_RING, ERR_OVERFLOW = 0, 1, 2, 3, 4, 5
STATUS_NAMES = {OK: 'ok', FALLBACK: 'fallback', ERR_GROUPS: 'groups', ERR_VOTE: 'vote', ERR_RING: 'ring',
                ERR_OVERFLOW: 'overflow'}


class LayoutError(Exception):
    """Raised by the fitting steps where the reference raises; ``status`` says which."""

    def __init__(self, status, msg):
        super().__init__(msg)
        self.status = status


# ---------------------------------------------------------------------------------------------- ceiling height
def refine_z1(y_bon_pix):
    """z1 of np_refine_by_fix_z(ceiling rows, floor rows, z0=50), all float32."""
    ceil = np.asarray(y_bon_pix[0], np.float32)
    floor = np.asarray(y_bon_pix[1], np.float32)
    v0 = -((ceil + 0.5) / H - 0.5) * PI
    v1 = -((floor + 0.5) / H - 0.5) * PI
    z1 = (Z0 / np.tan(v0)) * np.tan(v1)
    lo, hi = np.percentile(z1, 25), np.percentile(z1, 75)        # numpy's linear interpolation
    return z1[(lo <= z1) & (z1 <= hi)].mean()


def wall_tol(z1):
    return abs(0.16 * z1 / 1.6)                                    # float32, like the reference


# ---------------------------------------------------------------------------------------------- peaks
def find_peaks(sig, r_px, min_v, n=None):
    """Columns equal to the wrap-mode maximum over a window of r_px columns (offsets -(r_px//2) .. r_px-1-r_px//2, as
    scipy places an even window), above min_v; with n, the n largest by value (ties: lower column) in column order."""
    sig = np.asarray(sig, np.float32)
    lo = -(r_px // 2)
    idx = (np.arange(W)[:, None] + np.arange(lo, lo + r_px)[None, :]) % W
    peak = np.where(sig[idx].max(1) == sig)[0]
    peak = peak[sig[peak] > np.float32(min_v)]
    if n is not None:
        order = np.argsort(-sig[peak], kind='stable')
        peak = np.sort(peak[order[:n]])
    return peak


# ---------------------------------------------------------------------------------------------- geometry (float64)
def col_to_u(x):
    return ((x + 0.5) / W - 0.5) * 2 * PI


def row_to_v(y):
    return -((y + 0.5) / H - 0.5) * PI


def floor_xy(ceil_rows):
    """Every column's ceiling boundary projected on the plane z = 50: [1024][2] float64."""
    u = col_to_u(np.arange(W).astype(np.float64))
    c = Z0 / np.tan(row_to_v(np.asarray(ceil_rows, np.float32).astype(np.float64)))
    return np.stack([c * np.sin(u) + W / 2 - 0.5, -c * np.cos(u) + H / 2 - 0.5], 1)


def xy_to_coor(xy):
    x = xy[:, 0] - W / 2 + 0.5
    y = xy[:, 1] - H / 2 + 0.5
    u = np.arctan2(x, -y)
    v = np.arctan(Z0 / np.sqrt(x ** 2 + y ** 2))
    return np.stack([(u / (2 * PI) + 0.5) * W - 0.5, (-v / PI + 0.5) * H - 0.5], 1)


def y_from_x(x, u):
    """The y where the line x = const meets the ray of column angle u."""
    c = (x - W / 2 + 0.5) / np.sin(u)
    return -c * np.cos(u) + H / 2 - 0.5


def x_from_y(y, u):
    c = -(y - H / 2 + 0.5) / np.cos(u)
    return c * np.sin(u) + W / 2 - 0.5


def group_ids(peaks):
    """Column -> wall group: group j >= 1 spans [peak j-1, peak j), group 0 the wrap-around rest."""
    g = np.zeros(W, np.int64)
    g[np.asarray(peaks, np.int64)] = 1
    g = np.cumsum(g)
    g[g == g[-1]] = 0
    return g


# ---------------------------------------------------------------------------------------------- vote
def vote(vals, tol):
    """Best constant for one wall coordinate: the longest run of the sorted values spanning at most tol (by the pair
    distance + 1e-9) that covers at least 40 % of them, the first such run on ties; the median when there is none or
    when there are fewer values than tol.  Returns (fit, run fraction, mean |vals - fit|)."""
    s = np.sort(vals)
    m = len(s)
    i = np.arange(m)
    span = (i[None, :] - i[:, None] + 1).astype(np.float64)      # row i, column j: j - i + 1
    dist = np.abs(s[:, None] - s[None, :])
    dist[~np.eye(m, dtype=bool)] += 1e-9
    ok = (span >= m * 0.4) & (dist <= tol)
    if not ok.any() or m < tol:
        fit, frac = np.median(s), 0
    else:
        k = int(np.where(ok, span, -1.0).argmax())
        r, c = divmod(k, m)
        if not c > r:
            raise LayoutError(ERR_VOTE, 'vote: the best run is a single value')
        fit, frac = s[r:c + 1].mean(), (c - r + 1) / m
    return fit, frac, np.abs(s - fit).mean()


def _pick(xy, sel, tol):
    fx, sx, lx = vote(xy[sel, 0], tol)
    fy, sy, ly = vote(xy[sel, 1], tol)
    return (0, fx, sx) if (sx, -lx) > (sy, -ly) else (1, fy, sy)


# ---------------------------------------------------------------------------------------------- wall fitting
def walls_cuboid(xy, gid, tol):
    if len(np.unique(gid)) != 4:
        raise LayoutError(ERR_GROUPS, 'cuboid fit needs 4 wall groups, got %d' % len(np.unique(gid)))
    walls = [list(_pick(xy, gid == j, tol)) for j in range(4)]
    bal = [0, 0]
    for j, (axis, _, score) in enumerate(walls):
        bal[j % 2] += score if axis == 0 else -score
    first = 0 if bal[0] > bal[1] else 1
    for j in range(4):
        walls[j][0] = first ^ (j & 1)
    return [dict(axis=a, val=v, group=j) for j, (a, v, _) in enumerate(walls)]


def walls_general(peaks, xy, gid, tol):
    n = len(peaks)
    if n != len(np.unique(gid)):
        raise LayoutError(ERR_GROUPS, '%d peaks but %d wall groups' % (n, len(np.unique(gid))))
    walls = []
    for j in range(n):
        axis, val, score = _pick(xy, gid == j, tol)
        walls.append(dict(axis=axis, val=val, score=score, pending=True, group=j,
                          u0=col_to_u(peaks[(j - 1 + n) % n]), u1=col_to_u(peaks[j])))

    def forced(axis, val):
        return dict(axis=axis, val=val, score=0, pending=False, group=-1, u0=-1, u1=-1)

    def across(w, u):                   # the other coordinate where wall w meets the ray at angle u
        return (1, y_from_x(w['val'], u)) if w['axis'] == 0 else (0, x_from_y(w['val'], u))

    while True:
        cur = -1                         # highest-scoring undecided wall, the first one on ties
        for i, w in enumerate(walls):
            if w['pending'] and (cur == -1 or w['score'] > walls[cur]['score']):
                cur = i
        if cur == -1:
            break
        w = walls[cur]
        w['pending'] = False
        p, q = (cur - 1) % len(walls), (cur + 1) % len(walls)
        wp, wq = walls[p], walls[q]
        undecided = int(wp['pending']) + int(wq['pending'])
        if undecided == 2:
            continue
        if undecided == 1:
            if (not wp['pending'] and wp['axis'] == w['axis']) or (not wq['pending'] and wq['axis'] == w['axis']):
                if w['score'] >= -1:     # decide it later, after its other neighbour
                    w['pending'] = True
                    w['score'] -= 100
                elif not wp['pending']:
                    walls.insert(cur, forced(*across(wp, wp['u1'])))
                else:
                    walls.insert(q, forced(*across(wq, wq['u0'])))
            continue
        if wp['axis'] == wq['axis']:
            if w['axis'] == wp['axis']:  # three parallel walls in a row: turn the middle one
                w['axis'] ^= 1
                w['val'] = xy[gid == w['group'], w['axis']].mean()
        else:                            # neighbours already turn: replace this wall by the two implied by them
            if wp['axis'] == 0:
                v0, v1 = y_from_x(wp['val'], wp['u1']), x_from_y(wq['val'], wq['u0'])
            else:
                v0, v1 = x_from_y(wp['val'], wp['u1']), y_from_x(wq['val'], wq['u0'])
            walls[cur:cur + 1] = [forced(wq['axis'], v0), forced(wp['axis'], v1)]
    return walls


def wall_corners(walls):
    """Ceiling corners [n][2] (column, row) float64, rolled so the even row with the smallest column comes first."""
    n = len(walls)
    xy = np.zeros((n, 2))
    for j, w in enumerate(walls):
        nxt = walls[(j + 1) % n]
        xy[j] = (nxt['val'], w['val']) if w['axis'] == 1 else (w['val'], nxt['val'])
    cor = xy_to_coor(xy)
    return np.roll(cor, -2 * int(cor[::2, 0].argmin()), axis=0)


def polygon_xy(walls):
    """The floor polygon the reference checks (inference.py:115-119), float32 [n][2]."""
    out = np.zeros((len(walls), 2), np.float32)
    for i in range(len(walls)):
        out[i, walls[i]['axis']] = walls[i]['val']
        out[i, walls[i - 1]['axis']] = walls[i - 1]['val']
    return out


# ---------------------------------------------------------------------------------------------- validity
def _orient(a, b, c):
    return (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])


def _on_box(a, b, c):
    return min(a[0], b[0]) <= c[0] <= max(a[0], b[0]) and min(a[1], b[1]) <= c[1] <= max(a[1], b[1])


def _segments_meet(a, b, c, d):
    o1, o2, o3, o4 = _orient(a, b, c), _orient(a, b, d), _orient(c, d, a), _orient(c, d, b)
    if ((o1 > 0 and o2 < 0) or (o1 < 0 and o2 > 0)) and ((o3 > 0 and o4 < 0) or (o3 < 0 and o4 > 0)):
        return True
    return ((o1 == 0 and _on_box(a, b, c)) or (o2 == 0 and _on_box(a, b, d)) or
            (o3 == 0 and _on_box(c, d, a)) or (o4 == 0 and _on_box(c, d, b)))


def is_simple_ring(pts):
    """Validity of the closed ring through pts (float32 [n][2], evaluated in float64 without fused multiply-adds):
    after dropping consecutive repeated vertices (cyclically) at least 3 remain, no vertex folds its two edges back
    over each other (collinear with opposite directions), and no two non-adjacent edges intersect or touch."""
    p = [(float(x), float(y)) for x, y in np.asarray(pts, np.float32)]
    q = [v for i, v in enumerate(p) if v != p[i - 1]] if len(set(p)) > 1 else p[:1]
    n = len(q)
    if n < 3:
        return False
    for i in range(n):
        a, b, c = q[i - 1], q[i], q[(i + 1) % n]
        d1, d2 = (b[0] - a[0], b[1] - a[1]), (c[0] - b[0], c[1] - b[1])
        if d1[0] * d2[1] - d1[1] * d2[0] == 0 and d1[0] * d2[0] + d1[1] * d2[1] < 0:
            return False
    for i in range(n):
        for j in range(i + 2, n):
            if i == 0 and j == n - 1:
                continue
            if _segments_meet(q[i], q[(i + 1) % n], q[j], q[(j + 1) % n]):
                return False
    return True


# ---------------------------------------------------------------------------------------------- output
def pack(cor, z1):
    """infer_coory for the floor rows and the [2n][2] float32 cor_id, normalised by W and H."""
    h = np.float32(z1 - Z0)
    zz = np.float32(Z0 + h)
    c0 = Z0 / np.tan(row_to_v(cor[:, 1]))
    floor = (-np.arctan2(zz, c0) / PI + 0.5) * H - 0.5
    out = np.zeros((2 * len(cor), 2), np.float32)
    out[0::2, 0] = cor[:, 0]
    out[0::2, 1] = cor[:, 1]
    out[1::2, 0] = cor[:, 0]
    out[1::2, 1] = floor
    out[:, 0] /= W
    out[:, 1] /= H
    return out


def fit(y_bon_pix, y_cor, z1, r_px, min_v, force_cuboid):
    """gen_ww on the peaks: returns a dict of peaks, group ids, walls and ceiling corners, or raises LayoutError."""
    tol = wall_tol(z1)
    peaks = find_peaks(y_cor, r_px, min_v, 4 if force_cuboid else None)
    gid = group_ids(peaks)
    xy = floor_xy(y_bon_pix[0])
    walls = (walls_cuboid if force_cuboid else lambda x, g, t: walls_general(peaks, x, g, t))(xy, gid, tol)
    return dict(peaks=peaks, gid=gid, walls=walls, cor=wall_corners(walls))


def post_process(y_bon_pix, y_cor, r_px=26, min_v=None, force_cuboid=False, force_raw=False, max_rows=2048):
    """One panorama: returns dict(status, cor_id [2n][2] float32 or None, z1 float32, peaks, and the fits made)."""
    y_bon_pix = np.asarray(y_bon_pix, np.float32)
    z1 = refine_z1(y_bon_pix)
    out = dict(status=OK, z1=z1, cor_id=None, peaks=None, fallback=False)
    try:
        if force_raw:
            cor = np.stack([np.arange(W).astype(np.float64), y_bon_pix[0].astype(np.float64)], 1)
        else:
            if min_v is None:
                min_v = 0 if force_cuboid else 0.05
            f = fit(y_bon_pix, y_cor, z1, r_px, min_v, force_cuboid)
            out.update(peaks=f['peaks'], first=f)
            cor = f['cor']
            if not force_cuboid:
                ring = polygon_xy(f['walls'])
                out['xy2d'] = ring
                if len(ring) < 3:
                    raise LayoutError(ERR_RING, 'the general layout has %d walls: not a polygon' % len(ring))
                if not is_simple_ring(ring):
                    out['fallback'] = True
                    f2 = fit(y_bon_pix, y_cor, z1, r_px, 0, True)
                    out.update(peaks=f2['peaks'], second=f2)
                    cor = f2['cor']
        if 2 * len(cor) > max_rows:
            raise LayoutError(ERR_OVERFLOW, '%d corners do not fit in %d rows' % (len(cor), max_rows))
    except LayoutError as e:
        out['status'] = e.status
        out['error'] = str(e)
        return out
    out['status'] = FALLBACK if out['fallback'] else OK
    out['cor_id'] = pack(cor, z1)
    return out
