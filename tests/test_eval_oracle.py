"""No GPU: oracle/eval_general_ref.py against the real reference (tests/golden/eval_general.npz) and, for the polygon
areas shapely would give, against independent computations: scipy's ConvexHull / HalfspaceIntersection for convex
pairs, ear-clipped triangles for non-convex ones, and rectilinear pairs with areas known exactly."""
import os

import numpy as np
import pytest
from scipy.optimize import linprog
from scipy.spatial import ConvexHull, HalfspaceIntersection

from oracle import eval_general_ref as E

G = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'eval_general.npz'))
NAMES = [str(n) for n in G['names']]


def layout(name, side):
    """The reference's records of a pair's dt or gt corner list (stored once per distinct list)."""
    key = str(G['%s/%s_key' % (name, side)])
    return {k.split('/')[-1]: G[k] for k in G.files if k.startswith('layout/%s/' % key)}


@pytest.mark.parametrize('name', NAMES)
def test_oracle_matches_reference(name):
    rec = {side: layout(name, side) for side in ('dt', 'gt')}
    rows, cols = G['depth_rows'], G['columns']
    for side, r in rec.items():
        cor = r['cor']
        if 'bon' in r and not r['order_dependent']:
            np.testing.assert_array_equal(E.cor_2_1d(cor)[:, cols], r['bon'])
        if str(r['depth_exc']):
            with pytest.raises(E.DepthAssertion):
                E.layout_2_depth(cor)
        else:
            d = E.layout_2_depth(cor)[rows][:, cols]
            if r['order_dependent']:
                np.testing.assert_allclose(d, r['depth_rows'], rtol=1e-6)
            else:
                np.testing.assert_array_equal(d, r['depth_rows'])
        if 'z1' in r:
            z = E.heights(cor[1::2, 1], cor[0::2, 1])
            assert z.dtype == r['z1'].dtype
            np.testing.assert_array_equal(z, r['z1'])
    o = E.test_general(rec['dt']['cor'], rec['gt']['cor'])
    if name + '/rmse' in G and o['status'] in (E.OK, E.DT_INVALID):
        assert o['rmse'] == pytest.approx(float(G[name + '/rmse']), rel=1e-6, abs=1e-9)
        assert o['delta_1'] == pytest.approx(float(G[name + '/delta_1']), abs=2 / (512 * 1024))
    if o['status'] == E.ERR_GT_DEPTH:
        assert str(rec['gt']['depth_exc'])


def test_fixture_covers_every_status_and_an_order_dependent_case():
    pairs = [(layout(n, 'dt'), layout(n, 'gt')) for n in NAMES]
    seen = {E.test_general(d['cor'], g['cor'])['status'] for d, g in pairs}
    assert seen == set(E.STATUS_NAMES)
    assert any(bool(d['order_dependent']) for d, _ in pairs)
    assert layout('fallback_vs_room0', 'dt')['cor'].dtype == np.int64


# ---------------------------------------------------------------------------------------------- areas
def _halfspaces(poly):
    """A convex polygon as scipy halfspaces A x + b <= 0 (counter-clockwise vertices)."""
    p = np.asarray(poly, np.float64)
    if E.signed_area(p) < 0:
        p = p[::-1]
    q = np.roll(p, -1, 0)
    n = np.stack([q[:, 1] - p[:, 1], p[:, 0] - q[:, 0]], 1)          # outward normals
    return np.hstack([n, -(n * p).sum(1, keepdims=True)])


def _convex_intersection(a, b):
    """Area of the intersection of two convex polygons: scipy's halfspace intersection around the Chebyshev centre."""
    hs = np.vstack([_halfspaces(a), _halfspaces(b)])
    norm = np.linalg.norm(hs[:, :2], axis=1)
    res = linprog([0, 0, -1], A_ub=np.hstack([hs[:, :2], norm[:, None]]), b_ub=-hs[:, 2],
                  bounds=[(None, None), (None, None), (0, None)])
    if res.status != 0 or res.x[2] < 1e-9:                           # no interior: the intersection has no area
        return 0.0
    return ConvexHull(HalfspaceIntersection(hs, res.x[:2]).intersections).volume


def _ear_clip(poly):
    p = [tuple(v) for v in np.asarray(poly, np.float64)]
    if E.signed_area(p) < 0:
        p = p[::-1]
    tris = []
    while len(p) > 3:
        for i in range(len(p)):
            a, b, c = p[i - 1], p[i], p[(i + 1) % len(p)]
            if (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0]) <= 0:
                continue
            tri = np.array([a, b, c])
            if any(_inside_tri(tri, v) for v in p if v not in (a, b, c)):
                continue
            tris.append(tri)
            del p[i]
            break
    tris.append(np.array(p))
    return tris


def _inside_tri(t, v):
    d = [(t[(k + 1) % 3][0] - t[k][0]) * (v[1] - t[k][1]) - (t[(k + 1) % 3][1] - t[k][1]) * (v[0] - t[k][0])
         for k in range(3)]
    return all(x >= 0 for x in d)


def _regular(n, r, cx, cy, rot):
    a = rot + 2 * np.pi * np.arange(n) / n
    return np.stack([cx + r * np.cos(a), cy + r * np.sin(a)], 1)


@pytest.mark.parametrize('seed', range(6))
def test_convex_areas_against_scipy(seed):
    rs = np.random.RandomState(seed)
    a = _regular(rs.randint(3, 9), rs.uniform(1, 2), 0, 0, rs.uniform(0, 1))
    b = _regular(rs.randint(3, 9), rs.uniform(1, 2), rs.uniform(-1, 1), rs.uniform(-1, 1), rs.uniform(0, 1))
    if seed % 2:
        b = b[::-1]                                                  # clockwise rings too
    assert abs(E.signed_area(a)) == pytest.approx(ConvexHull(a).volume, rel=1e-12)
    assert E.intersection_area(a, b) == pytest.approx(_convex_intersection(a, b), rel=1e-9, abs=1e-12)


@pytest.mark.parametrize('seed', range(4))
def test_nonconvex_areas_against_ear_clipping(seed):
    rs = np.random.RandomState(10 + seed)

    def star(cx, cy):
        n = 2 * rs.randint(4, 7)
        r = np.where(np.arange(n) % 2, rs.uniform(0.4, 0.7), rs.uniform(1.2, 1.6))
        a = rs.uniform(0, 1) + 2 * np.pi * np.arange(n) / n
        return np.stack([cx + r * np.cos(a), cy + r * np.sin(a)], 1)

    a, b = star(0, 0), star(rs.uniform(-0.6, 0.6), rs.uniform(-0.6, 0.6))
    want = sum(_convex_intersection(s, t) for s in _ear_clip(a) for t in _ear_clip(b))
    assert sum(ConvexHull(t).volume for t in _ear_clip(a)) == pytest.approx(abs(E.signed_area(a)), rel=1e-12)
    assert E.intersection_area(a, b) == pytest.approx(want, rel=1e-9)


L_SHAPE = [(0, 0), (4, 0), (4, 2), (2, 2), (2, 4), (0, 4)]


@pytest.mark.parametrize('a, b, want', [
    (L_SHAPE, [(1, 1), (3, 1), (3, 3), (1, 3)], 3.0),               # crossing edges
    (L_SHAPE, [(0, 0), (4, 0), (4, 4), (0, 4)], 12.0),              # collinear edges, same direction
    (L_SHAPE, [(0, 0), (0, 4), (4, 4), (4, 0)], 12.0),              # the same, clockwise
    ([(0, 0), (2, 0), (2, 2), (0, 2)], [(2, 0), (4, 0), (4, 2), (2, 2)], 0.0),   # touching along an edge
    (L_SHAPE, [(2, 2), (4, 2), (4, 4), (2, 4)], 0.0),               # the notch: touching along two edges
    (L_SHAPE, L_SHAPE, 12.0),                                        # identical rings
    ([(0, 0), (6, 0), (6, 1), (0, 1)], [(1, -1), (2, -1), (2, 3), (1, 3)], 1.0),  # a cross
])
def test_rectilinear_areas_exact(a, b, want):
    assert E.intersection_area(np.array(a, float), np.array(b, float)) == want
    assert E.intersection_area(np.array(b, float), np.array(a, float)) == want
