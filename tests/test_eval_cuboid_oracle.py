"""CPU: oracle/eval_cuboid_ref.py against tests/golden/eval_cuboid.npz, minted from the real reference eval_cuboid.py,
and its clipping volume against scipy's HalfspaceIntersection + ConvexHull (what the reference's eval_3diou calls)."""
import os

import numpy as np
import pytest
from scipy.spatial import ConvexHull, HalfspaceIntersection

from oracle import eval_cuboid_ref as C

G = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'eval_cuboid.npz'))
NAMES = [str(n) for n in G['names']]
COLS = G['columns']                        # the columns whose boundary rows the fixture records


def _pair(name):
    return G[name + '/dt'], float(G[name + '/z0']), float(G[name + '/z1']), G[name + '/gt']


@pytest.mark.parametrize('name', NAMES)
def test_oracle_matches_reference(name):
    dt, z0, z1, gt = _pair(name)
    r = C.test_cuboid(dt, z0, z1, gt)
    exc = str(G[name + '/exc'])
    if not exc and r['status'] == C.ERR_HULL and float(G[name + '/iou3d']) < 1e-3:
        assert _far_or_unbounded(dt, gt), name    # qhull closed a region past the largest box (DESIGN.md section 10)
        return
    if exc:
        assert r['status'] != C.OK, name
        want = C.EXCEPTIONS[r['status']]
        assert exc in (want if isinstance(want, tuple) else (want,)), (name, exc, C.STATUS_NAMES[r['status']])
    else:
        assert r['status'] == C.OK, (name, C.STATUS_NAMES[r['status']])
        assert r['ce'] == pytest.approx(float(G[name + '/ce']), rel=1e-6, abs=1e-12)
        if not bool(G[name + '/tie']):        # else numpy's unstable argsort picks between walls that overlap
            assert r['pe_count'] == int(G[name + '/pe_count'])
        assert r['iou3d'] == pytest.approx(float(G[name + '/iou3d']), rel=1e-7, abs=1e-7)
    if name + '/bon_dt' in G.files:
        ref = np.concatenate([G[name + '/bon_dt'], G['gt_bon/' + str(G[name + '/gt_key'])]])
        mine = (r['bon'] if r['bon'] is not None else C.boundaries(dt, z0, z1, gt))[:, COLS]
        ok = np.isfinite(ref)
        if bool(G[name + '/tie']):          # only the columns where one row is sampled, or several equal ones
            ok &= _single_valued(dt, z0, gt)[:, COLS]
        assert (np.isfinite(mine) == np.isfinite(ref))[ok].all()
        np.testing.assert_array_equal(mine[ok], ref[ok])


def _single_valued(dt, z0, gt):
    """[4][1024]: the columns of each boundary whose points all have one row (the dt floor follows the dt ceiling)."""
    out = np.zeros((4, 1024), bool)
    for k, (cor4, z) in enumerate(((dt[0::2], -z0), (gt[0::2], -z0), (gt[1::2], z0))):
        xy = C.boundary_xy(cor4, z)
        xp = np.asarray(xy[:, 0], np.float64) % 1024
        for c in range(1024):
            ys = xy[xp == c, 1]
            out[(0, 2, 3)[k], c] = len(ys) > 0 and len(np.unique(ys)) == 1
    out[1] = out[0]
    return out


def _unbounded(dt=None, planes=None):
    """Whether the intersection of the dt's halfspaces (or of `planes`) has a recession direction (a linear program on
    the unit box)."""
    from scipy.optimize import linprog
    if planes is None:
        planes = C.halfspaces(*C.room_xyz(dt[1::2], dt[0::2]))
    A = planes[:, :3]
    A = A / np.maximum(np.linalg.norm(A, axis=1, keepdims=True), 1e-300)
    for c in np.vstack([np.eye(3), -np.eye(3)]):
        r = linprog(-c, A_ub=A, b_ub=np.zeros(len(A)), bounds=[(-1, 1)] * 3, method='highs')
        if r.status == 0 and -r.fun > 0.5:
            return True
    return False


def _far_or_unbounded(dt, gt):
    """Whether the dt's or the gt's region has a recession direction, or qhull puts one of its vertices past the largest
    starting box (BOX_SCALES[-1] times the rooms' scale)."""
    rooms = [C.room_xyz(c[1::2], c[0::2]) for c in (dt, gt)]
    R = C.scale_of(*[p for room in rooms for p in room])
    for fl, ce in rooms:
        h = C.halfspaces(fl, ce)
        if _unbounded(planes=h):
            return True
        try:
            far = np.abs(HalfspaceIntersection(h, np.zeros(3)).intersections).max()
        except Exception:                                   # noqa: BLE001
            return True
        if far > C.BOX_SCALES[-1] * R:
            return True
    return False


def test_fixture_covers_every_reference_error_and_a_tie():
    excs = {str(G[n + '/exc']) for n in NAMES}
    assert {'', 'ValueError', 'IndexError', 'AssertionError'} <= excs
    assert any(bool(G[n + '/tie']) for n in NAMES)
    assert any(not bool(G[n + '/tie']) and not str(G[n + '/exc']) for n in NAMES)


def test_bowtie_scores_the_intersection_of_all_planes():
    r = C.test_cuboid(*_pair('dt_bowtie'))
    assert r['status'] == C.OK and r['iou3d'] == pytest.approx(float(G['dt_bowtie/iou3d']), rel=1e-7)


def _scipy_volume(planes):
    return ConvexHull(HalfspaceIntersection(planes, np.zeros(3)).intersections).volume


def _random_room(rs, convex):
    """4 corners of a room around the camera in pixels: a jittered rectangle, or a non-convex quadrilateral (one corner
    pulled in past the diagonal)."""
    hx, hy = rs.uniform(1.0, 4.0, 2)
    poly = np.array([(hx, hy), (-hx, hy), (-hx, -hy), (hx, -hy)]) + rs.normal(0, 0.3, (4, 2))
    if not convex:
        k = rs.randint(4)
        poly[k] = 0.3 * poly[k] + 0.7 * poly[(k + 2) % 4] * rs.uniform(0.0, 0.4)
    poly -= rs.uniform(-0.5, 0.5, 2)
    u = np.arctan2(poly[:, 0], -poly[:, 1])
    d = np.hypot(poly[:, 0], poly[:, 1])
    col = (u / (2 * np.pi) + 0.5) * 1024 - 0.5
    hc = 1.4 + rs.normal(0, 0.1, 4)
    cor = np.zeros((8, 2), np.float32)
    order = np.argsort(col)
    cor[0::2, 0] = cor[1::2, 0] = col[order]
    cor[0::2, 1] = ((-np.arctan(hc / d) / np.pi + 0.5) * 512 - 0.5)[order]
    cor[1::2, 1] = ((np.arctan(1.6 / d) / np.pi + 0.5) * 512 - 0.5)[order]
    return cor


@pytest.mark.parametrize('convex', [True, False])
def test_clip_volume_matches_qhull(convex):
    rs = np.random.RandomState(7 if convex else 8)
    checked = 0
    for _ in range(150):
        dt, gt = _random_room(rs, convex), _random_room(rs, True)
        dfl, dce = C.room_xyz(dt[1::2], dt[0::2])
        gfl, gce = C.room_xyz(gt[1::2], gt[0::2])
        hd, hg = C.halfspaces(dfl, dce), C.halfspaces(gfl, gce)
        try:
            want = [_scipy_volume(np.concatenate([hd, hg])), _scipy_volume(hd), _scipy_volume(hg)]
        except Exception:                                   # noqa: BLE001 -- qhull refuses: the oracle must too
            assert C.iou3d(dt, gt)[0] == C.ERR_HULL
            continue
        R = C.scale_of(dfl, dce, gfl, gce)
        (v_in, t_in), (v_dt, t_dt), (v_gt, t_gt) = (C.room_volume(h, R) for h in (np.concatenate([hd, hg]), hd, hg))
        if t_dt or t_gt:                    # a region past the largest box: qhull closed it far away, or by roundoff
            h = hd if t_dt else hg
            far = np.abs(HalfspaceIntersection(h, np.zeros(3)).intersections).max()
            assert _unbounded(planes=h) or far > C.BOX_SCALES[-1] * R
            continue
        assert not t_in
        got = [v_in, v_dt, v_gt]
        rtol = 1e-9 if max(got) < 1e3 * R ** 3 else 1e-6    # far-reaching regions come from a larger, coarser box
        np.testing.assert_allclose(got, want, rtol=rtol, atol=1e-12 * R ** 3)
        checked += 1
    assert checked >= 100
