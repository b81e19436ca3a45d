"""CPU: pin oracle/layout_ref.py (the numpy restatement of reference inference.py:95-141) against tests/golden/layout.npz,
minted from the real reference by tests/golden/make_golden_layout.py.

Exact on peaks, group ids, wall axes, corner counts and exception kinds; 1e-9 relative on the float64 walls and
corners; one float32 ulp on z1.  The reference's top-4 peak order is unspecified inside a run of equal values
(numpy argsort); where the fixture marks such a tie, the reference's pick must hold the same values as the oracle's,
which follows the documented lower-column rule.  The validity verdict (shapely in the reference) is pinned by
hand-built polygons."""
import os

import numpy as np
import pytest

from oracle import layout_ref as L

G = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'layout.npz'))
NAMES = [str(n) for n in G['names']]
R_PX = int(G['r_px'])
EXC = {L.ERR_GROUPS: 'groups', L.ERR_VOTE: 'vote'}


def _g(name, key):
    return G[name + '/' + key]


@pytest.mark.parametrize('name', NAMES)
def test_z1_within_one_ulp(name):
    z1 = L.refine_z1(_g(name, 'y_bon'))
    want = _g(name, 'z1')
    assert z1.dtype == np.float32
    assert abs(float(z1) - float(want)) <= float(np.spacing(np.abs(want)))


@pytest.mark.parametrize('mode', ['gen', 'cub'])
@pytest.mark.parametrize('name', NAMES)
def test_fit_matches_reference(name, mode):
    yb, yc = _g(name, 'y_bon'), _g(name, 'y_cor')
    z1 = _g(name, 'z1')
    cub = mode == 'cub'
    min_v = 0 if cub else 0.05
    peaks = L.find_peaks(yc, R_PX, min_v, 4 if cub else None)
    want = _g(name, mode + '_peaks')
    tie = cub and bool(_g(name, 'cub_tie'))
    if tie:
        assert np.array_equal(np.sort(yc[peaks]), np.sort(yc[want]))
        top = np.sort(yc[peaks])[0]
        cand = L.find_peaks(yc, R_PX, min_v)
        tied = cand[yc[cand] == top]
        assert np.array_equal(np.intersect1d(peaks, tied), tied[:np.sum(yc[peaks] == top)])   # lowest columns win
        return
    assert np.array_equal(peaks, want)
    assert np.array_equal(L.group_ids(peaks), _g(name, mode + '_gid'))
    try:
        f = L.fit(yb, yc, z1, R_PX, min_v, cub)
    except L.LayoutError as e:
        assert EXC[e.status] == str(_g(name, mode + '_exc'))
        return
    assert str(_g(name, mode + '_exc')) == ''
    axis = np.array([w['axis'] for w in f['walls']])
    val = np.array([w['val'] for w in f['walls']])
    group = np.array([w['group'] for w in f['walls']])
    assert np.array_equal(axis, _g(name, mode + '_axis'))
    assert np.array_equal(group, _g(name, mode + '_group'))
    np.testing.assert_allclose(val, _g(name, mode + '_val'), rtol=1e-9, atol=0)
    assert f['cor'].shape == _g(name, mode + '_cor').shape
    np.testing.assert_allclose(f['cor'], _g(name, mode + '_cor'), rtol=1e-9, atol=0)
    cid = L.pack(f['cor'], z1)
    np.testing.assert_allclose(cid, _g(name, mode + '_cor_id'), rtol=1e-6, atol=0)
    if not cub:
        assert np.array_equal(L.polygon_xy(f['walls']), _g(name, 'gen_xy2d'))


@pytest.mark.parametrize('name', NAMES[:4] + ['plateau'])
def test_raw_mode_matches_reference(name):
    out = L.post_process(_g(name, 'y_bon'), _g(name, 'y_cor'), R_PX, force_raw=True)
    assert out['status'] == L.OK and out['cor_id'].shape == (2048, 2)
    np.testing.assert_allclose(out['cor_id'], _g(name, 'raw_cor_id'), rtol=1e-6, atol=0)


def test_fixture_covers_every_branch():
    kinds = {str(_g(n, 'gen_exc')) for n in NAMES}
    assert {'', 'groups', 'vote'} <= kinds
    statuses = {L.post_process(_g(n, 'y_bon'), _g(n, 'y_cor'), R_PX)['status'] for n in NAMES if n != 'plateau'}
    assert {L.OK, L.FALLBACK, L.ERR_RING, L.ERR_GROUPS, L.ERR_VOTE} <= statuses
    assert any(bool(_g(n, 'cub_tie')) for n in NAMES)


VALID = {
    'square': [(0, 0), (1, 0), (1, 1), (0, 1)],
    'clockwise L': [(0, 0), (0, 2), (1, 2), (1, 1), (2, 1), (2, 0)],
    'repeated vertex dropped': [(0, 0), (1, 0), (1, 0), (1, 1), (0, 1)],
    'straight continuation': [(0, 0), (1, 0), (2, 0), (2, 1), (0, 1)],
    'triangle': [(0, 0), (3, 0), (0, 2)],
}
INVALID = {
    'bow tie': [(0, 0), (1, 1), (1, 0), (0, 1)],
    'two distinct vertices': [(0, 0), (1, 0), (1, 0)],
    'all equal': [(1, 1), (1, 1), (1, 1)],
    'flat triangle': [(0, 0), (2, 0), (1, 0)],
    'fold back': [(0, 0), (2, 0), (1, 0), (1, 1)],
    'vertex touches an edge': [(0, 0), (2, 0), (2, 2), (1, 0), (0, 2)],
    'figure eight at a shared vertex': [(0, 0), (1, 1), (2, 0), (2, 2), (1, 1), (0, 2)],
    'collinear overlap of non-adjacent edges': [(0, 0), (3, 0), (3, 1), (2, 1), (2, 0), (1, 0), (1, -1), (0, -1)],
}


@pytest.mark.parametrize('name', list(VALID))
def test_valid_polygons(name):
    assert L.is_simple_ring(np.array(VALID[name], np.float32))


@pytest.mark.parametrize('name', list(INVALID))
def test_invalid_polygons(name):
    assert not L.is_simple_ring(np.array(INVALID[name], np.float32))


def test_top_n_ties_go_to_the_lower_column():
    sig = np.full(1024, 0.01, np.float32)
    sig[[50, 300, 700]] = 0.9
    assert np.array_equal(L.find_peaks(sig, 26, 0, 4), [0, 50, 300, 700])
    sig[:] = 1.0
    assert np.array_equal(L.find_peaks(sig, 26, 0, 4), [0, 1, 2, 3])


def test_even_window_is_asymmetric():
    sig = np.zeros(1024, np.float32)
    sig[500] = 0.5
    sig[513] = 0.6                  # 13 columns right of 500: outside its window (offsets -13 .. +12)
    sig[487] = 0.55                 # 13 columns left: inside
    assert 500 not in L.find_peaks(sig, 26, 0.05)
    sig[487] = 0.0
    assert 500 in L.find_peaks(sig, 26, 0.05)
