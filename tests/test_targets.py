"""GPU: hn_train_targets (csrc/targets.cu) against tests/golden/dataset_targets.npz (minted from the real reference) and
against oracle/dataset_ref.py on 256 seeded rooms with random stretch, flip and roll.

Bounds (DESIGN.md section 11): statuses and occlusion flags identical, except fixture-marked near-degenerate rooms where
numpy's float32 trigonometry and the device's can round a floor-plane point differently; the flipped and rolled corners
bit for bit; y_cor within 1 float32 ulp; y_bon within 1e-5 rad (the per-corner steps follow numpy's float32 sine, the
device rounds the float64 one), compared only where the reference's order-dependent lists cannot matter."""
import os

import numpy as np
import pytest
import torch

import __graft_entry__ as entry
from horizonnet_b200 import dataset as DS
from horizonnet_b200.augment import augment_corners, draw_params
from oracle import dataset_ref as D
from oracle.eval_general_ref import order_dependent

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'dataset_targets.npz')
BON_TOL = 1e-5


@pytest.fixture(scope='module', autouse=True)
def _built():
    entry.build()


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def _run(cor0s, cors, flip, dx):
    o = DS._launch_targets(cor0s, cors, flip, dx, 0.96, torch.device('cuda', 0))
    return {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in o.items() if k != '_keep'}


def test_targets_match_reference_fixture():
    g = dict(np.load(GOLD))
    n = len(g['status'])
    rows = g['rows']
    o = _run([g['cor0'][i, :rows[i]] for i in range(n)], [g['cor'][i, :rows[i]] for i in range(n)],
             g['flip'].tolist(), g['dx'].tolist())
    np.testing.assert_array_equal(o['status'], g['status'])
    worst_bon, worst_cor = 0.0, 0
    for i in range(n):
        r, name = rows[i], str(g['names'][i])
        if g['status'][i] in (D.ERR_ROWS, D.ERR_CORNERS):
            continue
        if not g['near_degenerate'][i]:
            np.testing.assert_array_equal(o['occlusion'][i, :r].astype(bool), g['occlusion'][i, :r], err_msg=name)
        if g['status'][i] != D.OK:
            assert np.isnan(o['y_bon'][i]).all() and np.isnan(o['y_cor'][i]).all(), name
            continue
        np.testing.assert_array_equal(o['cor'][i, :r], g['cor_out'][i, :r], err_msg=name)
        if (o['occlusion'][i, :r].astype(bool) != g['occlusion'][i, :r]).any():
            continue                                     # a near-degenerate flag flipped: y_cor has another corner set
        worst_cor = max(worst_cor, int(_ulps(o['y_cor'][i, 0, i % 8::8], g['y_cor'][i]).max()))
        if not g['order_dependent'][i]:
            worst_bon = max(worst_bon, float(np.abs(o['y_bon'][i][:, i % 8::8].astype(np.float64) - g['y_bon'][i]).max()))
    print('fixture: worst y_bon %.3g rad, worst y_cor %d ulp' % (worst_bon, worst_cor))
    assert worst_bon <= BON_TOL and worst_cor <= 1


def _seeded(count=256, seed=77):
    rs = np.random.RandomState(seed)
    cases = []
    for k in range(count):
        c0 = D.read_roll(D.synthetic_room(rs, D.ROOM_KINDS[k % len(D.ROOM_KINDS)]))
        p = draw_params(c0, 1024, stretch=k % 4 != 0, flip=True, rotate=k % 3 != 0, gamma=False, rng=rs)
        cs = augment_corners(c0, 512, 1024, p['kx'], p['ky']) if p['kx'] is not None else c0
        cases.append((c0, cs, p['flip'], p['dx'] if k % 3 != 0 else -1))
    return cases


def test_targets_match_oracle_on_seeded_rooms():
    cases = _seeded()
    o = _run(*[list(z) for z in zip(*cases)])
    worst_bon, worst_cor, skipped = 0.0, 0, 0
    for i, (c0, cs, flip, dx) in enumerate(cases):
        ref = D.targets(c0, cs, flip, dx, trig='device')
        r = len(c0)
        degenerate = D.near_degenerate(c0[::2])
        assert o['status'][i] == ref['status'] or degenerate, i
        occ = o['occlusion'][i, :r].astype(bool)
        if not np.array_equal(occ, ref['occlusion']):
            assert degenerate, i
            skipped += 1
            continue
        np.testing.assert_array_equal(o['cor'][i, :r], ref['cor'], err_msg=str(i))
        if ref['status'] != D.OK:
            continue
        worst_cor = max(worst_cor, int(_ulps(o['y_cor'][i], ref['y_cor']).max()))
        if not order_dependent(cs):
            worst_bon = max(worst_bon, float(np.abs(o['y_bon'][i].astype(np.float64) - ref['y_bon']).max()))
    print('256 rooms: worst y_bon %.3g rad, worst y_cor %d ulp, %d near-degenerate rooms skipped' %
          (worst_bon, worst_cor, skipped))
    assert worst_bon <= BON_TOL and worst_cor <= 1
    assert (o['status'] == D.OK).sum() >= 250


@pytest.mark.parametrize('name, status', [('two_corners', D.ERR_CORNERS), ('no_samples', D.ERR_BOUNDARY),
                                          ('all_occluded', D.ERR_OCCLUDED), ('odd_rows', D.ERR_ROWS)])
def test_error_status_raises_and_names_the_sample(name, status):
    g = dict(np.load(GOLD))
    i = list(g['names']).index(name)
    ok = [g['cor0'][0, :g['rows'][0]]]
    c = g['cor0'][i, :g['rows'][i]]
    exc = AssertionError if status == D.ERR_ROWS else ValueError
    with pytest.raises(exc, match='sample 1'):
        DS.train_targets(ok + [c], ok + [c], [False, False], [-1, -1])
    o = _run(ok + [c], ok + [c], [False, False], [-1, -1])
    assert o['status'].tolist() == [D.OK, status]
    assert np.isnan(o['y_bon'][1]).all() and np.isnan(o['y_cor'][1]).all() and np.isfinite(o['y_bon'][0]).all()
