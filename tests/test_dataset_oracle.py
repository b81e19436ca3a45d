"""No GPU: oracle/dataset_ref.py (the label path of dataset.PanoCorBonDataset) against tests/golden/dataset_targets.npz,
minted from the real reference; its exact LineString on hand-made cases; horizonnet_b200.dataset.read_corners against
dataset.py:57-67; the training CLI's learning-rate schedule against misc.utils.adjust_learning_rate."""
import os
import types

import numpy as np
import pytest

from oracle import dataset_ref as D

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'dataset_targets.npz')


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLD))


def test_oracle_reproduces_the_reference(gold):
    n = len(gold['status'])
    for i in range(n):
        r = int(gold['rows'][i])
        o = D.targets(gold['cor0'][i, :r], gold['cor'][i, :r], int(gold['flip'][i]), int(gold['dx'][i]))
        name = str(gold['names'][i])
        assert o['status'] == gold['status'][i], name
        if o['occlusion'] is not None:
            np.testing.assert_array_equal(o['occlusion'], gold['occlusion'][i, :r], err_msg=name)
        if o['status'] != D.OK:
            continue
        np.testing.assert_array_equal(o['cor'], gold['cor_out'][i, :r], err_msg=name)
        np.testing.assert_array_equal(o['y_bon'][:, i % 8::8], gold['y_bon'][i], err_msg=name)
        np.testing.assert_array_equal(o['y_cor'][0, i % 8::8], gold['y_cor'][i], err_msg=name)
    assert set(gold['status'].tolist()) == {D.OK, D.ERR_ROWS, D.ERR_CORNERS, D.ERR_BOUNDARY, D.ERR_OCCLUDED}
    assert gold['occlusion'].any() and gold['near_degenerate'].any() and gold['flip'].any() and (gold['kx'] > 0).any()


@pytest.mark.parametrize('seg, other, meets', [
    ([(0, 0), (2, 2)], [(0, 2), (2, 0)], True),                 # crossing
    ([(0, 0), (1, 1)], [(1, 1), (3, 0)], True),                 # touching at an endpoint
    ([(0, 0), (1, 1)], [(2, 0), (0.5, 0.5)], True),             # an endpoint of the other on the segment
    ([(0, 0), (2, 0)], [(1, 0), (3, 0)], True),                 # collinear overlap
    ([(0, 0), (1, 0)], [(2, 0), (3, 0)], False),                # collinear, disjoint
    ([(0, 0), (1, 1)], [(0, 1), (0.4, 0.6 + 1e-12)], False),    # a hair short of the segment
    ([(0, 0), (1, 1)], [(3, 0), (0, 3), (-1, 0)], False),       # a polyline around it
    ([(0, 0), (1, 1)], [(3, 0), (0.5, 0.5), (-1, 0)], True),    # a polyline through its interior vertex
])
def test_exact_linestring(seg, other, meets):
    assert D.LineString(seg).intersects(D.LineString(other)) is meets
    assert D.LineString(other).intersects(D.LineString(seg)) is meets


def test_exact_linestring_float32_tie():
    """Points collinear in float32 arithmetic only to within rounding: decided exactly, not by a tolerance."""
    a = np.float32(0.1)
    q = (float(a) * 3, float(np.float32(float(a) * 3)))
    exact = D.orient((0, 0), (float(a), float(a)), q)
    assert exact == (1 if q[1] > q[0] else -1 if q[1] < q[0] else 0)
    with pytest.raises(ValueError):
        D.LineString([(1, 2)])


def test_read_corners_matches_reference(tmp_path):
    from horizonnet_b200.dataset import read_corners
    cor = D.synthetic_room(np.random.RandomState(5), 'l_shape')
    cor = np.roll(cor, 4, 0)
    p = tmp_path / 'a.txt'
    p.write_text(''.join('%d %d\n' % (x, y) for x, y in cor) + '\n')
    want = np.roll(cor[:, :2], -2 * np.argmin(cor[::2, 0]), 0)        # dataset.py:57-62
    got = read_corners(str(p))
    assert got.dtype == np.float32
    np.testing.assert_array_equal(got, want)
    bad = cor.copy()
    bad[1, 0] += 20                                                     # ceiling and floor columns 20 px apart
    p.write_text(''.join('%d %d\n' % (x, y) for x, y in bad))
    with pytest.raises(AssertionError, match='a.txt'):
        read_corners(str(p))
    bad = cor.copy()
    bad[0, 1], bad[1, 1] = bad[1, 1], bad[0, 1]                         # ceiling below the floor
    p.write_text(''.join('%d %d\n' % (x, y) for x, y in bad))
    with pytest.raises(AssertionError, match='a.txt'):
        read_corners(str(p))


def _adjust_learning_rate(args):
    """misc/utils.py:35-46, restated for the golden sequence below."""
    if args.cur_iter < args.warmup_iters:
        frac = args.cur_iter / args.warmup_iters
        args.running_lr = args.warmup_lr + (args.lr - args.warmup_lr) * frac
    else:
        frac = (float(args.cur_iter) - args.warmup_iters) / (args.max_iters - args.warmup_iters)
        args.running_lr = args.lr * max((1. - frac), 0.) ** args.lr_pow


# misc.utils.adjust_learning_rate for lr 1e-4, warmup_lr 1e-6, lr_pow 0.9, 2 warm-up iterations of 8, at iterations 0..8
GOLDEN_LR = [1e-06, 5.05e-05, 0.0001, 8.486661467891868e-05, 6.942531626616071e-05, 5.358867312681466e-05,
             3.720410580113015e-05, 1.993718664752192e-05, 0.0]


def test_lr_schedule_matches_reference():
    from horizonnet_b200.train import learning_rate
    args = types.SimpleNamespace(lr=1e-4, warmup_lr=1e-6, lr_pow=0.9, warmup_iters=2, max_iters=8)
    for it in range(9):
        args.cur_iter = it
        _adjust_learning_rate(args)
        assert args.running_lr == GOLDEN_LR[it]
        assert learning_rate(it, 1e-4, 1e-6, 0.9, 2, 8) == GOLDEN_LR[it]
