"""Mint tests/golden/dataset_targets.npz by running the REAL reference dataset.PanoCorBonDataset.__getitem__ on CPU.

Run with a checkout of the reference (sunset1995/HorizonNet) named by HORIZONNET_REFERENCE:
    HORIZONNET_REFERENCE=path/to/HorizonNet python tests/golden/make_golden_dataset.py
Two shims, nothing else patched: shapely is not installed, so ``LineString`` is oracle.dataset_ref's exact one (tested
on hand-made cases in tests/test_dataset_oracle.py); scipy >= 1.9 rejects ``cdist(..., p=1)`` for the default metric, so
cdist is the 'minkowski' metric with p=1 (as make_golden.py does).

Inputs: synthetic cuboids, L-shapes, notched rooms (whose bump hides corners) and edge-on notched rooms (a wall along a
camera ray) with augmentation off, flip + rotate, and stretch + flip + rotate + gamma; the draws are replayed from the
seed as golden_augment does.  Hand-made cases cover each exception.  Per sample: the rolled corners as read (cor0), the
stretched ones (cor), flip, dx (-1: no roll), the reference's status (the stage that raised), occlusion flags, its
flipped and rolled corners, and y_bon / y_cor at every 8th column from (sample % 8).  Flags: near_degenerate
(oracle.dataset_ref.near_degenerate) and order_dependent (eval_general_ref.order_dependent of cor)."""
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.environ.get('HORIZONNET_REFERENCE')
if not REF or not os.path.isfile(os.path.join(REF, 'dataset.py')):
    sys.exit('set HORIZONNET_REFERENCE to a checkout of the reference HorizonNet (the directory holding dataset.py)')
sys.path.insert(0, REF)

from oracle import dataset_ref as D                                 # noqa: E402
from oracle.eval_general_ref import order_dependent                 # noqa: E402
from horizonnet_b200.augment import augment_corners, draw_params    # noqa: E402

for name in ('shapely', 'shapely.geometry'):
    sys.modules.setdefault(name, types.ModuleType(name))
sys.modules['shapely.geometry'].LineString = D.LineString            # shim 1
sys.modules['shapely.geometry'].Polygon = object
import dataset as ref_ds                                             # noqa: E402  (reference dataset.py)
_cdist = ref_ds.cdist
ref_ds.cdist = lambda a, b, p=1: _cdist(a, b, 'minkowski', p=p)      # shim 2

N_ROOMS = 96
AUGS = [dict(flip=False, rotate=False, gamma=False, stretch=False), dict(flip=True, rotate=True, gamma=False, stretch=False),
        dict(flip=True, rotate=True, gamma=True, stretch=True)]
MAX_ROWS = 16


class Stage(Exception):
    pass


def hand_made():
    """(name, corners, expected status) for each exception of the label path."""
    room = D.synthetic_room(np.random.RandomState(1), 'cuboid')
    return [
        ('two_corners', room[:4], D.ERR_CORNERS),
        ('no_samples', np.array([[10.2, 150], [10.2, 350], [10.5, 140], [10.5, 360], [10.8, 150], [10.8, 350]],
                                np.float32), D.ERR_BOUNDARY),
        ('all_occluded', np.array([[100, 150], [100, 350]] * 3, np.float32), D.ERR_OCCLUDED),
    ]


def run(root, name, cor, aug, seed):
    """One sample through the reference -> (record dict, the rolled corners)."""
    with open(os.path.join(root, 'label_cor', name + '.txt'), 'w') as f:
        for x, y in cor:
            f.write('%r %r\n' % (float(x), float(y)))
    os.symlink(os.path.join(root, 'blank.png'), os.path.join(root, 'img', name + '.png'))
    ds = ref_ds.PanoCorBonDataset(root, return_cor=True, **aug)
    idx = ds.img_fnames.index(name + '.png')
    c0 = D.read_roll(cor)
    seen = {}
    orig_occ, orig_c21 = ref_ds.find_occlusion, ref_ds.cor_2_1d

    def occ(c):
        try:
            o = orig_occ(c)
        except ValueError as e:
            raise Stage(D.ERR_CORNERS) from e
        seen['occ'] = o
        return o

    def c21(c, h, w):
        try:
            return orig_c21(c, h, w)
        except ValueError as e:
            raise Stage(D.ERR_BOUNDARY) from e
    ref_ds.find_occlusion, ref_ds.cor_2_1d = occ, c21
    np.random.seed(seed)
    try:
        x, bon, y_cor, cor_out = ds[idx]
        status = D.OK
    except Stage as e:
        status = e.args[0]
    except ValueError:                                             # the odd-row assertion, or dist.min(0) of nothing
        status = D.ERR_ROWS if len(c0) % 2 else D.ERR_OCCLUDED
    finally:
        ref_ds.find_occlusion, ref_ds.cor_2_1d = orig_occ, orig_c21
    np.random.seed(seed)
    p = draw_params(c0, 1024, stretch=aug['stretch'], flip=aug['flip'], rotate=aug['rotate'], gamma=aug['gamma'])
    cs = augment_corners(c0, 512, 1024, p['kx'], p['ky'])
    dx = p['dx'] if aug['rotate'] else -1
    rec = dict(status=status, cor0=c0, cor=cs, flip=int(p['flip']), dx=dx, kx=p['kx'] or 0.0, ky=p['ky'] or 0.0,
               occlusion=seen['occ'].repeat(2) if 'occ' in seen else np.zeros(len(c0), bool))
    if status == D.OK:
        assert np.array_equal(np.asarray(cor_out, np.float32), D.flip_roll_corners(cs, p['flip'], dx)), name
        assert np.asarray(cor_out).dtype == np.float32, name                # numpy 2 keeps the stretched corners float32
        rec.update(cor_out=np.asarray(cor_out, np.float32), y_bon=bon.numpy(), y_cor=y_cor.numpy())
    return rec


def main():
    rs = np.random.RandomState(2024)
    recs, names = [], []
    with tempfile.TemporaryDirectory() as root:
        os.makedirs(os.path.join(root, 'img'))
        os.makedirs(os.path.join(root, 'label_cor'))
        from PIL import Image
        Image.fromarray(np.full((512, 1024, 3), 128, np.uint8)).save(os.path.join(root, 'blank.png'))
        cases = []
        for r in range(N_ROOMS):
            cases.append(('room%03d' % r, D.synthetic_room(rs, D.ROOM_KINDS[r % len(D.ROOM_KINDS)]), AUGS[r % 3]))
        for name, cor, _ in hand_made():
            cases.append((name, cor, AUGS[0]))
        cases.append(('odd_rows', D.synthetic_room(np.random.RandomState(3), 'cuboid')[:7], AUGS[0]))
        for s, (name, cor, aug) in enumerate(cases):
            recs.append(run(root, name, cor, aug, seed=1000 + s))
            names.append(name)
            os.remove(os.path.join(root, 'img', name + '.png'))
            os.remove(os.path.join(root, 'label_cor', name + '.txt'))
    n = len(recs)
    out = dict(names=np.array(names), status=np.array([r['status'] for r in recs], np.int32),
               flip=np.array([r['flip'] for r in recs], np.int32), dx=np.array([r['dx'] for r in recs], np.int32),
               kx=np.array([r['kx'] for r in recs]), ky=np.array([r['ky'] for r in recs]),
               rows=np.array([len(r['cor0']) for r in recs], np.int32))
    for key in ('cor0', 'cor', 'cor_out'):
        a = np.zeros((n, MAX_ROWS, 2), np.float32)
        for i, r in enumerate(recs):
            if key in r:
                a[i, :len(r[key])] = r[key]
        out[key] = a
    occ = np.zeros((n, MAX_ROWS), bool)
    ybon = np.full((n, 2, 128), np.nan, np.float32)
    ycor = np.full((n, 128), np.nan, np.float32)
    for i, r in enumerate(recs):
        occ[i, :len(r['occlusion'])] = r['occlusion']
        if 'y_bon' in r:
            ybon[i] = r['y_bon'][:, i % 8::8]
            ycor[i] = r['y_cor'][0, i % 8::8]
    out.update(occlusion=occ, y_bon=ybon, y_cor=ycor)
    out['near_degenerate'] = np.array([len(r['cor0']) >= 6 and D.near_degenerate(r['cor0'][::2]) for r in recs])
    out['order_dependent'] = np.array([r['status'] == D.OK and order_dependent(r['cor']) for r in recs])
    np.savez_compressed(os.path.join(HERE, 'dataset_targets.npz'), **out)
    print('dataset_targets.npz: %d samples, statuses %s, %d occluded corners, %d near-degenerate, %d order-dependent'
          % (n, np.bincount(out['status']), occ[:, ::2].sum(), out['near_degenerate'].sum(), out['order_dependent'].sum()))


if __name__ == '__main__':
    main()
