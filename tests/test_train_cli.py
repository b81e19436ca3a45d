"""GPU: dataset.PanoCorBonBatches and ``python -m horizonnet_b200.train`` on a temporary dataset directory of synthetic
512 x 1024 PNG rooms with label_cor files.  The batches must equal the image oracle (augment_ref.augment_image, 3e-7 as
smoke()) and the target oracle (dataset_ref) under the loader's own draws, and the same seed must give the same stream.
The CLI must write train.py's checkpoints, finite scalars, and lower the training loss on a repeated set."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import __graft_entry__ as entry
from horizonnet_b200.augment import augment_corners, draw_params
from horizonnet_b200.dataset import PanoCorBonBatches, read_corners
from oracle import augment_ref
from oracle import dataset_ref as D

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _image(seed):
    """A smooth-ish synthetic panorama: walls in grey levels with noise."""
    rs = np.random.RandomState(seed)
    base = rs.randint(40, 200, size=(8, 16, 3)).astype(np.float32)
    img = np.kron(base, np.ones((64, 64, 1), np.float32)) + rs.randint(0, 30, size=(512, 1024, 3))
    return np.clip(img, 0, 255).astype(np.uint8)


def make_dataset(root, n, seed=0):
    from PIL import Image
    os.makedirs(os.path.join(root, 'img'), exist_ok=True)
    os.makedirs(os.path.join(root, 'label_cor'), exist_ok=True)
    rs = np.random.RandomState(seed)
    for i in range(n):
        cor = D.synthetic_room(rs, D.ROOM_KINDS[i % 3])
        Image.fromarray(_image(seed * 100 + i)).save(os.path.join(root, 'img', 'pano%02d.png' % i))
        with open(os.path.join(root, 'label_cor', 'pano%02d.txt' % i), 'w') as f:
            f.write(''.join('%d %d\n' % (x, y) for x, y in cor))
    return root


@pytest.fixture(scope='module')
def data(tmp_path_factory):
    entry.build()
    return make_dataset(str(tmp_path_factory.mktemp('ds')), 6)


def test_batches_match_oracles(data):
    ld = PanoCorBonBatches(data, 3, flip=True, rotate=True, gamma=True, stretch=True, shuffle=True, seed=7,
                           num_threads=3, return_cor=True)
    rs = np.random.RandomState(7)
    order = rs.permutation(6)
    batches = list(ld)
    assert len(batches) == 2
    for g, (x, y_bon, y_cor, cors) in enumerate(batches):
        for b in range(3):
            i = int(order[3 * g + b])
            c0 = read_corners(os.path.join(data, 'label_cor', 'pano%02d.txt' % i))
            p = draw_params(c0, 1024, rng=rs)
            xr = augment_ref.augment_image(_image(i), p['kx'], p['ky'], p['flip'], p['dx'], p['p'])
            assert float(np.abs(x[b].cpu().numpy() - xr).max()) <= 3e-7
            cs = augment_corners(c0, 512, 1024, p['kx'], p['ky'])
            ref = D.targets(c0, cs, p['flip'], p['dx'], trig='device')
            assert ref['status'] == D.OK
            np.testing.assert_array_equal(cors[b].cpu().numpy(), ref['cor'])
            ulp = np.abs(y_cor[b].cpu().numpy().view(np.int32).astype(np.int64) - ref['y_cor'].view(np.int32))
            assert ulp.max() <= 1
            assert float(np.abs(y_bon[b].cpu().numpy().astype(np.float64) - ref['y_bon']).max()) <= 1e-5
    again = list(PanoCorBonBatches(data, 3, flip=True, rotate=True, gamma=True, stretch=True, shuffle=True, seed=7,
                                   num_threads=2))
    for a, b in zip(batches, again):
        for u, v in zip(a[:3], b):
            assert torch.equal(u, v)


def test_batches_refuse_other_sizes(tmp_path):
    from PIL import Image
    root = make_dataset(str(tmp_path), 2)
    Image.fromarray(np.zeros((256, 512, 3), np.uint8)).save(os.path.join(root, 'img', 'pano01.png'))
    with pytest.raises(ValueError, match='pano01.png'):
        list(PanoCorBonBatches(root, 2))


def test_train_cli_runs_and_learns(data, tmp_path):
    ck, logs = str(tmp_path / 'ckpt'), str(tmp_path / 'logs')
    cmd = [sys.executable, '-m', 'horizonnet_b200.train', '--id', 't', '--ckpt', ck, '--logs', logs,
           '--backbone', 'resnet18', '--train_root_dir', data, '--valid_root_dir', data, '--batch_size_train', '2',
           '--batch_size_valid', '4', '--epochs', '3', '--save_every', '1', '--num_workers', '2', '--lr', '3e-4',
           '--no_flip', '--no_rotate', '--no_gamma', '--no_pano_stretch', '--disp_iter', '2']
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout + r.stderr
    files = os.listdir(os.path.join(ck, 't'))
    assert 'checkpoint.pth.tar' in files
    assert any(f.startswith('best_model_') for f in files), files
    assert {'epoch_1.pth', 'epoch_2.pth', 'epoch_3.pth'} <= set(files)
    from horizonnet_b200.inference import load_checkpoint
    net = load_checkpoint(os.path.join(ck, 't', 'epoch_3.pth'), torch.device('cuda'))
    assert net.backbone == 'resnet18' and net.use_rnn
    recs = [json.loads(l) for l in open(os.path.join(logs, 't', 'scalars.jsonl'))]
    tags = {r['tag'] for r in recs}
    assert {'train/bon', 'train/cor', 'train/total', 'train/lr', 'valid/bon', 'valid/cor', 'valid/total', 'valid/2DIoU',
            'valid/3DIoU', 'valid/rmse', 'valid/delta_1'} == tags
    assert all(np.isfinite(r['value']) for r in recs)
    total = {r['step']: r['value'] for r in recs if r['tag'] == 'train/total'}
    assert sorted(total) == list(range(1, 10))                       # 3 steps per epoch
    first, last = np.mean([total[s] for s in (1, 2, 3)]), np.mean([total[s] for s in (7, 8, 9)])
    print('mean training loss: epoch 1 %.4f, epoch 3 %.4f' % (first, last))
    assert last < first
    r = subprocess.run([sys.executable, '-m', 'horizonnet_b200.train', '--id', 'u', '--backbone', 'densenet121',
                        '--train_root_dir', data, '--valid_root_dir', '', '--ckpt', ck, '--logs', logs],
                       cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode != 0 and 'densenet121' in r.stderr
