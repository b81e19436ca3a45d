"""Throughput of the training data path on the GPU (DESIGN.md section 11).

Reports, in one run on one GPU (its name and power limit read in the same run):
  * panoramas/s of the training loop of ``python -m horizonnet_b200.train`` (resnet50, bi-LSTM, batch 8, every
    augmentation on) reading a synthetic on-disk dataset through dataset.PanoCorBonBatches, against the same
    train_step on device-resident tensors;
  * the time of one hn_train_targets call at N = 8 and 64 (CUDA events over many calls);
  * the host time per batch of 8 for PIL decode + draws (PanoCorBonBatches' host side, one thread pool of 8).
Usage: python profiles/train_throughput.py [--steps 30] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as entry                                        # noqa: E402


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def make_dataset(root, n):
    from PIL import Image
    from oracle.dataset_ref import ROOM_KINDS, synthetic_room
    os.makedirs(os.path.join(root, 'img'))
    os.makedirs(os.path.join(root, 'label_cor'))
    rs = np.random.RandomState(0)
    for i in range(n):
        base = rs.randint(40, 200, size=(8, 16, 3)).astype(np.float32)
        img = np.kron(base, np.ones((64, 64, 1), np.float32)) + rs.randint(0, 30, size=(512, 1024, 3))
        Image.fromarray(np.clip(img, 0, 255).astype(np.uint8)).save(os.path.join(root, 'img', 'p%03d.png' % i))
        cor = synthetic_room(rs, ROOM_KINDS[i % 3])
        with open(os.path.join(root, 'label_cor', 'p%03d.txt' % i), 'w') as f:
            f.write(''.join('%d %d\n' % (x, y) for x, y in cor))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--out', default=None, help='also write the JSON here')
    a = ap.parse_args()
    entry.build()
    from horizonnet_b200 import dataset as DS
    from horizonnet_b200.model import HorizonNet
    from horizonnet_b200.train import train_step
    from horizonnet_b200.weights import synthetic_state_dict
    from oracle import dataset_ref as D
    dev = torch.device('cuda', 0)
    res = {'gpu': gpu_info(), 'batch': 8, 'backbone': 'resnet50', 'use_rnn': True}
    net = HorizonNet('resnet50', True)
    net.load_state_dict(synthetic_state_dict(0, 'random'))
    net = net.to(dev).train()
    opt = torch.optim.Adam(net.parameters(), lr=1e-5)
    B, K = 8, a.steps
    with tempfile.TemporaryDirectory() as root:
        make_dataset(root, B * 8)
        ld = DS.PanoCorBonBatches(root, B, flip=True, rotate=True, gamma=True, stretch=True, shuffle=True,
                                  drop_last=True, seed=1, device=dev, num_threads=8)
        # bare step on device-resident tensors (one batch of the loader, reused)
        x, yb, yc = next(iter(ld))
        for _ in range(3):
            train_step(net, opt, x, yb, yc)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(K):
            train_step(net, opt, x, yb, yc)
        torch.cuda.synchronize()
        bare = (time.perf_counter() - t0) / K
        # the CLI's loop: batches from disk through the loader
        def loop(n_steps):
            done = 0
            while done < n_steps:
                for x, yb, yc in ld:
                    train_step(net, opt, x, yb, yc)
                    done += 1
                    if done == n_steps:
                        break
            torch.cuda.synchronize()
        loop(3)
        t0 = time.perf_counter()
        loop(K)
        looped = (time.perf_counter() - t0) / K
        res['bare_step_ms'] = round(bare * 1e3, 2)
        res['bare_panos_per_s'] = round(B / bare, 1)
        res['loop_step_ms'] = round(looped * 1e3, 2)
        res['loop_panos_per_s'] = round(B / looped, 1)
        # host side of one batch: decode + draws
        idx = list(range(B))
        ld._host(0, idx)
        t0 = time.perf_counter()
        for _ in range(5):
            ld._host(0, idx)
        res['host_ms_per_batch'] = round((time.perf_counter() - t0) / 5 * 1e3, 2)
    # hn_train_targets alone
    rs = np.random.RandomState(3)
    for N in (8, 64):
        cors = [D.read_roll(D.synthetic_room(rs, D.ROOM_KINDS[i % 4])) for i in range(N)]
        flip, dx = [i % 2 == 0 for i in range(N)], [int(rs.randint(1024)) for _ in range(N)]
        keep = [DS._launch_targets(cors, cors, flip, dx, 0.96, dev) for _ in range(3)]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 200
        outs = []
        e0.record()
        for _ in range(reps):
            outs.append(DS._launch_targets(cors, cors, flip, dx, 0.96, dev))
        e1.record()
        torch.cuda.synchronize()
        res['targets_ms_n%d' % N] = round(e0.elapsed_time(e1) / reps, 4)
        assert all(int(o['status'].max()) == 0 for o in keep)
    print(json.dumps(res))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
