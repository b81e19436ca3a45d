"""Throughput of the cuboid evaluation (csrc/layout_cuboid.cu) and of evaluate_cuboid(), batch 32.

  * evaluation kernels: hn_layout_eval_cuboid on 32 (dt, gt) pairs (device ms per call, CUDA events over many calls):
    the golden cuboid rooms against jittered copies and the reference's force_cuboid outputs against rooms;
  * evaluate_cuboid() (inference with force_cuboid plus the scoring, one host copy per batch) against
    infer_layout(force_cuboid=True) alone, panoramas/s, resnet50 with the bi-LSTM, timed in alternating rounds;
  * the numpy oracle (oracle/eval_cuboid_ref.py) on the CPU, ms per pair, on the same pairs.
Prints one JSON object with the card name, power limit and SM clock limit (read-only nvidia-smi query).

    python profiles/eval_cuboid_throughput.py [--batch 32] [--rounds 5] [--iters 20] [--oracle_pairs 8] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'profiles'))

from head_throughput import card     # noqa: E402
from eval_throughput import sm_clock     # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--oracle_pairs', type=int, default=8)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    import __graft_entry__ as entry
    from horizonnet_b200 import _lib
    from horizonnet_b200 import eval_cuboid as EC
    from horizonnet_b200.evaluate import _pad
    from horizonnet_b200.inference import infer_layout
    from horizonnet_b200.model import HorizonNet
    from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas
    from oracle import eval_cuboid_ref as C
    entry.build()
    B = args.batch
    dev = torch.device('cuda', 0)

    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'eval_cuboid.npz'))
    names = [str(n) for n in g['names'] if '_jitter' in str(n) or '_cub_' in str(n)]
    names = (names * (B // len(names) + 1))[:B]
    scale = np.array([1024, 512], np.float32)
    dts = [g[n + '/dt'] / scale for n in names]
    gts = [g[n + '/gt'] for n in names]
    z0s = [float(g[n + '/z0']) for n in names]
    z1s = [float(g[n + '/z1']) for n in names]

    out = dict(card(), sm_clock_max=sm_clock(), batch=B,
               pairs='golden cuboid rooms vs jittered copies and the reference force_cuboid outputs vs rooms')
    for _ in range(3):
        EC.eval_cuboid(dts, z0s, z1s, gts, return_status=True)
    # the call itself, on padded device inputs (what evaluate_cuboid runs after inference)
    dt, dt_rows = _pad(dts, dev)
    gt, gt_rows = _pad(gts, dev)
    z0 = torch.tensor(z0s, device=dev, dtype=torch.float64)
    z1 = torch.tensor(z1s, device=dev, dtype=torch.float64)
    o = EC._outputs(B, dev)
    lib = _lib.lib()

    def kernel():
        _lib.check(lib.hn_layout_eval_cuboid(dt.data_ptr(), dt_rows.data_ptr(), None, z0.data_ptr(), z1.data_ptr(),
                                             gt.data_ptr(), gt_rows.data_ptr(), B, 8, o['ce'].data_ptr(),
                                             o['pe'].data_ptr(), o['iou3d'].data_ptr(), o['status'].data_ptr(), None),
                   'hn_layout_eval_cuboid')

    for _ in range(3):
        kernel()
    ms = []
    for _ in range(args.rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            kernel()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b) / args.iters)
    out['eval_kernels_ms_per_batch'] = {'median': statistics.median(ms), 'min': min(ms), 'max': max(ms)}
    out['statuses'] = {str(k): int(v) for k, v in zip(*np.unique(o['status'].cpu().numpy(), return_counts=True))}

    net = HorizonNet('resnet50', True).eval()
    net.load_state_dict(synthetic_state_dict(0, 'random'), strict=True)
    net = net.to(dev)
    x = synthetic_panoramas(B, seed=1000).to(dev)
    vgts = [gts[i % len(gts)] for i in range(B)]
    runs = {'infer_layout_cuboid': lambda: infer_layout(net, x, force_cuboid=True, return_status=True),
            'evaluate_cuboid': lambda: EC.evaluate_cuboid(net, x, vgts, return_status=True)}
    with torch.no_grad():
        for f in runs.values():
            for _ in range(3):
                f()
        torch.cuda.synchronize()
        times = {k: [] for k in runs}
        for _ in range(args.rounds):
            for k, f in runs.items():
                t0 = time.perf_counter()
                for _ in range(max(1, args.iters // 4)):
                    f()
                torch.cuda.synchronize()
                times[k].append((time.perf_counter() - t0) / max(1, args.iters // 4))
    for k, ts in times.items():
        out[k + '_panoramas_per_s'] = {'median': B / statistics.median(ts), 'min': B / max(ts), 'max': B / min(ts)}

    t0 = time.perf_counter()
    n = min(args.oracle_pairs, B)
    for i in range(n):
        C.test_cuboid(C.dt_pixels(dts[i]), z0s[i], z1s[i], gts[i])
    out['oracle_cpu_ms_per_pair'] = (time.perf_counter() - t0) * 1e3 / n
    out['oracle_cpu_pairs'] = names[:n]
    s = json.dumps(out, indent=1)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, 'w').write(s + '\n')


if __name__ == '__main__':
    main()
