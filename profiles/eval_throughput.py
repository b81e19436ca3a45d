"""Throughput of the layout evaluation (csrc/layout_eval.cu) and of validate(), batch 32.

  * evaluation kernels: hn_layout_eval_general on 32 (dt, gt) pairs (device ms per call, CUDA events over many calls): the
    golden rooms against jittered copies and the random-weight model's 1024-corner force_raw rings;
  * validate() (inference with force_raw plus the scoring, one host copy per batch) against infer_layout(force_raw=True)
    alone, panoramas/s, resnet50 with the bi-LSTM, timed in alternating rounds;
  * the numpy oracle (oracle/eval_general_ref.py, the reference's algorithm) on the CPU, ms per pair, on the same pairs.
Prints one JSON object with the card name, power limit and SM clock limit (read-only nvidia-smi query).

    python profiles/eval_throughput.py [--batch 32] [--rounds 5] [--iters 20] [--oracle_pairs 8] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'profiles'))

from head_throughput import card     # noqa: E402


def sm_clock():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                      # the numbers are still printed without it
        return 'unknown (%s)' % e


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
    from horizonnet_b200 import evaluate as EV
    from horizonnet_b200.inference import infer_layout
    from horizonnet_b200.model import HorizonNet
    from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas
    from oracle import eval_general_ref as E
    entry.build()
    B = args.batch
    dev = torch.device('cuda', 0)

    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'eval_general.npz'))
    names = [str(n) for n in g['names'] if str(n).startswith(('room', 'raw'))]
    names = (names * (B // len(names) + 1))[:B]
    scale = np.array([1024, 512], np.float32)
    cor = lambda n, side: g['layout/%s/cor' % str(g['%s/%s_key' % (n, side)])]   # noqa: E731
    dts = [cor(n, 'dt') / scale for n in names]
    gts = [cor(n, 'gt') for n in names]

    out = dict(card(), sm_clock_max=sm_clock(), batch=B, pairs='golden rooms vs jittered copies and 1024-corner rings')
    for _ in range(3):
        EV._eval(dts, gts)
    # the call itself, on padded device inputs (what validate runs after inference)
    dt, dt_rows = EV._pad(dts, dev)
    gt, gt_rows = EV._pad(gts, dev)
    R = max(dt.shape[1], gt.shape[1])
    dt = torch.nn.functional.pad(dt, (0, 0, 0, R - dt.shape[1]))
    gt = torch.nn.functional.pad(gt, (0, 0, 0, R - gt.shape[1]))
    o = EV._outputs(B, dev)
    from horizonnet_b200 import _lib
    lib = _lib.lib()

    def kernel():
        _lib.check(lib.hn_layout_eval_general(dt.data_ptr(), dt_rows.data_ptr(), None, gt.data_ptr(), gt_rows.data_ptr(),
                                              B, R, o['iou2d'].data_ptr(), o['iou3d'].data_ptr(), o['rmse'].data_ptr(),
                                              o['delta_1'].data_ptr(), o['status'].data_ptr(), None, None),
                   'hn_layout_eval_general')

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

    net = HorizonNet('resnet50', True).eval()
    net.load_state_dict(synthetic_state_dict(0, 'random'), strict=True)
    net = net.to(dev)
    x = synthetic_panoramas(B, seed=1000).to(dev)
    vgts = [gts[i % len(gts)] for i in range(B)]
    runs = {'infer_layout_raw': lambda: infer_layout(net, x, force_raw=True, return_status=True),
            'validate': lambda: EV.validate(net, x, vgts, return_status=True)}
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
        E.test_general(E.dt_pixels(dts[i]), gts[i])
    out['oracle_cpu_ms_per_pair'] = (time.perf_counter() - t0) * 1e3 / n
    out['oracle_cpu_pairs'] = names[:n]
    s = json.dumps(out, indent=1)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, 'w').write(s + '\n')


if __name__ == '__main__':
    main()
