"""Throughput of the layout post-processing (csrc/layout.cu) and of infer_layout, batch 32.

  * layout kernel: hn_layout_postproc on 32 panoramas' TTA outputs (device ms per call, CUDA events, general and cuboid);
  * infer_layout (no augmentation, general layout) against the eval forward alone, panoramas/s, resnet50 with the bi-LSTM,
    timed in alternating rounds;
  * the numpy oracle (oracle/layout_ref.py, the reference's algorithm) on the CPU, ms per panorama, on the same signals.
Prints one JSON object with the card name and power limit (read-only nvidia-smi query).

    python profiles/layout_throughput.py [--batch 32] [--rounds 5] [--iters 10] [--out FILE]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    import __graft_entry__ as entry
    from horizonnet_b200 import _lib
    from horizonnet_b200.inference import infer_layout, MAX_ROWS
    from horizonnet_b200.model import HorizonNet
    from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas
    from oracle import layout_ref
    entry.build()
    B = args.batch
    dev = torch.device('cuda', 0)

    # signals: the golden rooms (clean and noisy) and the random-weight model's outputs, repeated to B
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'layout.npz'))
    names = [str(n) for n in g['names'] if str(n).startswith(('room', 'randombn'))]
    names = (names * (B // len(names) + 1))[:B]
    yb = torch.from_numpy(np.stack([g[n + '/y_bon'] for n in names])).to(dev)
    yc = torch.from_numpy(np.stack([g[n + '/y_cor'] for n in names])).to(dev)
    cor = torch.empty(B, MAX_ROWS, 2, device=dev)
    ints = [torch.empty(B, dtype=torch.int32, device=dev) for _ in range(2)]
    fl = [torch.empty(B, device=dev) for _ in range(2)]
    lib = _lib.lib()

    def kernel(cuboid):
        _lib.check(lib.hn_layout_postproc(yb.data_ptr(), yc.data_ptr(), B, 26, 0.0 if cuboid else 0.05, int(cuboid), 0,
                                          MAX_ROWS, cor.data_ptr(), ints[0].data_ptr(), fl[0].data_ptr(),
                                          fl[1].data_ptr(), ints[1].data_ptr(), None, None, None), 'hn_layout_postproc')

    out = dict(card(), batch=B)
    for cuboid in (False, True):
        for _ in range(3):
            kernel(cuboid)
        ms = []
        for _ in range(args.rounds):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.iters):
                kernel(cuboid)
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b) / args.iters)
        out['layout_kernel_ms_' + ('cuboid' if cuboid else 'general')] = {
            'median': statistics.median(ms), 'min': min(ms), 'max': max(ms)}

    net = HorizonNet('resnet50', True).eval()
    net.load_state_dict(synthetic_state_dict(0, 'random'), strict=True)
    net = net.to(dev)
    x = synthetic_panoramas(B, seed=1000).to(dev)
    runs = {'forward': lambda: net(x), 'infer_layout': lambda: infer_layout(net, x, return_status=True)}
    with torch.no_grad():
        for f in runs.values():
            for _ in range(3):
                f()
        torch.cuda.synchronize()
        times = {k: [] for k in runs}
        for _ in range(args.rounds):
            for k, f in runs.items():
                t0 = time.perf_counter()
                for _ in range(args.iters):
                    f()
                torch.cuda.synchronize()
                times[k].append((time.perf_counter() - t0) / args.iters)
    for k, ts in times.items():
        out[k + '_panoramas_per_s'] = {'median': B / statistics.median(ts), 'min': B / max(ts), 'max': B / min(ts)}

    ybh, ych = yb.cpu().numpy(), yc.cpu().numpy()
    for cuboid in (False, True):
        t0 = time.perf_counter()
        for i in range(B):
            layout_ref.post_process(ybh[i], ych[i], 26, force_cuboid=cuboid)
        out['oracle_cpu_ms_per_panorama_' + ('cuboid' if cuboid else 'general')] = (time.perf_counter() - t0) * 1e3 / B
    s = json.dumps(out, indent=1)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, 'w').write(s + '\n')


if __name__ == '__main__':
    main()
