"""Time and device memory of a train-mode forward without autograd, ``net.train(); with torch.no_grad(): net(x)`` (what
BatchNorm re-estimation calls), for HorizonNet('resnet50', True) at batch 8 with tensor cores on.

Time: CUDA events around `iters` back-to-back calls, median over `rounds` after a warm-up.  Memory: the library
allocates with cudaMalloc, not through torch's caching allocator, so device memory in use is read from the driver
(torch.cuda.mem_get_info: total - free) before the model is created and after the first call; the difference covers
the library's workspace and tape plus what torch holds (parameters, input, outputs), which is reported on its own as
torch_reserved_mb.  Prints one JSON object with the card name and power limit (read-only nvidia-smi query).

    python profiles/train_forward_nograd.py [--batch 8] [--rounds 5] [--iters 10] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(',')]
        return {'gpu': name, 'power_limit': limit}
    except Exception as e:                      # the numbers are still printed, without the card beside them
        return {'gpu': 'unknown', 'power_limit': 'unknown', 'error': str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None, help='also write the JSON here')
    args = ap.parse_args()

    import torch
    import __graft_entry__ as entry
    from horizonnet_b200.model import HorizonNet
    from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas
    entry.build()
    dev = torch.device('cuda', 0)
    x = synthetic_panoramas(args.batch, seed=1000).to(dev)

    def used_mb():
        torch.cuda.synchronize(dev)
        free, total = torch.cuda.mem_get_info(dev)
        return (total - free) / 2 ** 20

    before, reserved_before = used_mb(), torch.cuda.memory_reserved(dev)
    net = HorizonNet('resnet50', True)
    net.load_state_dict(synthetic_state_dict(0, 'random'), strict=True)
    net = net.to(dev).train()
    with torch.no_grad():
        net(x)
        after = used_mb()
        for _ in range(args.warmup):
            net(x)
        torch.cuda.synchronize(dev)
        times = []
        for _ in range(args.rounds):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.iters):
                net(x)
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b) / args.iters)
    net.check()
    med = statistics.median(times)
    res = dict(card(), batch=args.batch, rounds=args.rounds, iters_per_round=args.iters,
               ms_per_call=round(med, 3), ms_range=[round(min(times), 3), round(max(times), 3)],
               panoramas_per_s=round(args.batch * 1000.0 / med, 1),
               device_used_mb=round(after - before, 1),
               torch_reserved_mb=round((torch.cuda.memory_reserved(dev) - reserved_before) / 2 ** 20, 1))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
