"""Eval-forward throughput of the two heads of HorizonNet('resnet50', use_rnn): bi-LSTM (use_rnn=True) against the
per-column MLP (use_rnn=False), batch 32, tensor cores on, timed with CUDA events.  The two models are timed in
alternating rounds in one process, after a warm-up, so that clock and thermal drift hit both alike.  Prints one JSON
object: the card name and power limit (read-only nvidia-smi query), ms per batch and panoramas/s per head (median and
range over the rounds), and the per-class device profile of one forward of each (hn_model_profile_read).

    python profiles/head_throughput.py [--batch 32] [--rounds 5] [--iters 10] [--out FILE]
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
    ap.add_argument('--batch', type=int, default=32)
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
    nets = {}
    for name, use_rnn in (('rnn', True), ('mlp', False)):
        net = HorizonNet('resnet50', use_rnn).eval()
        net.load_state_dict(synthetic_state_dict(0, 'random', use_rnn=use_rnn), strict=True)
        nets[name] = net.to(dev)
    with torch.no_grad():
        for net in nets.values():
            for _ in range(args.warmup):
                net(x)
        torch.cuda.synchronize()
        times = {name: [] for name in nets}
        for _ in range(args.rounds):
            for name, net in nets.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.iters):
                    net(x)
                b.record()
                b.synchronize()
                times[name].append(a.elapsed_time(b) / args.iters)
        profiles = {}
        for name, net in nets.items():
            net.set_profile(True)
            net.read_profile(reset=True)
            net(x)
            torch.cuda.synchronize()
            profiles[name] = {k: round(v[0], 3) for k, v in net.read_profile(reset=True).items()}
            net.set_profile(False)
            net.check()
    res = dict(card(), batch=args.batch, rounds=args.rounds, iters_per_round=args.iters)
    for name, t in times.items():
        med = statistics.median(t)
        res[name] = {'ms_per_batch': round(med, 3), 'ms_range': [round(min(t), 3), round(max(t), 3)],
                     'panoramas_per_s': round(args.batch * 1000.0 / med, 1), 'profile_ms': profiles[name]}
    res['mlp_saves_ms_per_batch'] = round(res['rnn']['ms_per_batch'] - res['mlp']['ms_per_batch'], 3)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
