"""Throughput of the two encoders of HorizonNet(backbone, use_rnn=True): resnet18 against resnet50, eval forward at batch 32
(tensor cores on) and the training step (train-mode forward with tape + backward) at batch 8, timed with CUDA events.
Both models are timed in alternating rounds in one process, after a warm-up, so that clock and thermal drift hit both
alike.  Prints one JSON object: the card name and power limit (read-only nvidia-smi query), ms per batch and panoramas/s
per backbone (median and range over the rounds), and the per-class device profile of one eval forward of each
(hn_model_profile_read).

    python profiles/backbone_throughput.py [--batch 32] [--train-batch 8] [--rounds 5] [--iters 10] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'profiles'))

from head_throughput import card            # noqa: E402

BACKBONES = ('resnet18', 'resnet50')


def timed_rounds(fns, rounds, iters):
    """{name: [ms per call of each round]}, the names alternating within every round."""
    import torch
    times = {name: [] for name in fns}
    for _ in range(rounds):
        for name, fn in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                fn()
            b.record()
            b.synchronize()
            times[name].append(a.elapsed_time(b) / iters)
    return times


def summary(t, batch):
    med = statistics.median(t)
    return {'ms_per_batch': round(med, 3), 'ms_range': [round(min(t), 3), round(max(t), 3)],
            'panoramas_per_s': round(batch * 1000.0 / med, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--train-batch', type=int, default=8)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--train-iters', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None, help='also write the JSON here')
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    import __graft_entry__ as entry
    from horizonnet_b200.model import HorizonNet
    from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas
    entry.build()
    dev = torch.device('cuda', 0)
    x = synthetic_panoramas(args.batch, seed=1000).to(dev)
    xt = synthetic_panoramas(args.train_batch, seed=1001).to(dev)
    gen = torch.Generator().manual_seed(9)
    y_bon = (torch.rand(args.train_batch, 2, 1024, generator=gen) - 0.5).to(dev)
    y_cor = torch.rand(args.train_batch, 1, 1024, generator=gen).to(dev)
    nets, train_nets = {}, {}
    for name in BACKBONES:
        sd = synthetic_state_dict(0, 'random', backbone=name)
        for dst, train in ((nets, False), (train_nets, True)):
            net = HorizonNet(name, True)
            net.load_state_dict(sd, strict=True)
            net = net.to(dev)
            dst[name] = net.train() if train else net.eval()

    def train_step(net):
        def step():
            bon, cor = net(xt)
            loss = F.l1_loss(bon, y_bon) + F.binary_cross_entropy_with_logits(cor, y_cor)
            loss.backward()
        return step

    with torch.no_grad():
        for net in nets.values():
            for _ in range(args.warmup):
                net(x)
        torch.cuda.synchronize()
        eval_times = timed_rounds({n: (lambda net=net: net(x)) for n, net in nets.items()}, args.rounds, args.iters)
        profiles = {}
        for name, net in nets.items():
            net.set_profile(True)
            net.read_profile(reset=True)
            net(x)
            torch.cuda.synchronize()
            profiles[name] = {k: round(v[0], 3) for k, v in net.read_profile(reset=True).items()}
            net.set_profile(False)
            net.check()
    steps = {n: train_step(net) for n, net in train_nets.items()}
    for fn in steps.values():
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize()
    train_times = timed_rounds(steps, args.rounds, args.train_iters)
    for net in train_nets.values():
        net.check()
    res = dict(card(), batch=args.batch, train_batch=args.train_batch, rounds=args.rounds, iters_per_round=args.iters,
               train_iters_per_round=args.train_iters)
    for name in BACKBONES:
        res[name] = {'eval': dict(summary(eval_times[name], args.batch), profile_ms=profiles[name]),
                     'train_step': summary(train_times[name], args.train_batch)}
    res['eval_speedup_resnet18'] = round(res['resnet50']['eval']['ms_per_batch'] / res['resnet18']['eval']['ms_per_batch'], 3)
    res['train_speedup_resnet18'] = round(res['resnet50']['train_step']['ms_per_batch'] /
                                          res['resnet18']['train_step']['ms_per_batch'], 3)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
