"""Does the bi-LSTM of one batch run beside the encoder of the next?  Two measurements on cuda:0, printed as one JSON
object together with the card name and power limit (read-only nvidia-smi query) and the number of 16-CTA clusters the
device co-schedules for the recurrence (max_clusters, printed by the library under HN_LSTM_VERBOSE=1):

1. hn_lstm_layer at T = 256, timed with CUDA events (median of --reps launches after a warm-up), B = 8, 16, 24
   and 32.  The library runs one 8-column group per cluster when all 2 x ceil(B/8) clusters fit in one wave of
   max_clusters, two groups per cluster otherwise; `gpc` and `clusters` say what each B ran.
2. Three pipelined batch-32 steps (HorizonNet.forward_pipelined) under torch.profiler after a warm-up: every kernel
   with its stream, start and duration (the per-stream timeline), and how long recurrence kernels ran while a kernel
   of the other stream was running.

    python profiles/stream_overlap.py [--reps 20] [--out FILE] [--trace FILE]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'profiles'))

from head_throughput import card          # noqa: E402


def max_clusters(lib, torch):
    """The library prints the occupancy answer once per process under HN_LSTM_VERBOSE=1: run a tiny layer with
    stderr captured."""
    xd = torch.zeros(2, 1, 4096, device='cuda:0')
    w = torch.zeros(2048, 512, device='cuda:0')
    out = torch.empty(2, 1, 1024, device='cuda:0')
    with tempfile.TemporaryFile(mode='w+') as f:
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            lib.hn_lstm_layer(xd.data_ptr(), w.data_ptr(), w.data_ptr(), out.data_ptr(), 2, 1, None)
            torch.cuda.synchronize()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        text = f.read()
    for line in text.splitlines():
        if 'max active 16-CTA clusters' in line:
            return int(line.rsplit('=', 1)[1])
    return None


def time_lstm(lib, torch, B, reps, mc):
    g = torch.Generator().manual_seed(B)
    x = (torch.randn(256, B, 4096, generator=g) * 0.5).to('cuda:0')
    w0 = (torch.rand(2048, 512, generator=g) * 0.08 - 0.04).to('cuda:0')
    w1 = (torch.rand(2048, 512, generator=g) * 0.08 - 0.04).to('cuda:0')
    out = torch.empty(256, B, 1024, device='cuda:0')
    st = torch.cuda.current_stream().cuda_stream

    def once():
        lib.hn_lstm_layer(x.data_ptr(), w0.data_ptr(), w1.data_ptr(), out.data_ptr(), 256, B, st)

    for _ in range(3):
        once()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        once()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ng = (B + 7) // 8
    gpc = 1 if mc is None or 2 * ng <= mc else 2
    return {'gpc': gpc, 'clusters': 2 * ((ng + gpc - 1) // gpc), 'ms': round(statistics.median(ts), 3),
            'ms_range': [round(min(ts), 3), round(max(ts), 3)]}


def pipelined_timeline(torch, steps=3, warmup=3):
    from torch.profiler import profile, ProfilerActivity
    from horizonnet_b200.model import HorizonNet
    from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas
    net = HorizonNet('resnet50', True).eval()
    net.load_state_dict(synthetic_state_dict(0, 'random'), strict=True)
    net = net.to('cuda:0')
    xs = [synthetic_panoramas(32, seed=1000 + i).to('cuda:0') for i in range(2)]
    with torch.no_grad():
        for i in range(warmup):
            net.forward_pipelined(xs[i % 2])
        net.flush()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(steps):
                net.forward_pipelined(xs[i % 2])
            net.flush()
            torch.cuda.synchronize()
        net.check()
    kernels = []
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.time_range.elapsed_us() > 0 and 'emcpy' not in e.name \
                and 'emset' not in e.name:
            kernels.append({'name': e.name, 'stream': getattr(e, 'device_resource_id', None) or getattr(e, 'stream', None),
                            'start_us': e.time_range.start, 'dur_us': e.time_range.elapsed_us()})
    kernels.sort(key=lambda k: k['start_us'])
    if kernels:
        t0 = kernels[0]['start_us']
        for k in kernels:
            k['start_us'] = round(k['start_us'] - t0, 2)
            k['dur_us'] = round(k['dur_us'], 2)
    rnn = [k for k in kernels if 'lstm' in k['name']]
    rnn_streams = {k['stream'] for k in rnn}
    other = [k for k in kernels if k['stream'] not in rnn_streams]

    def overlap(k):
        a0, a1 = k['start_us'], k['start_us'] + k['dur_us']
        iv = sorted((max(a0, o['start_us']), min(a1, o['start_us'] + o['dur_us'])) for o in other)
        tot, end = 0.0, a0
        for s, e in iv:
            if e > s and e > end:
                tot += e - max(s, end)
                end = e
        return tot
    span = (kernels[-1]['start_us'] + kernels[-1]['dur_us']) if kernels else 0.0
    return {'steps': steps, 'span_us': round(span, 1), 'ms_per_step': round(span / steps / 1000.0, 3),
            'recurrence_kernel_us': round(sum(k['dur_us'] for k in rnn), 1),
            'recurrence_us_beside_other_stream': round(sum(overlap(k) for k in rnn), 1),
            'kernels': kernels}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--out', default=None, help='also write the summary JSON here')
    ap.add_argument('--trace', default=None, help='write the summary with the full kernel timeline here')
    args = ap.parse_args()
    os.environ['HN_LSTM_VERBOSE'] = '1'
    import torch
    import __graft_entry__ as entry
    from horizonnet_b200 import _lib
    entry.build()
    lib = _lib.lib()
    mc = max_clusters(lib, torch)
    res = dict(card(), max_clusters=mc)
    res['lstm_T256'] = {'B%d' % B: time_lstm(lib, torch, B, args.reps, mc) for B in (8, 16, 24, 32)}
    tl = pipelined_timeline(torch)
    res['pipelined_b32'] = {k: v for k, v in tl.items() if k != 'kernels'}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')
    if args.trace:
        with open(args.trace, 'w') as f:
            json.dump(dict(res, kernels=tl['kernels']), f)
            f.write('\n')


if __name__ == '__main__':
    main()
