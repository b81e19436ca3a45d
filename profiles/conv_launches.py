"""Per-launch time of every convolution of the plain resnet50_rnn forward (batch 32, 512 x 1024), from torch.profiler.

The tensor-core convolution kernels (conv_tc_kernel, gemm_tc_kernel, bott_tc_kernel) run in a fixed order per forward:
the units of tests/tc_cases.resnet50_rnn_convs (layer1's conv2 + conv3 fused into one bott_tc_kernel; with the model option
fold_downsample, the default, each block-0 downsample inside its conv3), then the two LSTM input projections.  Each launch is listed with its plan (hn_conv_tc_plan), its algorithmic FLOPs and a model of the
operand bytes it pulls from L2 into shared memory.  HN_TC_PDL applies: with programmatic dependent launch on (the
default) a kernel's duration includes the time it waits for its predecessor, HN_TC_PDL=0 gives the clean attribution.

    python profiles/conv_launches.py --out table.json [--reps 5] [--fold-downsample 0]
"""
import argparse
import json
import math
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

B = 32
CONV_KERNELS = ('conv_tc_kernel', 'gemm_tc_kernel', 'bott_tc_kernel')


def expected_launches(fold=False):
    """(name, launch dict or None for the fused layer1 bottleneck) in forward order.  fold: the model option
    fold_downsample (on by default) -- no downsample launches; the block-0 conv3 of layers 2-4 runs as one two-source
    launch over [t2 | x] (a 'fold' launch dict, plan_of), layer1.0's inside bott_tc_kernel."""
    import tc_cases as T
    convs = T.resnet50_rnn_convs()
    ds = {n.rsplit('.', 1)[0]: (H, W, Ci, st[0]) for n, H, W, Ci, Co, k, st in convs if n.endswith('downsample')}
    out = []
    for name, H, W, Ci, Co, k, st in convs:
        blk = name.rsplit('.', 1)[0]
        if fold and name.endswith('downsample'):
            continue
        if name.startswith('layer1') and name.endswith('conv3'):
            continue
        if name.startswith('layer1') and name.endswith('conv2'):
            out.append((name[:-1] + '2+conv3', None))
            continue
        if fold and name.endswith('conv3') and blk in ds:
            Hx, Wx, Cx, s = ds[blk]
            out.append((name + '+downsample', dict(name=name + '+downsample', fold=True, B=B, H=Hx, W=Wx, Cin=Cx, Cmid=Ci,
                                                   Cout=Co, k=1, stride=(s, s))))
            continue
        out.append((name, T.launch(name, B, H, W, Ci, Co, k, st, residual=name.endswith('conv3'))))
    for layer in range(2):
        out.append((f'xproj{layer}', T.launch(f'xproj{layer}', 1, 1, 256 * B, 1024, 4096, 1, (1, 1), 0, 0, out_f32=True)))
    return out


def plan_of(c):
    """hn_conv_tc_plan of a launch dict, or hn_conv_tc_fold_plan of a fold launch."""
    import ctypes
    import tc_cases as T
    from horizonnet_b200 import _lib
    if not c.get('fold'):
        return T.plan(c)
    out = (ctypes.c_int * len(T.PLAN_FIELDS))()
    rc = _lib.lib().hn_conv_tc_fold_plan(c['B'], c['H'], c['W'], c['Cin'], c['Cmid'], c['Cout'], c['stride'][0], T.SMS,
                                         out)
    return dict(zip(T.PLAN_FIELDS, out)) if rc == 0 else None


def model_bytes(c, p):
    """Operand bytes (both planes) a launch moves from L2 into shared memory, as the producer loops issue them."""
    bn, kc, n = p['BN'], p['num_kc'], p['num_tiles']
    b_tile = kc * bn * 64 * 4
    if p['dxr']:
        a_tile = (kc // 3) * 130 * 64 * 4
    else:
        a_tile = kc * 128 * 64 * 4
    return n * (a_tile + b_tile)


def round_fit(rows, sms):
    """Least-squares fit of the conv_tc_kernel<128> launches: us per tile round = slope * K chunks + intercept, a round
    being the ceil(num_tiles / sms) tiles each persistent CTA runs.  The intercept is the fixed cost paid once per tile."""
    pts = [(r['num_kc'], r['us'] / math.ceil(r['num_tiles'] / sms)) for r in rows if r['kernel'] == 'conv_tc_kernel<128>']
    n = len(pts)
    if n < 2:
        return None
    mx, my = sum(x for x, _ in pts) / n, sum(y for _, y in pts) / n
    sxx = sum((x - mx) ** 2 for x, _ in pts)
    slope = sum((x - mx) * (y - my) for x, y in pts) / sxx
    icpt = my - slope * mx
    return {'launches': n, 'us_per_chunk': round(slope, 3), 'us_per_tile': round(icpt, 2),
            'max_residual_us': round(max(abs(y - slope * x - icpt) for x, y in pts), 2),
            'tile_rounds': sum(math.ceil(r['num_tiles'] / sms) for r in rows if r['kernel'] == 'conv_tc_kernel<128>')}


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:          # noqa: BLE001
        return f'unavailable: {e}'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--fold-downsample', type=int, choices=(0, 1), default=1, help='model option fold_downsample')
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import __graft_entry__ as entry
    import tc_cases as T
    from horizonnet_b200.model import HorizonNet
    from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas

    entry.build()
    dev = torch.device('cuda', 0)
    net = HorizonNet('resnet50', True).eval()
    net.load_state_dict(synthetic_state_dict(0, 'random'), strict=True)
    net = net.to(dev)
    x = synthetic_panoramas(B, seed=1000).to(dev)
    with torch.no_grad():
        net(x)                                      # creates the handle the option applies to
        net.set_option('fold_downsample', args.fold_downsample)
        for _ in range(3):
            net(x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with torch.no_grad():
            for _ in range(args.reps):
                net(x)
        torch.cuda.synchronize()
    kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
            and any(k in e.name for k in CONV_KERNELS)]
    kern.sort(key=lambda e: e.time_range.start)
    exp = expected_launches(fold=bool(args.fold_downsample))
    if len(kern) != args.reps * len(exp):
        with open(args.out, 'w') as f:
            json.dump({'error': 'launch count', 'kernels': [e.name for e in kern]}, f, indent=1)
        raise SystemExit(f'conv_launches.py: {len(kern)} convolution kernels for {args.reps} forwards, expected '
                         f'{args.reps} x {len(exp)}')
    rows = []
    for i, (name, c) in enumerate(exp):
        evs = [kern[r * len(exp) + i] for r in range(args.reps)]
        us = sorted(e.time_range.end - e.time_range.start for e in evs)
        row = {'name': name, 'kernel': re.search(r'(conv_tc_kernel<\d+>|gemm_tc_kernel|bott_tc_kernel)', evs[0].name).group(1),
               'us': us[len(us) // 2],
               'us_min': us[0], 'us_max': us[-1]}
        if c is not None:
            p = plan_of(c)
            if p is None:
                raise SystemExit(f'conv_launches.py: no plan for {name}')
            want = 'gemm_tc_kernel' if p['gemm_kernel'] else f'conv_tc_kernel<{p["BN"]}>'
            if want not in row['kernel']:
                raise SystemExit(f'conv_launches.py: launch {i} ({name}) ran {row["kernel"]}, the plan says {want}')
            Ho, Wo = c['H'] // c['stride'][0], c['W'] // c['stride'][1]
            flops = 2.0 * c['B'] * Ho * Wo * c['Cout'] * (c['Cin'] * c['k'] * c['k'] + c.get('Cmid', 0))
            row.update({f: p[f] for f in ('BN', 'mode', 'dxr', 'box_rows', 'parity', 'num_kc', 'n_tiles', 'num_tiles',
                                           'grid')})
            row['gflop'] = round(flops / 1e9, 3)
            row['tflops'] = round(flops / (row['us'] * 1e-6) / 1e12, 1)
            row['l2_mb_model'] = round(model_bytes(c, p) / 1e6, 2)
            row['l2_tbs_model'] = round(model_bytes(c, p) / (row['us'] * 1e-6) / 1e12, 2)
        rows.append(row)
    env = {k: v for k, v in os.environ.items() if k.startswith('HN_')}
    fam = {}
    for r in rows:
        f = r['name'].split('.')[0]
        fam[f] = round(fam.get(f, 0.0) + r['us'] / 1e3, 3)
    res = {'card': card(), 'batch': B, 'reps': args.reps, 'env': env, 'options': {'fold_downsample': args.fold_downsample},
           'what': 'median device duration over the reps of each convolution launch of the plain forward (torch.profiler)',
           'family_ms': fam, 'conv_tc_kernel_ms': round(sum(r['us'] for r in rows if 'conv_tc_kernel' in r['kernel']) / 1e3, 3),
           'total_ms': round(sum(r['us'] for r in rows) / 1e3, 3),
           'round_fit': round_fit(rows, torch.cuda.get_device_properties(dev).multi_processor_count), 'launches': rows}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: res[k] for k in ('card', 'env', 'family_ms', 'conv_tc_kernel_ms', 'total_ms', 'round_fit')}))


if __name__ == '__main__':
    main()
