"""Runs unit cases of tests/tc_cases.py in a fresh process, so that the HN_TC_* switches, which the library reads once per
process, take effect.  Prints one JSON line per case.  Also holds the LSTM layer check the GPU tests share.

    python tests/tc_runner.py conv NAME...        -> {"name", "ratio", "plan"}"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch                                              # noqa: E402

import gpu_utils as gu                                    # noqa: E402
import tc_cases                                           # noqa: E402


def lstm_error(T, B, dev='cuda:0'):
    """hn_lstm_layer against an fp64 recurrence of the same inputs (test_gpu_parity.py: test_lstm_layer_vs_oracle)."""
    from horizonnet_b200 import _lib
    g = torch.Generator().manual_seed(T * 100 + B)
    xproj = torch.randn(T, B, 4096, generator=g) * 0.5
    whh = [torch.rand(2048, 512, generator=g) * 0.08 - 0.04 for _ in range(2)]
    ref = lstm_reference(xproj, whh)
    out = torch.full((T, B, 1024), float('nan'), device=dev)
    xd, w0, w1 = xproj.to(dev), whh[0].to(dev), whh[1].to(dev)
    _lib.check(_lib.lib().hn_lstm_layer(xd.data_ptr(), w0.data_ptr(), w1.data_ptr(), out.data_ptr(), T, B,
                                        torch.cuda.current_stream().cuda_stream), 'hn_lstm_layer')
    torch.cuda.synchronize()
    return (out.cpu().double() - ref).abs().max().item()


def lstm_reference(xproj, whh):
    """Both directions of one LSTM layer in fp64 from the input projection [T][B][4096]."""
    T, B = xproj.shape[:2]
    out = []
    for d in range(2):
        xp = xproj[:, :, d * 2048:(d + 1) * 2048].double()
        w = whh[d].double()
        h = torch.zeros(B, 512, dtype=torch.float64)
        c = torch.zeros(B, 512, dtype=torch.float64)
        o = torch.empty(T, B, 512, dtype=torch.float64)
        for t in (range(T - 1, -1, -1) if d else range(T)):
            i, f, gg, og = (xp[t] + h @ w.t()).chunk(4, dim=1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
            h = torch.sigmoid(og) * torch.tanh(c)
            o[t] = h
        out.append(o)
    return torch.cat(out, dim=2)


def main(argv):
    import __graft_entry__ as entry
    entry.build()
    kind, names = argv[0], argv[1:]
    cases = {c['name']: c for c in tc_cases.ALL_CASES}
    assert kind == 'conv', kind
    for n in names:
        c = cases[n]
        print(json.dumps({'name': n, 'ratio': gu.run_tc_case(c), 'plan': tc_cases.plan(c, gu.device_sms())}), flush=True)


if __name__ == '__main__':
    main(sys.argv[1:])
