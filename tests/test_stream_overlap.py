"""-m gpu: results that must not depend on how the work is spread over the GPU.

- The LSTM recurrence runs one or two 8-column groups per 16-CTA cluster (two when one group per cluster would need
  a second wave of clusters: B = 32 and 40 on an H100); columns are independent, so every B must give, bit for bit,
  what 8-column launches give.
- The persistent tensor-core kernels claim their tiles from a per-stream counter at run time; which CTA computes a
  tile must not change it, whether the launch runs alone, next to a recurrence, next to another launch, or right
  after itself under programmatic dependent launch.
- The pipelined forward (encoder and recurrence on two streams) must equal the plain forward bit for bit.
- hn_lstm_layer only enqueues the recurrence, so a convolution launched after it on another stream runs beside it."""
import pytest
import torch

import __graft_entry__ as entry
from horizonnet_b200 import _lib
from horizonnet_b200.model import HorizonNet
from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas
import gpu_utils as gu

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.fixture(scope='module', autouse=True)
def _built():
    entry.build()
    _lib.lib()


def _lstm_inputs(T, B, seed):
    g = torch.Generator().manual_seed(seed)
    xproj = torch.randn(T, B, 4096, generator=g) * 0.5
    whh = [torch.rand(2048, 512, generator=g) * 0.08 - 0.04 for _ in range(2)]
    return xproj, whh


def _lstm(xproj_dev, w0, w1, stream=None):
    T, B = xproj_dev.shape[:2]
    out = torch.full((T, B, 1024), float('nan'), device=DEV)
    stream = stream or torch.cuda.current_stream()
    stream.wait_stream(torch.cuda.current_stream())        # the call only enqueues: the NaN fill must come first
    _lib.check(_lib.lib().hn_lstm_layer(xproj_dev.data_ptr(), w0.data_ptr(), w1.data_ptr(), out.data_ptr(), T, B,
                                        stream.cuda_stream), 'hn_lstm_layer')
    return out


def test_lstm_layer_returns_before_the_recurrence_runs():
    xproj, whh = _lstm_inputs(256, 32, 9)
    xd, w0, w1 = xproj.to(DEV), whh[0].to(DEV), whh[1].to(DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(100_000_000)                      # about 50 ms at the H100's 1980 MHz
    h = _lstm(xd, w0, w1, s)
    busy = not s.query()
    s.synchronize()
    assert busy, 'hn_lstm_layer returned only after its stream had drained'
    assert torch.equal(h, _lstm(xd, w0, w1))


@pytest.mark.parametrize('B', [16, 24, 32, 40])
def test_lstm_two_groups_per_cluster_match_one(B):
    T = 256
    xproj, whh = _lstm_inputs(T, B, 500 + B)
    xd, w0, w1 = xproj.to(DEV), whh[0].to(DEV), whh[1].to(DEV)
    out = _lstm(xd, w0, w1)
    parts = [_lstm(xd[:, c:c + 8].contiguous(), w0, w1) for c in range(0, B, 8)]
    torch.cuda.synchronize()
    assert torch.equal(out, torch.cat(parts, dim=1))
    err = (out.cpu().double() - gu.lstm_reference(xproj, whh)).abs().max().item()
    assert err < 2e-6, err


# ------------------------------------------------------------------------------- tile scheduler
def _conv_case(seed):
    """A 3x3 256 -> 256 convolution with residual: 512 tiles of conv_tc_kernel, several per CTA."""
    g = torch.Generator().manual_seed(seed)
    B, Ci, H, W, Co = 8, 256, 32, 256, 256
    x = torch.randn(B, Ci, H, W, generator=g)
    w = torch.randn(Co, Ci, 3, 3, generator=g) / (Ci * 9) ** 0.5
    scale, shift = torch.rand(Co, generator=g) + 0.5, torch.randn(Co, generator=g) * 0.1
    res = torch.randn(B, Co, H, W, generator=g)
    return dict(xin=gu.to_halo_nhwc(x, 1).to(DEV), wp=gu.pack_weight(w).to(DEV), scale=scale.to(DEV),
                shift=shift.to(DEV), res=gu.to_halo_nhwc(res, 1).to(DEV), shape=(B, Ci, H, W, Co))


def _conv_launch(c, stream):
    """Enqueues hn_conv2d (tensor-core kernel) on `stream` without synchronising; returns the output buffer."""
    B, Ci, H, W, Co = c['shape']
    out = torch.full((B, H, W + 2, Co), float('nan'), device=DEV)
    with torch.cuda.stream(stream):
        rc = _lib.lib().hn_conv2d(c['xin'].data_ptr(), B, H, W, Ci, 1, c['wp'].data_ptr(), c['scale'].data_ptr(),
                                  c['shift'].data_ptr(), c['res'].data_ptr(), Co, 3, 3, 1, 1, 1, 1, 1,
                                  out.data_ptr(), 1, 1, stream.cuda_stream)
    _lib.check(rc, 'hn_conv2d')
    return out


def _alone(c):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    out = _conv_launch(c, s)
    s.synchronize()
    return out


def test_conv_beside_recurrence():
    c = _conv_case(1)
    ref = _alone(c)
    xproj, whh = _lstm_inputs(256, 32, 7)
    xd, w0, w1 = xproj.to(DEV), whh[0].to(DEV), whh[1].to(DEV)
    torch.cuda.synchronize()
    s_rnn, s_enc = torch.cuda.Stream(priority=-1), torch.cuda.Stream()
    h = _lstm(xd, w0, w1, s_rnn)
    outs = [_conv_launch(c, s_enc) for _ in range(4)]
    torch.cuda.synchronize()
    for o in outs:
        assert torch.equal(o, ref)
    assert torch.equal(h, _lstm(xd, w0, w1))


def test_conv_back_to_back_on_one_stream():
    c = _conv_case(2)
    ref = _alone(c)
    s = torch.cuda.Stream()
    outs = [_conv_launch(c, s) for _ in range(3)]      # each claims from the counter the previous one reset
    s.synchronize()
    for o in outs:
        assert torch.equal(o, ref)


def test_conv_on_two_streams_at_once():
    c1, c2 = _conv_case(3), _conv_case(4)
    r1, r2 = _alone(c1), _alone(c2)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = []
    for _ in range(3):
        outs.append((_conv_launch(c1, s1), _conv_launch(c2, s2)))
    torch.cuda.synchronize()
    for o1, o2 in outs:
        assert torch.equal(o1, r1) and torch.equal(o2, r2)


# ------------------------------------------------------------------------------- pipelined forward
@pytest.mark.parametrize('B', [32, 5])
def test_pipelined_forward_matches_plain(B):
    sd = synthetic_state_dict(0, 'random')
    net = HorizonNet('resnet50', True).eval()
    net.load_state_dict(sd, strict=True)
    net = net.to(DEV)
    xs = [synthetic_panoramas(B, seed=40 + i).to(DEV) for i in range(3)]
    with torch.no_grad():
        plain = [tuple(t.clone() for t in net(x)) for x in xs]
        piped = [net.forward_pipelined(x) for x in xs]       # batch i's recurrence runs beside batch i+1's encoder
        net.flush()
        torch.cuda.synchronize()
        net.check()
    for (pb, pc), (qb, qc) in zip(plain, piped):
        assert torch.equal(pb, qb) and torch.equal(pc, qc)
