"""HorizonNet('resnet18', use_rnn): the torchvision BasicBlock encoder with a 256-wide feature sequence, both heads, through
every layer: spec, synthetic weights, oracle, module surface (CPU) and the library's eval forward, entry points, narrow
height-reduction kernel, 3x3 residual launches, train-mode forward and training step (GPU).  Fixtures: tests/golden/*_r18*
(make_golden_r18.py); checker: oracle/horizonnet_r18_ref.py (with horizonnet_ref.TrainMode for train mode).

Run as a script (``python tests/test_resnet18.py dxr``) it prints the 3x3 residual cases as JSON lines: the dx-reuse switch
HN_TC_DXR is read once per process, so the switched-off path needs a fresh one."""
import json
import os
import subprocess
import sys
from collections import OrderedDict

HERE = os.path.dirname(os.path.abspath(__file__))
if __name__ == '__main__':
    sys.path.insert(0, os.path.dirname(HERE))
    sys.path.insert(0, HERE)

import numpy as np                                                   # noqa: E402
import pytest                                                        # noqa: E402
import torch                                                         # noqa: E402
import torch.nn.functional as F                                      # noqa: E402

from horizonnet_b200._spec import state_dict_spec, HEAD_BIAS, c_last  # noqa: E402
from horizonnet_b200.model import HorizonNet                         # noqa: E402
from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas   # noqa: E402
from oracle import horizonnet_ref, horizonnet_r18_ref as r18         # noqa: E402

DEV = 'cuda:0'
N_PARAMS = {True: 142, False: 128}
N_NUMEL = {True: 23486020, False: 14157892}
N_UNITS = 36                                  # conv units of the tape = BatchNorm2d modules


def _sfx(use_rnn):
    return '_r18' if use_rnn else '_r18_norn'


def _sd(seed, bn, use_rnn):
    return synthetic_state_dict(seed, bn, use_rnn=use_rnn, backbone='resnet18')


def _sample(t, n=4096):
    flat = t.detach().reshape(-1).double().cpu().numpy()
    return flat[::max(1, flat.size // n)][:n].astype(np.float32)


FORWARD_GOLDEN = [('forward_r18_identity', 'identity', True), ('forward_r18_randombn', 'random', True),
                  ('forward_r18_norn_randombn', 'random', False)]


# ------------------------------------------------------------------------------- CPU: spec, weights, oracle, module
@pytest.mark.parametrize('use_rnn', [True, False])
def test_spec_matches_the_reference_resnet18_layout(golden_dir, use_rnn):
    ref = json.load(open(os.path.join(golden_dir, f'state_dict_keys{_sfx(use_rnn)}.json')))
    spec = state_dict_spec(use_rnn, 'resnet18')
    assert len(spec) == len(ref) == (250 if use_rnn else 236)
    for (k, shape, _), (k2, (s2, _)) in zip(ref, spec.items()):
        assert k == k2 and tuple(shape) == tuple(s2)
    params = [s for s, kind in spec.values() if kind not in ('bn_mean', 'bn_var', 'bn_count')]
    assert len(params) == N_PARAMS[use_rnn] and sum(int(np.prod(s)) for s in params) == N_NUMEL[use_rnn]
    assert sum(k.endswith('.running_mean') for k in spec) == N_UNITS
    assert c_last('resnet18') == 256 and c_last() == 1024
    head = 'bi_rnn.weight_ih_l0' if use_rnn else 'linear.0.weight'
    assert spec[head][0] == ((2048, 256) if use_rnn else (512, 256))
    # the resnet50 layouts are untouched by the backbone argument
    assert list(state_dict_spec(use_rnn)) == list(state_dict_spec(use_rnn, 'resnet50'))


def test_synthetic_resnet18_weights_follow_the_reference_init():
    sd = _sd(0, 'identity', True)
    assert list(sd) == list(state_dict_spec(True, 'resnet18'))
    w = sd['feature_extractor.encoder.layer1.0.conv1.1.weight']
    assert w.shape == (64, 64, 3, 3) and abs(float(w.std()) - (2.0 / (64 * 9)) ** 0.5) < 0.01
    mlp = _sd(0, 'identity', False)
    for k, v in mlp.items():
        if not k.startswith('linear'):
            assert torch.equal(v, sd[k]), k
    assert 0.9 * 256 ** -0.5 < float(mlp['linear.0.weight'].abs().max()) <= 256 ** -0.5


@pytest.mark.parametrize('name,bn,use_rnn', FORWARD_GOLDEN)
def test_oracle_matches_the_reference_resnet18_forward(golden_dir, name, bn, use_rnn):
    g = np.load(os.path.join(golden_dir, name + '.npz'))
    sd = _sd(int(g['seed']), bn, use_rnn)
    x = synthetic_panoramas(int(g['batch']), seed=int(g['x_seed']))
    with torch.no_grad():
        bon, cor, stages = r18.forward(sd, x, use_rnn=use_rnn, return_stages=True)
    assert np.abs(bon.numpy() - g['bon']).max() < 2e-5
    assert np.abs(cor.numpy() - g['cor']).max() < 2e-5
    assert tuple(stages['feature'].shape) == (int(g['batch']), 256, 256)
    for k, v in stages.items():
        assert tuple(v.shape) == tuple(g[k + '_shape']), k
        assert np.abs(_sample(v) - g[k + '_sample']).max() <= 2e-6 * float(g[k + '_maxabs']) + 1e-6, k


def train_golden_r18(golden_dir):
    """tests/golden/train_r18.npz -> (g, sd, x, the two dropout masks [256, B, 1024], moved running statistics)."""
    g = np.load(os.path.join(golden_dir, 'train_r18.npz'))
    B = int(g['batch'])
    bits = np.unpackbits(g['masks_bits'])[:2 * 256 * B * 1024].reshape(2, 256, B, 1024)
    masks = [torch.from_numpy(bits[i].astype(np.float32) * 2.0) for i in range(2)]
    sd = _sd(int(g['wseed']), 'random', True)
    x = synthetic_panoramas(B, seed=int(g['x_seed']))
    running, off = {}, 0
    for k in [k for k in sd if k.endswith('running_mean') or k.endswith('running_var')]:
        n = sd[k].numel()
        running[k] = torch.from_numpy(g['running'][off:off + n].copy())
        off += n
    return g, sd, x, masks, running


def test_oracle_matches_the_reference_resnet18_train_forward(golden_dir):
    g, sd, x, masks, running = train_golden_r18(golden_dir)
    tm = horizonnet_ref.TrainMode(masks=masks)
    with torch.no_grad():
        bon, cor = r18.forward(sd, x, train=tm)
    assert np.abs(bon.numpy() - g['bon']).max() < 2e-5 and np.abs(cor.numpy() - g['cor']).max() < 2e-5
    for k, v in running.items():
        assert torch.allclose(tm.running[k], v, rtol=1e-5, atol=1e-6), k
    assert g['num_batches_tracked'].sum() == N_UNITS


def _golden_targets(g):
    batch = int(g['batch'])
    gen = torch.Generator().manual_seed(int(g['y_seed']))
    return torch.rand(batch, 2, 1024, generator=gen) - 0.5, torch.rand(batch, 1, 1024, generator=gen)


@pytest.mark.parametrize('use_rnn', [True, False])
def test_oracle_backward_matches_the_reference_resnet18_backward(golden_dir, use_rnn):
    g = np.load(os.path.join(golden_dir, f'train_backward{_sfx(use_rnn)}.npz'))
    batch, n = int(g['batch']), int(g['n'])
    sd = _sd(int(g['wseed']), 'random', use_rnn)
    x = synthetic_panoramas(batch, seed=int(g['x_seed']))
    y_bon, y_cor = _golden_targets(g)
    torch.manual_seed(int(g['train_seed']))
    if use_rnn:
        masks = [torch.empty(256, batch, 1024).bernoulli_(0.5).div_(0.5) for _ in range(2)]
    else:
        masks = [None, torch.empty(batch, 256, 512).bernoulli_(0.5).div_(0.5)]
    names = [str(k) for k in g['names']]
    assert len(names) == N_PARAMS[use_rnn]
    psd = {k: (v.clone().requires_grad_() if k in names else v) for k, v in sd.items()}
    bon, cor = r18.forward(psd, x, use_rnn=use_rnn, train=horizonnet_ref.TrainMode(masks=masks))
    loss = F.l1_loss(bon, y_bon) + F.binary_cross_entropy_with_logits(cor, y_cor)
    assert abs(loss.item() - float(g['loss'])) < 1e-6
    grads = torch.autograd.grad(loss, [psd[k] for k in names])
    gmax = float(g['absmax'].max())
    worst = 0.0
    for i, gr in enumerate(grads):
        flat = gr.reshape(-1)
        got = flat[::max(1, flat.numel() // n)][:n].numpy()
        scale = float(g['absmax'][i]) + 1e-4 * gmax
        worst = max(worst, float(np.abs(got - g['samples'][i][:got.size]).max()) / scale,
                    abs(float(flat.abs().max()) - float(g['absmax'][i])) / scale)
    assert worst < 5e-4, worst


@pytest.mark.parametrize('use_rnn', [True, False])
def test_module_surface_of_the_resnet18_model(golden_dir, use_rnn):
    keys = [k for k, _, _ in json.load(open(os.path.join(golden_dir, f'state_dict_keys{_sfx(use_rnn)}.json')))]
    net = HorizonNet('resnet18', use_rnn)
    assert list(net.state_dict().keys()) == keys
    net.load_state_dict(_sd(0, 'identity', use_rnn), strict=True)
    assert net.backbone == 'resnet18' and net.use_rnn is use_rnn
    assert sum(p.numel() for p in net.parameters()) == N_NUMEL[use_rnn]
    assert len(list(net.named_parameters())) == N_PARAMS[use_rnn]
    assert sum(isinstance(m, torch.nn.BatchNorm2d) for m in net.modules()) == N_UNITS
    if use_rnn:
        assert net.bi_rnn.input_size == 256 and net.linear.in_features == 1024
        assert torch.equal(net.linear.bias, torch.tensor(HEAD_BIAS, dtype=torch.float32))
    else:
        assert net.linear[0].in_features == 256 and net.linear[0].out_features == 512
        assert torch.equal(net.linear[3].bias, torch.tensor(HEAD_BIAS, dtype=torch.float32))
    blocks = net.feature_extractor.list_blocks()
    assert [len(b) for b in blocks] == [4, 1, 1, 1, 1]
    assert [type(m).__name__ for m in blocks[1][0]] == ['_BasicBlock', '_BasicBlock']
    b0 = net.feature_extractor.encoder.layer2[0]
    assert b0.conv1[1].stride == (2, 2) and b0.conv2[1].stride == (1, 1) and hasattr(b0, 'downsample')
    assert not hasattr(net.feature_extractor.encoder.layer1[0], 'downsample')


def test_other_backbones_still_raise():
    for backbone in ('resnet34', 'resnet101', 'resnet152', 'densenet121', 'densenet169'):
        for use_rnn in (False, True):
            with pytest.raises(NotImplementedError):
                HorizonNet(backbone, use_rnn)


def test_resnet18_checkpoint_round_trip_as_the_reference_utils_record_it(tmp_path, golden_dir):
    """misc/utils.py:49-65 save_model / load_trained_model, as recorded in tests/golden/reference_checkpoint_r18.json:
    kwargs {'backbone': 'resnet18', 'use_rnn': True} rebuild the model with every tensor."""
    import types
    g = json.load(open(os.path.join(golden_dir, 'reference_checkpoint_r18.json')))
    assert g['load_trained_model_restored_every_tensor'] is True
    assert g['kwargs'] == {'backbone': 'resnet18', 'use_rnn': True}
    sd = _sd(4, 'random', True)
    net = HorizonNet('resnet18', True)
    net.load_state_dict(sd, strict=True)
    path = str(tmp_path / 'ck.pth')
    torch.save(OrderedDict({'args': types.SimpleNamespace(lr=1e-4).__dict__,
                            'kwargs': {'backbone': net.backbone, 'use_rnn': net.use_rnn},
                            'state_dict': net.state_dict()}), path)
    ck = torch.load(path, map_location='cpu')
    assert list(ck.keys()) == g['top_level_keys'] and ck['args'] == g['args'] and ck['kwargs'] == g['kwargs']
    got = [[k, list(v.shape), str(v.dtype), float(v.double().sum())] for k, v in ck['state_dict'].items()]
    assert [e[:3] for e in got] == [e[:3] for e in g['state_dict']]
    for e, r in zip(got, g['state_dict']):
        assert e[3] == pytest.approx(r[3], rel=1e-12, abs=1e-9), e[0]
    net2 = HorizonNet(**ck['kwargs'])
    net2.load_state_dict(ck['state_dict'])
    for k, v in net2.state_dict().items():
        assert torch.equal(v, sd[k]), k


# 3x3 conv-row launches with a residual: BasicBlock conv2 of every layer (conv_tc_kernel; layers 1-2 take dx reuse)
def residual_cases():
    from tc_cases import launch
    out = []
    for name, B, H, W, C in (('l1_b2', 2, 128, 256, 64), ('l1_b3', 3, 128, 256, 64), ('l2_b1', 1, 64, 128, 128),
                             ('l2_b2', 2, 64, 128, 128), ('l3_b2', 2, 32, 64, 256), ('l4_b3', 3, 16, 32, 512)):
        c = launch('r18_conv2_' + name, B, H, W, C, C, 3, (1, 1), residual=True)
        c['relu'] = True
        out.append(c)
    return out


@pytest.mark.parametrize('sms', [132, 114])
def test_residual_3x3_launches_are_planned(sms):
    from tc_cases import plan
    for c in residual_cases():
        p = plan(c, sms)
        assert p is not None and p['mode'] == 1 and p['gemm_kernel'] == 0, c['name']
        assert p['dxr'] == (1 if c['W'] >= 128 else 0), c['name']
        assert p['n_tiles'] * p['BN'] == c['Cout'] and p['num_kc'] == 9 * c['Cin'] // 64


# ------------------------------------------------------------------------------- GPU
@pytest.fixture(scope='module')
def _built():
    import __graft_entry__ as entry
    from horizonnet_b200 import _lib
    entry.build()
    _lib.lib()


def _net(sd, use_rnn, tensor_cores=True, train=False):
    net = HorizonNet('resnet18', use_rnn)
    net.load_state_dict(sd, strict=True)
    net.use_tensor_cores(tensor_cores)
    net = net.to(DEV)
    return net.train() if train else net.eval()


def _oracle_on_gpu(sd, x, use_rnn, **kw):
    """The oracle's fp32 arithmetic on the GPU (TF32 off) for the batch-32 comparisons; CPU runs would take minutes."""
    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            return r18.forward({k: v.to(DEV) for k, v in sd.items()}, x.to(DEV), use_rnn=use_rnn, **kw)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags


@pytest.mark.gpu
@pytest.mark.parametrize('tensor_cores', [False, True])
@pytest.mark.parametrize('name,bn,use_rnn', FORWARD_GOLDEN)
def test_resnet18_forward_matches_the_reference_golden(_built, golden_dir, name, bn, use_rnn, tensor_cores):
    g = np.load(os.path.join(golden_dir, name + '.npz'))
    net = _net(_sd(int(g['seed']), bn, use_rnn), use_rnn, tensor_cores)
    x = synthetic_panoramas(int(g['batch']), seed=int(g['x_seed']))
    with torch.no_grad():
        bon, cor = net(x.to(DEV))
    net.check()
    for stage in ('layer1', 'layer4', 'feature', 'rnn_out' if use_rnn else 'mlp_hidden'):
        v = net.debug_stage(stage).cpu()
        assert tuple(v.shape) == tuple(g[stage + '_shape']), stage
        tol = (2e-5 if not tensor_cores else 2e-4) * float(g[stage + '_maxabs']) + 1e-6
        assert np.abs(_sample(v) - g[stage + '_sample']).max() <= tol, stage
    assert tuple(net.debug_stage('feature').shape) == (int(g['batch']), 256, 256)
    tol = 1e-4 * max(1.0, float(max(np.abs(g['bon']).max(), np.abs(g['cor']).max())))
    assert np.abs(bon.cpu().numpy() - g['bon']).max() < tol
    assert np.abs(cor.cpu().numpy() - g['cor']).max() < tol


@pytest.mark.gpu
@pytest.mark.parametrize('tensor_cores', [False, True])
@pytest.mark.parametrize('use_rnn', [True, False])
def test_resnet18_bs32_matches_the_oracle_on_every_sample(_built, use_rnn, tensor_cores):
    sd = _sd(0, 'random', use_rnn)
    net = _net(sd, use_rnn, tensor_cores)
    x = synthetic_panoramas(32, seed=1000)
    with torch.no_grad():
        bon, cor = net(x.to(DEV))
    net.check()
    rb, rc = _oracle_on_gpu(sd, x, use_rnn)
    for r in range(32):
        tol = 1e-4 * max(1.0, float(rb[r].abs().max()), float(rc[r].abs().max()))
        assert (bon[r] - rb[r]).abs().max().item() < tol and (cor[r] - rc[r]).abs().max().item() < tol, r


@pytest.mark.gpu
@pytest.mark.parametrize('use_rnn', [True, False])
def test_resnet18_pipelined_host_and_tta_entry_points(_built, use_rnn, monkeypatch):
    from horizonnet_b200.inference import tta_forward
    from oracle import tta_ref
    sd = _sd(3, 'random', use_rnn)
    net = _net(sd, use_rnn)
    xs = [synthetic_panoramas(b, seed=50 + i).to(DEV) for i, b in enumerate((2, 3, 1, 2))]
    with torch.no_grad():
        ref = [net(x) for x in xs]
        outs = [net.forward_pipelined(x) for x in xs]
        net.flush()
        torch.cuda.synchronize()
    net.check()
    for (rb, rc), (ob, oc) in zip(ref, outs):
        assert torch.equal(rb, ob) and torch.equal(rc, oc)
    hx = [x.cpu().pin_memory() for x in xs[:2]]
    hb, hc = net.forward_host(hx[0])
    assert torch.equal(hb, ref[0][0].cpu()) and torch.equal(hc, ref[0][1].cpu())
    net.submit_host(hx[0])
    net.submit_host(hx[1])
    for i in range(2):
        pb, pc = net.collect_host()
        assert torch.equal(pb, ref[i][0].cpu()) and torch.equal(pc, ref[i][1].cpu()), i
    monkeypatch.setattr(tta_ref.horizonnet_ref, 'forward', lambda sd_, x_, **k: r18.forward(sd_, x_, use_rnn=use_rnn, **k))
    x = synthetic_panoramas(1, seed=102)
    ob, oc = tta_ref.tta_forward(sd, x, flip=True, rotate=[0.25, 0.333])
    tb, tc = tta_forward(net, x, flip=True, rotate=[0.25, 0.333])
    assert np.abs(tb - ob).max() < 1.6e-2 and np.abs(tc - oc).max() < 1e-4


# the four convs conv_tc_kernel does not take: (name, Cin, Cout, H, W) of the input
NARROW = [('ghc0.1', 32, 32, 64, 256), ('ghc0.2', 32, 16, 32, 256), ('ghc0.3', 16, 8, 16, 256), ('ghc1.3', 32, 16, 8, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize('B', [1, 3, 5])
@pytest.mark.parametrize('name,Ci,Co,H,W', NARROW)
def test_narrow_height_reduction_kernel_vs_fp64(_built, name, Ci, Co, H, W, B):
    """hn_conv2d impl 3 (conv_narrow.cu through split planes) against fp64: the split-plane bound of the tensor-core cases,
    every element written (NaN prefill), the halo columns the circular wrap, nothing past the end, nothing negative."""
    import gpu_utils as gu
    from horizonnet_b200 import _lib
    g = torch.Generator().manual_seed(100 * Ci + 10 * Co + B + H)
    x = torch.randn(B, Ci, H, W, generator=g).to(DEV)
    w = (torch.randn(Co, Ci, 3, 3, generator=g) / (Ci * 9) ** 0.5).to(DEV)
    scale, shift = (torch.rand(Co, generator=g) + 0.5).to(DEV), (torch.randn(Co, generator=g) * 0.1).to(DEV)
    Ho = (H - 1) // 2 + 1
    n_out = B * Ho * (W + 2) * Co
    buf = torch.full((n_out + 4096,), float('nan'), device=DEV)
    buf[n_out:] = gu.CANARY
    out = buf[:n_out].view(B, Ho, W + 2, Co)
    xin, wp = gu.to_halo_nhwc(x, 1), gu.pack_weight(w)
    rc = _lib.lib().hn_conv2d(xin.data_ptr(), B, H, W, Ci, 1, wp.data_ptr(), scale.data_ptr(), shift.data_ptr(), None, Co,
                              3, 3, 2, 1, 1, 1, 1, out.data_ptr(), 1, 3, torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, 'hn_conv2d')
    torch.cuda.synchronize()
    assert not torch.isnan(out).any() and bool((buf[n_out:] == gu.CANARY).all())
    assert torch.equal(out[:, :, 0], out[:, :, -2]) and torch.equal(out[:, :, -1], out[:, :, 1])
    y = gu.from_halo_nhwc(out, 1).double()
    assert bool((y >= 0).all())
    ref = gu.conv2d_reference(x.double(), w.double(), scale, shift, (2, 1), 1, 1, True)
    acc = gu._conv_abs(x.double().abs(), w.double().abs(), (2, 1), 1, 1)
    ones = gu._conv_abs(torch.ones_like(x[:1]).double(), w.double().abs(), (2, 1), 1, 1)
    bound = scale.double().abs().view(1, -1, 1, 1) * (gu.C_OPERAND * gu.EPS21 * acc + gu.EPS20 * ones) + \
        gu.EPS21 * ref.abs() + gu.EPS21
    ratio = gu._worst_ratio(y - ref, bound)
    gu.record('narrow_conv.jsonl', {'case': name, 'B': B, 'err_over_bound': ratio})
    assert ratio <= 1.0, ratio
    # the other impls reject nothing they used to take, and the narrow kernel refuses a residual
    assert _lib.lib().hn_conv2d(xin.data_ptr(), B, H, W, Ci, 1, wp.data_ptr(), scale.data_ptr(), shift.data_ptr(),
                                out.data_ptr(), Co, 3, 3, 2, 1, 1, 1, 1, out.data_ptr(), 1, 3, None) != 0


def _run_residual_cases():
    import gpu_utils as gu
    from tc_cases import plan
    for c in residual_cases():
        print(json.dumps({'name': c['name'], 'ratio': gu.run_tc_case(c), 'plan': plan(c, gu.device_sms())}), flush=True)


@pytest.mark.gpu
def test_residual_3x3_launches_vs_fp64_with_dx_reuse_on_and_off(_built):
    runs = {}
    for env in ('1', '0'):
        e = dict(os.environ, HN_TC_DXR=env)
        p = subprocess.run([sys.executable, os.path.abspath(__file__), 'dxr'], env=e, capture_output=True, text=True,
                           timeout=900)
        assert p.returncode == 0, (env, p.stdout[-2000:], p.stderr[-4000:])
        runs[env] = {r['name']: r for r in (json.loads(l) for l in p.stdout.splitlines() if l.startswith('{'))}
    assert len(runs['1']) == len(runs['0']) == len(residual_cases())
    for c in residual_cases():
        on, off = runs['1'][c['name']], runs['0'][c['name']]
        assert on['ratio'] <= 1.0 and off['ratio'] <= 1.0, (c['name'], on['ratio'], off['ratio'])
        assert on['plan']['dxr'] == (1 if c['W'] >= 128 else 0) and off['plan']['dxr'] == 0, c['name']


@pytest.mark.gpu
@pytest.mark.parametrize('tensor_cores', [False, True])
def test_resnet18_train_forward_matches_the_reference_golden(_built, golden_dir, tensor_cores):
    g, sd, x, masks, running = train_golden_r18(golden_dir)
    net = _net(sd, True, tensor_cores, train=True)
    net.dropout_masks_override = tuple(masks)
    with torch.no_grad():
        bon, cor = net(x.to(DEV))
    net.check()
    tol = 3e-4 if tensor_cores else 1e-4
    assert np.abs(bon.cpu().numpy() - g['bon']).max() < tol
    assert np.abs(cor.cpu().numpy() - g['cor']).max() < tol
    after = net.state_dict()
    for k, v in running.items():
        assert torch.allclose(after[k].cpu(), v, rtol=1e-4, atol=1e-5), k
    assert [int(after[k]) for k in after if k.endswith('num_batches_tracked')] == list(g['num_batches_tracked'])


def _relu_masks_of_the_tape(net, use_rnn):
    out = {}
    for i in range(N_UNITS):
        name, y = net.debug_train_unit(i, 0)
        if not name.endswith('downsample.1'):
            out[name] = (y > 0).cpu()
    if not use_rnn:
        out['linear.1'] = (net.debug_stage('mlp_hidden') > 0).cpu()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('tensor_cores', [True, False])
@pytest.mark.parametrize('use_rnn', [True, False])
def test_resnet18_training_step_gradients_match_the_golden_backward(_built, golden_dir, use_rnn, tensor_cores):
    """The training step on the fixture's weights, input, targets and dropout masks: the loss of
    train_backward_r18*.npz, and every parameter's gradient against torch.autograd through the oracle (which that fixture
    pins to the reference) with the device's ReLU decisions (see test_no_rnn_head.py)."""
    g = np.load(os.path.join(golden_dir, f'train_backward{_sfx(use_rnn)}.npz'))
    batch = int(g['batch'])
    sd = _sd(int(g['wseed']), 'random', use_rnn)
    x = synthetic_panoramas(batch, seed=int(g['x_seed']))
    y_bon, y_cor = _golden_targets(g)
    torch.manual_seed(int(g['train_seed']))
    if use_rnn:
        masks = [torch.empty(256, batch, 1024).bernoulli_(0.5).div_(0.5) for _ in range(2)]
        override = tuple(masks)
    else:
        masks = [None, torch.empty(batch, 256, 512).bernoulli_(0.5).div_(0.5)]
        override = (None, masks[1].permute(1, 0, 2).contiguous())
    net = _net(sd, use_rnn, tensor_cores, train=True)
    net.dropout_masks_override = override
    bon, cor = net(x.to(DEV))
    loss = F.l1_loss(bon, y_bon.to(DEV)) + F.binary_cross_entropy_with_logits(cor, y_cor.to(DEV))
    loss.backward()
    net.check()
    names = [k for k, _ in net.named_parameters()]
    assert names == [str(k) for k in g['names']] and len(names) == N_PARAMS[use_rnn]
    assert abs(loss.item() - float(g['loss'])) < 1e-4
    psd = {k: (v.clone().requires_grad_() if k in names else v) for k, v in sd.items()}
    tm = horizonnet_ref.TrainMode(masks=masks, relu_masks=_relu_masks_of_the_tape(net, use_rnn))
    rbon, rcor = r18.forward(psd, x, use_rnn=use_rnn, train=tm)
    rloss = F.l1_loss(rbon, y_bon) + F.binary_cross_entropy_with_logits(rcor, y_cor)
    assert abs(loss.item() - rloss.item()) < 1e-5
    ref = dict(zip(names, torch.autograd.grad(rloss, [psd[k] for k in names])))
    gmax = max(float(v.abs().max()) for v in ref.values())
    assert all(p.grad is not None and p.grad.shape == p.shape for p in net.parameters())
    # a height-reduction conv bias feeds a train-mode BatchNorm, which subtracts it again with the batch mean: its gradient
    # is zero in exact arithmetic, so both sides hold rounding noise and a relative comparison says nothing
    zero = {k for k in names if k.startswith('reduce_height_module') and k.endswith('0.1.bias')}
    for k, p in net.named_parameters():
        if k in zero:
            assert float((p.grad.cpu() - ref[k]).abs().max()) <= 1e-5 * gmax, k
    worst = sorted(((float((p.grad.cpu() - ref[k]).abs().max()) / (float(ref[k].abs().max()) + 1e-4 * gmax), k)
                    for k, p in net.named_parameters() if k not in zero), reverse=True)
    assert worst[0][0] < 5e-3, worst[:8]
    head = [e for e in worst if e[1].startswith(('linear', 'bi_rnn.weight_ih_l0'))]
    assert head[0][0] < 5e-3, head


if __name__ == '__main__':
    assert sys.argv[1:] == ['dxr'], sys.argv
    import __graft_entry__ as entry
    entry.build()
    _run_residual_cases()
