"""HorizonNet('resnet50', use_rnn=False): the per-column MLP head of reference model.py:234-243 (what train.py --no_rnn
builds), through every layer: spec, synthetic weights, oracle, module surface (CPU) and the library's eval forward,
entry points, train-mode forward and training step (GPU).  Fixtures: tests/golden/*_norn.* (make_golden_norn.py);
checker: oracle/horizonnet_norn_ref.py (with horizonnet_ref.TrainMode for train mode)."""
import ctypes
import hashlib
import json
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from horizonnet_b200 import _lib
from horizonnet_b200._spec import state_dict_spec, HEAD_BIAS
from horizonnet_b200.model import HorizonNet
from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas
from oracle import horizonnet_ref, horizonnet_norn_ref

DEV = 'cuda:0'
N_PARAMS_NORN = 227                       # 241 - 16 bi_rnn.* - linear.weight/bias + linear.0/3 weight/bias


def _sample(t, n=4096):
    flat = t.detach().reshape(-1).double().numpy()
    return flat[::max(1, flat.size // n)][:n].astype(np.float32)


def _digest(sd):
    h = hashlib.sha256()
    for k, v in sd.items():
        h.update(k.encode())
        h.update(v.numpy().tobytes())
    return h.hexdigest()


def train_golden_norn(golden_dir):
    """tests/golden/train_norn.npz -> (g, sd, x, mask [B,256,512] in the reference's layout, moved running statistics)."""
    g = np.load(os.path.join(golden_dir, 'train_norn.npz'))
    B = int(g['batch'])
    bits = np.unpackbits(g['masks_bits'])[:B * 256 * 512].reshape(B, 256, 512)
    mask = torch.from_numpy(bits.astype(np.float32) * 2.0)
    sd = synthetic_state_dict(int(g['wseed']), 'random', use_rnn=False)
    x = synthetic_panoramas(B, seed=int(g['x_seed']))
    bn_keys = [k for k in sd if k.endswith('running_mean') or k.endswith('running_var')]
    running, off = {}, 0
    for k in bn_keys:
        n = sd[k].numel()
        running[k] = torch.from_numpy(g['running'][off:off + n].copy())
        off += n
    return g, sd, x, mask, running


# ------------------------------------------------------------------------------- CPU: spec, weights, oracle, module
def test_spec_matches_the_reference_no_rnn_layout(golden_dir):
    ref = json.load(open(os.path.join(golden_dir, 'state_dict_keys_norn.json')))
    spec = state_dict_spec(use_rnn=False)
    assert len(spec) == len(ref) == 434
    for (k, shape, _), (k2, (s2, _)) in zip(ref, spec.items()):
        assert k == k2 and tuple(shape) == tuple(s2)
    n_params = sum(int(np.prod(s)) for s, kind in spec.values() if kind not in ('bn_mean', 'bn_var', 'bn_count'))
    assert n_params == 69489708
    assert [k for k in spec if k.startswith('linear')] == ['linear.0.weight', 'linear.0.bias', 'linear.3.weight',
                                                          'linear.3.bias']
    rnn = state_dict_spec()
    assert [k for k in rnn if not k.startswith(('bi_rnn', 'linear'))] == [k for k in spec if not k.startswith('linear')]


def test_synthetic_weights_of_the_rnn_model_are_unchanged_and_shared_with_the_mlp_model():
    # sha256 over (key, bytes) of every tensor, taken from the commit before the MLP head existed: every golden file of the
    # bi-LSTM model depends on these draws
    expected = {(0, 'identity'): 'e03039b4c8183b5f61e3cefa4b0e56cb98dfc836fb03260c8c6f1afcd14b9203',
                (1, 'random'): '91cb41fbb74d1296e1f229b6c3cf02674832ce17916875f64f4bfe21a4853e88'}
    for (seed, bn), digest in expected.items():
        rnn = synthetic_state_dict(seed, bn)
        assert _digest(rnn) == digest, (seed, bn)
        mlp = synthetic_state_dict(seed, bn, use_rnn=False)
        assert list(mlp) == list(state_dict_spec(use_rnn=False))
        for k, v in mlp.items():
            if not k.startswith('linear'):
                assert torch.equal(v, rnn[k]), k
        assert torch.equal(mlp['linear.3.bias'], torch.tensor(HEAD_BIAS, dtype=torch.float32))
        for k, bound in (('linear.0.weight', 1024 ** -0.5), ('linear.0.bias', 1024 ** -0.5), ('linear.3.weight', 512 ** -0.5)):
            assert 0.9 * bound < float(mlp[k].abs().max()) <= bound, k


@pytest.mark.parametrize('name,bn', [('identity', 'identity'), ('randombn', 'random')])
def test_oracle_matches_the_reference_no_rnn_forward(golden_dir, name, bn):
    g = np.load(os.path.join(golden_dir, f'forward_norn_{name}.npz'))
    sd = synthetic_state_dict(int(g['seed']), bn, use_rnn=False)
    x = synthetic_panoramas(int(g['batch']), seed=int(g['x_seed']))
    with torch.no_grad():
        bon, cor, stages = horizonnet_norn_ref.forward(sd, x, return_stages=True)
    assert np.abs(bon.numpy() - g['bon']).max() < 2e-5
    assert np.abs(cor.numpy() - g['cor']).max() < 2e-5
    assert 'rnn_out' not in stages and 'mlp_hidden' in stages
    for k, v in stages.items():
        assert tuple(v.shape) == tuple(g[k + '_shape']), k
        assert np.abs(_sample(v) - g[k + '_sample']).max() <= 2e-6 * float(g[k + '_maxabs']) + 1e-6, k


def test_oracle_matches_the_reference_no_rnn_train_forward(golden_dir):
    """One mask, torch.empty(B,256,512).bernoulli_(0.5).div_(0.5) after manual_seed: the oracle fed with it, and the
    oracle drawing it with F.dropout from torch's generator, both reproduce the reference under net.train()."""
    g, sd, x, mask, running = train_golden_norn(golden_dir)
    tm = horizonnet_ref.TrainMode(masks=[None, mask])
    with torch.no_grad():
        bon, cor = horizonnet_norn_ref.forward(sd, x, train=tm)
    assert np.abs(bon.numpy() - g['bon']).max() < 2e-5 and np.abs(cor.numpy() - g['cor']).max() < 2e-5
    for k, v in running.items():
        assert torch.allclose(tm.running[k], v, rtol=1e-5, atol=1e-6), k
    assert g['num_batches_tracked'].sum() == 69
    torch.manual_seed(int(g['train_seed']))
    with torch.no_grad():
        bon2, cor2 = horizonnet_norn_ref.forward(sd, x, train=horizonnet_ref.TrainMode())
    assert torch.equal(bon2, bon) and torch.equal(cor2, cor)


def test_oracle_backward_matches_the_reference_no_rnn_backward(golden_dir):
    g = np.load(os.path.join(golden_dir, 'train_backward_norn.npz'))
    batch, n = int(g['batch']), int(g['n'])
    sd = synthetic_state_dict(int(g['wseed']), 'random', use_rnn=False)
    x = synthetic_panoramas(batch, seed=int(g['x_seed']))
    gen = torch.Generator().manual_seed(int(g['y_seed']))
    y_bon, y_cor = torch.rand(batch, 2, 1024, generator=gen) - 0.5, torch.rand(batch, 1, 1024, generator=gen)
    torch.manual_seed(int(g['train_seed']))
    mask = torch.empty(batch, 256, 512).bernoulli_(0.5).div_(0.5)
    names = [str(k) for k in g['names']]
    assert len(names) == N_PARAMS_NORN
    psd = {k: (v.clone().requires_grad_() if k in names else v) for k, v in sd.items()}
    bon, cor = horizonnet_norn_ref.forward(psd, x, train=horizonnet_ref.TrainMode(masks=[None, mask]))
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
    assert worst < 2e-4, worst


def test_module_surface_of_the_no_rnn_model(golden_dir):
    keys = [k for k, _, _ in json.load(open(os.path.join(golden_dir, 'state_dict_keys_norn.json')))]
    net = HorizonNet('resnet50', False)
    assert list(net.state_dict().keys()) == keys
    net.load_state_dict(synthetic_state_dict(0, 'identity', use_rnn=False), strict=True)
    assert not hasattr(net, 'bi_rnn') and not hasattr(net, 'drop_out')
    assert net.use_rnn is False and net.backbone == 'resnet50'
    kinds = [type(m) for m in net.linear.children()]
    assert kinds == [torch.nn.Linear, torch.nn.ReLU, torch.nn.Dropout, torch.nn.Linear]
    assert net.linear[0].in_features == 1024 and net.linear[0].out_features == 512 and net.linear[2].p == 0.5
    fresh = HorizonNet('resnet50', False)
    assert torch.equal(fresh.linear[3].bias, torch.tensor(HEAD_BIAS, dtype=torch.float32))
    assert sum(p.numel() for p in fresh.parameters()) == 69489708
    assert len(list(fresh.named_parameters())) == N_PARAMS_NORN

    def blocks(m):
        return [[type(c).__name__ for c in grp] for grp in m.feature_extractor.list_blocks()]
    assert blocks(fresh) == blocks(HorizonNet('resnet50', True))
    # the MLP model is in train mode after construction (dropout of linear[2] and BatchNorm), in eval mode after .eval()
    assert fresh._train_mode_active() and not fresh.eval()._train_mode_active()
    for backbone in ('resnet34', 'resnet101', 'densenet121'):
        for use_rnn in (False, True):
            with pytest.raises(NotImplementedError):
                HorizonNet(backbone, use_rnn)


def test_no_rnn_checkpoint_round_trip_through_the_real_reference_utils(tmp_path, golden_dir):
    """The reference's save_model / load_trained_model (misc/utils.py:49-65) on the MLP model, as recorded in
    tests/golden/reference_checkpoint_norn.json: kwargs {'backbone': 'resnet50', 'use_rnn': False} rebuild it."""
    import types
    g = json.load(open(os.path.join(golden_dir, 'reference_checkpoint_norn.json')))
    assert g['load_trained_model_restored_every_tensor'] is True
    assert g['kwargs'] == {'backbone': 'resnet50', 'use_rnn': False}
    sd = synthetic_state_dict(4, 'random', use_rnn=False)
    net = HorizonNet('resnet50', False)
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
    assert net2.use_rnn is False and not hasattr(net2, 'bi_rnn')
    for k, v in net2.state_dict().items():
        assert torch.equal(v, sd[k]), k


def _layer1_launch(B):
    """MLP layer 1 as the library launches it: a 1x1 conv over the 256*B rows of SEQ, K = 1024 -> 512, fp32 output."""
    from tc_cases import launch
    c = launch(f'mlp1_b{B}', 1, 1, 256 * B, 1024, 512, 1, (1, 1), 0, 0, out_f32=True)
    c['relu'] = True
    return c


@pytest.mark.parametrize('sms', [132, 114])
@pytest.mark.parametrize('B', [1, 2, 3, 8, 32])
def test_layer1_launch_is_planned_by_the_tensor_core_kernel(B, sms):
    from tc_cases import plan
    p = plan(_layer1_launch(B), sms)
    assert p is not None
    assert p['M'] == 256 * B and p['mode'] == 0 and p['gemm_kernel'] == 0      # conv_tc_kernel in GEMM-row mode
    assert p['num_kc'] * 64 == 1024 and p['n_tiles'] * p['BN'] == 512
    assert 1 <= p['grid'] <= sms and p['num_tiles'] >= p['grid']


# ------------------------------------------------------------------------------- GPU
def _net(sd, tensor_cores=True):
    net = HorizonNet('resnet50', False).eval()
    net.load_state_dict(sd, strict=True)
    net.use_tensor_cores(tensor_cores)
    return net.to(DEV)


def _train_net(sd, tensor_cores=True):
    net = HorizonNet('resnet50', False)
    net.load_state_dict(sd, strict=True)
    net.use_tensor_cores(tensor_cores)
    return net.to(DEV).train()


@pytest.fixture(scope='module')
def _built():
    import __graft_entry__ as entry
    entry.build()
    _lib.lib()


@pytest.mark.gpu
@pytest.mark.parametrize('tensor_cores', [False, True])
@pytest.mark.parametrize('name,bn', [('identity', 'identity'), ('randombn', 'random')])
def test_no_rnn_forward_matches_the_reference_golden(_built, golden_dir, name, bn, tensor_cores):
    g = np.load(os.path.join(golden_dir, f'forward_norn_{name}.npz'))
    sd = synthetic_state_dict(int(g['seed']), bn, use_rnn=False)
    net = _net(sd, tensor_cores)
    x = synthetic_panoramas(int(g['batch']), seed=int(g['x_seed']))
    with torch.no_grad():
        bon, cor = net(x.to(DEV))
    net.check()
    for stage in ('feature', 'mlp_hidden'):
        v = net.debug_stage(stage).cpu()
        assert tuple(v.shape) == tuple(g[stage + '_shape']), stage
        flat = v.reshape(-1).numpy()
        got = flat[::max(1, flat.size // 4096)][:4096]
        tol = (2e-5 if not tensor_cores else 2e-4) * float(g[stage + '_maxabs']) + 1e-6
        assert np.abs(got - g[stage + '_sample']).max() <= tol, stage
    ref_max = max(np.abs(g['bon']).max(), np.abs(g['cor']).max())
    tol = 1e-4 * max(1.0, float(ref_max))
    assert np.abs(bon.cpu().numpy() - g['bon']).max() < tol
    assert np.abs(cor.cpu().numpy() - g['cor']).max() < tol
    with pytest.raises(RuntimeError, match='rnn_out'):
        net.debug_stage('rnn_out')


@pytest.mark.gpu
def test_no_rnn_bs32_rows_equal_bs1_bitwise_and_match_oracle(_built):
    sd = synthetic_state_dict(0, 'random', use_rnn=False)
    net = _net(sd)
    x = synthetic_panoramas(32, seed=1000)
    with torch.no_grad():
        bon32, cor32 = net(x.to(DEV))
    net.check()
    for r in (0, 13, 31):
        with torch.no_grad():
            b1, c1 = net(x[r:r + 1].to(DEV))
            rb, rc = horizonnet_norn_ref.forward(sd, x[r:r + 1])
        assert torch.equal(bon32[r:r + 1], b1) and torch.equal(cor32[r:r + 1], c1), r
        tol = 1e-4 * max(1.0, float(rb.abs().max()), float(rc.abs().max()))
        assert (b1.cpu() - rb).abs().max().item() < tol and (c1.cpu() - rc).abs().max().item() < tol, r


@pytest.mark.gpu
def test_no_rnn_pipelined_host_and_pipelined_host_entry_points_equal_forward(_built):
    sd = synthetic_state_dict(3, 'random', use_rnn=False)
    net = _net(sd)
    xs = [synthetic_panoramas(b, seed=50 + i).to(DEV) for i, b in enumerate((2, 3, 1, 2))]
    with torch.no_grad():
        ref = [net(x) for x in xs]
        outs = [net.forward_pipelined(x) for x in xs]
        net.flush()
        torch.cuda.synchronize()
        for (rb, rc), (ob, oc) in zip(ref, outs):
            assert torch.equal(rb, ob) and torch.equal(rc, oc)
        o1 = net.forward_pipelined(xs[0])
        p2 = net(xs[1])
        o3 = net.forward_pipelined(xs[2])
        net.flush()
        torch.cuda.synchronize()
    net.check()
    assert torch.equal(o1[0], ref[0][0]) and torch.equal(p2[0], ref[1][0]) and torch.equal(o3[1], ref[2][1])
    hx = [x.cpu().pin_memory() for x in xs[:2]]
    hb, hc = net.forward_host(hx[0])
    assert torch.equal(hb, ref[0][0].cpu()) and torch.equal(hc, ref[0][1].cpu())
    net.submit_host(hx[0])
    net.submit_host(hx[1])
    for i in range(2):
        pb, pc = net.collect_host()
        assert torch.equal(pb, ref[i][0].cpu()) and torch.equal(pc, ref[i][1].cpu()), i


@pytest.mark.gpu
def test_no_rnn_tta_matches_the_oracle(_built, monkeypatch):
    from horizonnet_b200.inference import tta_forward
    from oracle import tta_ref
    monkeypatch.setattr(tta_ref.horizonnet_ref, 'forward', horizonnet_norn_ref.forward)   # tta_ref driven by the MLP oracle
    sd = synthetic_state_dict(2, 'random', use_rnn=False)
    net = _net(sd)
    x = synthetic_panoramas(1, seed=102)
    ob, oc = tta_ref.tta_forward(sd, x, flip=True, rotate=[0.25, 0.333])
    tb, tc = tta_forward(net, x, flip=True, rotate=[0.25, 0.333])
    assert np.abs(tb - ob).max() < 1.6e-2 and np.abs(tc - oc).max() < 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize('B', [2, 32])
def test_layer1_launch_relu_fp32_output_vs_fp64(_built, B):
    """hn_conv2d impl 2 (conv_tc_kernel<128>, fp32 epilogue) with ReLU on the MLP layer-1 shape: within the split-plane
    bound of test_tc_kernels.py, every element written (NaN prefill, canary), and nothing negative."""
    import gpu_utils as gu
    c = _layer1_launch(B)
    ratio = gu.run_tc_case(c, DEV)
    gu.record('no_rnn_layer1.jsonl', {'B': B, 'err_over_bound': ratio})
    assert ratio <= 1.0, ratio
    x, w, scale, shift, _ = gu.tc_case_inputs(c, DEV)
    y, raw = gu.conv2d(x, w, scale, shift, (1, 1), 0, 0, True, impl=2, in_halo=0, out_halo=0)
    assert not torch.isnan(raw).any() and bool((raw >= 0).all()) and bool((raw == 0).any())


@pytest.mark.gpu
def test_k512_head_kernel_vs_fp64_and_zero_weight_gives_the_bias_exactly(_built):
    sd = synthetic_state_dict(4, 'random', use_rnn=False)
    net = _net(sd)
    x = synthetic_panoramas(2, seed=3).to(DEV)
    with torch.no_grad():
        bon, cor = net(x)
    hidden = net.debug_stage('mlp_hidden').cpu().double()              # [B, 256, 512]: exactly the head kernel's input
    out = hidden @ sd['linear.3.weight'].double().t() + sd['linear.3.bias'].double()
    out = out.view(2, 256, 3, 4).permute(0, 2, 1, 3).reshape(2, 3, 1024)
    acc = hidden.abs() @ sd['linear.3.weight'].double().abs().t()
    bound = 1e-6 * acc.view(2, 256, 3, 4).permute(0, 2, 1, 3).reshape(2, 3, 1024) + 1e-7
    assert bool(((cor.cpu().double() - out[:, :1]).abs() <= bound[:, :1]).all())
    assert bool(((bon.cpu().double() - out[:, 1:]).abs() <= bound[:, 1:]).all())
    sd['linear.3.weight'] = torch.zeros_like(sd['linear.3.weight'])
    net = _net(sd)
    with torch.no_grad():
        bon, cor = net(x)
    assert torch.all(cor == -1.0)
    assert torch.all(bon[:, 0] == torch.tensor(-0.478)) and torch.all(bon[:, 1] == torch.tensor(0.425))


@pytest.mark.gpu
@pytest.mark.parametrize('tensor_cores', [False, True])
def test_no_rnn_train_forward_matches_the_reference_golden(_built, golden_dir, tensor_cores):
    g, sd, x, mask, running = train_golden_norn(golden_dir)
    net = _train_net(sd, tensor_cores)
    net.dropout_masks_override = (None, mask.permute(1, 0, 2).contiguous())      # library rows t*B + b
    with torch.no_grad():
        bon, cor = net(x.to(DEV))
    net.check()
    # tensor cores: measured 1.6e-4 on an H100 (outputs up to 1.5): batch statistics over 2 panoramas amplify the split-fp16
    # rounding, and unlike the bi-LSTM head no saturating gate compresses it on the way out; the fp32 kernels stay in 1e-4
    tol = 3e-4 if tensor_cores else 1e-4
    assert np.abs(bon.cpu().numpy() - g['bon']).max() < tol
    assert np.abs(cor.cpu().numpy() - g['cor']).max() < tol
    after = net.state_dict()
    for k, v in running.items():
        assert torch.allclose(after[k].cpu(), v, rtol=1e-4, atol=1e-5), k
    assert [int(after[k]) for k in after if k.endswith('num_batches_tracked')] == list(g['num_batches_tracked'])


@pytest.mark.gpu
def test_no_rnn_philox_mask_is_seeded_and_train_forward_refuses_rnn_dropout(_built):
    sd = synthetic_state_dict(5, 'random', use_rnn=False)
    x = synthetic_panoramas(2, seed=31)
    net = _train_net(sd)
    torch.manual_seed(77)
    with torch.no_grad():
        bon, cor = net(x.to(DEV))
    seed = net.last_dropout_seed
    none, m = net.dropout_masks(seed, 2, DEV)
    assert none is None and m.shape == (256, 2, 512)
    assert set(torch.unique(m).tolist()) == {0.0, 2.0} and abs(float((m > 0).float().mean()) - 0.5) < 0.005
    tm = horizonnet_ref.TrainMode(masks=[None, m.permute(1, 0, 2).cpu()])
    with torch.no_grad():
        rbon, rcor = horizonnet_norn_ref.forward(sd, x, train=tm)
    # tensor-core train-mode forward, see test_no_rnn_train_forward_matches_the_reference_golden (measured 1.5e-4)
    assert (bon.cpu() - rbon).abs().max().item() < 3e-4 and (cor.cpu() - rcor).abs().max().item() < 3e-4
    net2 = _train_net(sd)
    torch.manual_seed(77)
    with torch.no_grad():
        bon2, cor2 = net2(x.to(DEV))
        bon3, _ = net2(x.to(DEV))
    assert torch.equal(bon2, bon) and torch.equal(cor2, cor) and not torch.equal(bon3, bon)
    # the C entry point refuses an LSTM dropout for a model without an LSTM
    lib = _lib.lib()
    h = net._handles[0]
    xd = x.to(DEV)
    out_b, out_c = torch.empty(2, 2, 1024, device=DEV), torch.empty(2, 1, 1024, device=DEV)
    n_bn = lib.hn_model_num_bn(h['ptr'])
    flags = (ctypes.c_ubyte * n_bn)(*([1] * n_bn))
    factors = (ctypes.c_double * n_bn)(*([-1.0] * n_bn))
    rc = lib.hn_train_forward(h['ptr'], xd.data_ptr(), 2, 3, out_b.data_ptr(), out_c.data_ptr(), flags, factors, n_bn, 1,
                              0.5, 0.5, None, None, None)
    assert rc != 0 and 'rnn_dropout must be 0' in lib.hn_last_error().decode()


def _oracle_grads(sd, x, mask, names, y_bon, y_cor, relu_masks=None, frozen=()):
    psd = {k: (v.clone().requires_grad_() if k in names else v) for k, v in sd.items()}
    tm = horizonnet_ref.TrainMode(masks=[None, mask], relu_masks=relu_masks, frozen=frozen)
    rbon, rcor = horizonnet_norn_ref.forward(psd, x, train=tm)
    rloss = F.l1_loss(rbon, y_bon) + F.binary_cross_entropy_with_logits(rcor, y_cor)
    return rbon.detach(), rloss.item(), dict(zip(names, torch.autograd.grad(rloss, [psd[k] for k in names])))


def _relu_masks_of_the_tape(net):
    """The device's ReLU decisions: the 69 conv units of the tape and the MLP hidden layer (linear[1]).  Two fp32 forwards
    differ by ~1e-4 deep in the net, which flips near-zero pre-activations; each flip moves a gradient element by its full
    value, so the comparison takes the decisions from the device (see test_gpu_parity.py)."""
    out = {}
    for i in range(69):
        name, y = net.debug_train_unit(i, 0)
        if not name.endswith('downsample.1'):
            out[name] = (y > 0).cpu()
    out['linear.1'] = (net.debug_stage('mlp_hidden') > 0).cpu()
    return out


def _worst(net, ref):
    gmax = max(float(v.abs().max()) for v in ref.values())
    out = []
    for k, p in net.named_parameters():
        if k not in ref:
            assert p.grad is None, k
            continue
        assert p.grad is not None and p.grad.shape == p.shape, k
        out.append((float((p.grad.cpu() - ref[k]).abs().max()) / (float(ref[k].abs().max()) + 1e-4 * gmax), k))
    return sorted(out, reverse=True)


@pytest.mark.gpu
@pytest.mark.parametrize('tensor_cores', [True, False])
def test_no_rnn_training_step_gradients_match_autograd_of_the_oracle(_built, tensor_cores):
    sd = synthetic_state_dict(1, 'random', use_rnn=False)
    x = synthetic_panoramas(2, seed=41)
    gen = torch.Generator().manual_seed(9)
    y_bon, y_cor = torch.rand(2, 2, 1024, generator=gen) - 0.5, torch.rand(2, 1, 1024, generator=gen)
    net = _train_net(sd, tensor_cores)
    torch.manual_seed(11)
    bon, cor = net(x.to(DEV))
    loss = F.l1_loss(bon, y_bon.to(DEV)) + F.binary_cross_entropy_with_logits(cor, y_cor.to(DEV))
    loss.backward()
    net.check()
    prof = net.train_profile()
    assert prof['lstm'] == 0.0 and prof['head'] > 0.0
    mask = net.dropout_masks(net.last_dropout_seed, 2, DEV)[1].permute(1, 0, 2).cpu()
    names = [k for k, _ in net.named_parameters()]
    assert len(names) == N_PARAMS_NORN
    rbon, rloss, ref = _oracle_grads(sd, x, mask, names, y_bon, y_cor)
    tol = 3e-4 if tensor_cores else 1e-4             # see test_no_rnn_train_forward_matches_the_reference_golden
    assert (bon.detach().cpu() - rbon).abs().max().item() < tol and abs(loss.item() - rloss) < 1e-5
    assert _worst(net, ref)[0][0] < 0.5
    _, rloss2, ref2 = _oracle_grads(sd, x, mask, names, y_bon, y_cor, _relu_masks_of_the_tape(net))
    assert abs(loss.item() - rloss2) < 1e-5
    same = _worst(net, ref2)
    assert same[0][0] < 5e-3, same[:8]
    head = [e for e in same if e[1].startswith('linear')]
    assert len(head) == 4 and head[0][0] < 1e-3, head


@pytest.mark.gpu
def test_no_rnn_training_step_with_frozen_blocks_and_a_loop_that_lowers_the_loss(_built):
    sd = synthetic_state_dict(2, 'random', use_rnn=False)
    x = synthetic_panoramas(2, seed=43)
    gen = torch.Generator().manual_seed(10)
    y_bon, y_cor = torch.rand(2, 2, 1024, generator=gen) - 0.5, torch.rand(2, 1, 1024, generator=gen)
    net = _train_net(sd)
    blocks = net.feature_extractor.list_blocks()
    for i in range(2):                                                  # train.py --freeze_earlier_blocks 1
        for m in blocks[i]:
            m.eval()
            for p in m.parameters():
                p.requires_grad = False
    frozen = [n for n, m in net.named_modules() if isinstance(m, torch.nn.BatchNorm2d) and not m.training]
    assert len(frozen) == 11
    bon, cor = net(x.to(DEV))
    loss = F.l1_loss(bon, y_bon.to(DEV)) + F.binary_cross_entropy_with_logits(cor, y_cor.to(DEV))
    loss.backward()
    net.check()
    mask = net.dropout_masks(net.last_dropout_seed, 2, DEV)[1].permute(1, 0, 2).cpu()
    live = [k for k, p in net.named_parameters() if p.requires_grad]
    _, rloss, ref = _oracle_grads(sd, x, mask, live, y_bon, y_cor, _relu_masks_of_the_tape(net), frozen)
    assert abs(loss.item() - rloss) < 1e-5
    worst = _worst(net, ref)
    assert worst[0][0] < 5e-3, worst[:8]
    # train.py:216-223 + :272-281 on one fixed batch: Adam steps lower the loss, eval afterwards matches the oracle
    sd = synthetic_state_dict(3, 'random', use_rnn=False)
    xd = synthetic_panoramas(2, seed=47).to(DEV)
    yb, yc = y_bon.to(DEV), y_cor.to(DEV)
    net = _train_net(sd)
    opt = torch.optim.Adam(net.parameters(), lr=1e-3, betas=(0.9, 0.999))
    losses = []
    for _ in range(5):
        torch.manual_seed(0)
        opt.zero_grad()
        bon, cor = net(xd)
        loss = F.l1_loss(bon, yb) + F.binary_cross_entropy_with_logits(cor, yc)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    net.check()
    assert all(np.isfinite(losses)) and losses[-1] < losses[0] - 0.02, losses
    net.eval()
    with torch.no_grad():
        ebon, ecor = net(xd)
        rbon, rcor = horizonnet_norn_ref.forward({k: v.cpu() for k, v in net.state_dict().items()}, xd.cpu())
    assert (ebon.cpu() - rbon).abs().max().item() < 2e-4 and (ecor.cpu() - rcor).abs().max().item() < 2e-4


@pytest.mark.gpu
def test_no_rnn_profile_counts_both_mlp_layers_as_the_linear_head(_built):
    sd = synthetic_state_dict(0, 'identity', use_rnn=False)
    net = _net(sd)
    x = synthetic_panoramas(2, seed=5).to(DEV)
    with torch.no_grad():
        net(x)
        net.set_profile(True)
        net.read_profile(reset=True)
        net(x)
    prof = net.read_profile(reset=True)
    net.set_profile(False)
    assert len(prof) == 8
    assert prof['lstm_input_projection'] == (0.0, 0.0, 0) and prof['lstm_recurrence'] == (0.0, 0.0, 0)
    ms, flops, n = prof['linear_head']
    assert n == 2 and ms > 0 and flops == pytest.approx(2.0 * 256 * 2 * (1024 * 512 + 512 * 12))
