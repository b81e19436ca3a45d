"""The training step's backward, one step at a time, against an fp64 replay of the device's own tape (tests/train_replay.py).

The whole-step tests (test_gpu_parity.py, test_no_rnn_head.py, test_resnet18.py) compare every parameter gradient with
autograd through the CPU fp32 oracle; the oracle runs its own forward, and train-mode BatchNorm on a small batch
amplifies the forward's rounding difference, so those bounds are 5e-3.  Here every backward step is recomputed in fp64
from the inputs the device gave that step (its tape: z, y and d(loss)/d(y) of every conv unit, the dropout masks, the
MLP's hidden layer), so each comparison carries the rounding of one step and the bound can be close to the kernel tests'.

CPU (unmarked): the replay is checked against itself first -- its graph against the pinned oracles' forward, and the
chained per-unit backward against torch.autograd through the whole fp64 forward.
"""
import pytest
import torch

import gpu_utils as gu
import train_replay as tr
from horizonnet_b200 import _lib
from horizonnet_b200.model import HorizonNet
from horizonnet_b200.weights import synthetic_panoramas, synthetic_state_dict
from oracle import horizonnet_norn_ref, horizonnet_ref, horizonnet_r18_ref

DEV = 'cuda:0'
# the frozen configuration: list_blocks()[0:2] in eval mode like train.py --freeze_earlier_blocks 1 (the stem and
# layer1: 11 BatchNorm2d in resnet50), plus one height-reduction unit, whose conv bias then has the frozen gradient
# scale * sum(g) instead of 0
FROZEN_PREFIXES = ('feature_extractor.encoder.bn1', 'feature_extractor.encoder.layer1.')
FROZEN_GHC = 'reduce_height_module.ghc_lst.1.layer.0.layers.1'
RUNNING = ('.running_mean', '.running_var', '.num_batches_tracked')


def _params(sd):
    return [k for k, v in sd.items() if v.is_floating_point() and not k.endswith(RUNNING)]


def _fp64(sd, device='cpu'):
    return {k: (v.to(device=device, dtype=torch.float64) if v.is_floating_point() else v) for k, v in sd.items()}


def _oracle(backbone, use_rnn, sd, x, masks, frozen):
    """The pinned oracle's fp64 train-mode forward with the library-layout dropout masks."""
    tm = horizonnet_ref.TrainMode(masks=masks if use_rnn else [None, masks[1].permute(1, 0, 2)], frozen=frozen)
    if backbone == 'resnet18':
        return horizonnet_r18_ref.forward(sd, x, use_rnn=use_rnn, dtype=torch.float64, train=tm)
    mod = horizonnet_ref if use_rnn else horizonnet_norn_ref
    return mod.forward(sd, x, dtype=torch.float64, train=tm)


def _masks(use_rnn, B, gen):
    width = 1024 if use_rnn else 512
    ms = [torch.empty(256, B, width).bernoulli_(0.5, generator=gen).mul_(2.0) for _ in range(2)]
    return [m.double() for m in ms] if use_rnn else [None, ms[1].double()]


# ------------------------------------------------------------------------------------------------ CPU self-check
def _frozen_like_the_gpu_test(units):
    return {u.name for u in units if u.name.startswith(FROZEN_PREFIXES)} | {FROZEN_GHC}


@pytest.mark.parametrize('backbone,use_rnn,frozen', [('resnet18', True, False), ('resnet18', False, True),
                                                     ('resnet50', True, True), ('resnet50', False, False)])
def test_replay_reproduces_the_oracle_and_autograd(backbone, use_rnn, frozen):
    """At batch 1 in fp64: the replay's graph walked forward gives the pinned oracle's bon / cor, and the chained per-unit
    replay driven by a fixed (dbon, dcor) gives what torch.autograd gives through that whole forward -- every parameter,
    every unit's d(y), d(stem y).  frozen: the BatchNorm2d units the frozen GPU configuration runs in eval mode."""
    sd = synthetic_state_dict(5, 'random', use_rnn=use_rnn, backbone=backbone)
    x = synthetic_panoramas(1, seed=7)
    gen = torch.Generator().manual_seed(3)
    masks = _masks(use_rnn, 1, gen)
    dbon = torch.randn(1, 2, 1024, generator=gen, dtype=torch.float64) / 1024
    dcor = torch.randn(1, 1, 1024, generator=gen, dtype=torch.float64) / 1024
    units, gout = tr.build_graph(backbone)
    frozen = _frozen_like_the_gpu_test(units) if frozen else set()
    sd64 = _fp64(sd)
    names = _params(sd)
    psd = dict(sd64)
    for k in names:
        psd[k] = sd64[k].clone().requires_grad_()
    image = tr.normalised_image(x)

    # (1) tape-producing forward == the oracle
    _, ys = tr.forward_tape(units, psd, image, frozen)
    bon, cor, hidden = tr.head_forward([ys[g] for g in gout], psd, use_rnn, masks)
    with torch.no_grad():
        rbon, rcor = _oracle(backbone, use_rnn, sd, x, masks, frozen)
    for got, ref in ((bon, rbon), (cor, rcor)):
        assert float((got.detach() - ref).abs().max()) <= 1e-12 * float(ref.abs().max())

    # (2) autograd through the whole forward
    whole = torch.autograd.grad((bon, cor), [psd[k] for k in names] + ys, (dbon, dcor))
    ref_p = dict(zip(names, whole[:len(names)]))
    ref_dy = whole[len(names):]
    ys = [y.detach() for y in ys]
    hidden_mask = None if hidden is None else hidden.detach() > 0
    del bon, cor, hidden, whole

    # (3) the chained replay: head, then every unit from the accumulated d(y)
    _, _, _, dgout, got_p = tr.head_step([ys[g] for g in gout], sd64, use_rnn, masks, hidden_mask, dbon, dcor)
    got_dy = {g: d for g, d in zip(gout, dgout)}
    pooled = tr.pool(ys[0])

    def act(k):
        return image if k == 'image' else pooled if k == 'pool' else ys[k]

    def report(kind, key, v):
        if kind == 'unit':
            u = units[key]
            got_p[u.wkey], got_p[u.name + '.weight'], got_p[u.name + '.bias'] = v['weight'], v['gamma'], v['beta']
            if u.bkey:
                got_p[u.bkey] = v['bias']
        elif kind == 'dy':
            got_dy[key] = v
        else:
            got_dy[0] = v[1]

    tr.walk_backward(units, gout, sd64, frozen, act, dgout, lambda i, acc: acc, report)
    assert sorted(got_p) == sorted(names)
    assert sorted(got_dy) == list(range(len(units)))
    gmax = max(float(v.abs().max()) for v in ref_p.values())
    for k in names:
        err = float((got_p[k] - ref_p[k]).abs().max())
        if k.endswith('0.1.bias') and k[:-len('0.1.bias')] + '1' not in frozen:
            # conv bias in front of a train-mode BatchNorm: 0 up to rounding on both sides
            assert err <= 1e-10 * gmax, k
        else:
            assert err <= 1e-10 * float(ref_p[k].abs().max()), (k, err)
    for i, u in enumerate(units):
        err = float((got_dy[i] - ref_dy[i]).abs().max())
        assert err <= 1e-10 * float(ref_dy[i].abs().max()), (u.name, err)


def test_graph_follows_the_backbone_specs():
    """Unit order and wiring: the stem reads the image, layer1.0 reads the max-pool, the last unit of each block carries
    the identity (or the downsample), and every scale ends in ghc_lst.{s}.layer.3."""
    for backbone, n, ds in (('resnet50', 69, 4), ('resnet18', 36, 3)):
        units, gout = tr.build_graph(backbone)
        assert len(units) == n
        assert units[0].src == 'image' and units[0].k == 7 and units[0].stride == (2, 2)
        assert [u.name for u in units if u.name.endswith('downsample.1')] == \
            [f'feature_extractor.encoder.layer{li}.0.downsample.1' for li in range(5 - ds, 5)]
        assert sum(u.src == 'pool' or u.res == 'pool' for u in units) == 2
        assert [units[g].name for g in gout] == [f'reduce_height_module.ghc_lst.{s}.layer.3.layers.1' for s in range(4)]
        assert all(u.relu != u.name.endswith('downsample.1') for u in units)
        assert all(u.res is None or units.index(u) > (u.res if u.res != 'pool' else 0) for u in units)


# ------------------------------------------------------------------------------------------------ GPU replay
# Bounds per section, by the kernels that computed the device side: (fp32 CUDA-core kernels, tensor-core kernels), about
# 4x the worst ratio measured over the configurations below on an H100 80GB HBM3 (700 W power limit), and never above the
# kernel tests' ceilings (2e-5 fp32, 1e-4 split-fp16 tensor cores and the head).  Measured worst of three runs (fp32,
# tensor cores):  forward 6.1e-6, 2.8e-6   head 1.2e-6, 2.4e-6   unit 4.9e-6, 1.7e-6   wgrad 3.3e-6, 7.0e-5
#                 stem 1.9e-6, 2.4e-6   maxpool 1.0e-6, 1.2e-6   pool_sum 2.2e-8, 1.4e-7
# wgrad (the conv weight gradients after the stem) takes the tensor-core bound with tensor cores on: the training step
# then runs them on wgrad_tc.cu wherever that kernel takes the shape.  Its worst ratios (3.4e-5 to 7.0e-5) are all at
# layer-1 / layer2.0 weight gradients, whose sums run over 2-3 x 32768 non-negative input pixels, 16-24 x the 4096 of
# its kernel test; 4x of 7.0e-5 would exceed the ceiling, so the bound is the ceiling.  unit = the data gradient a unit
# sends to its producers and its BatchNorm (and frozen conv-bias) gradients.
BOUND = {
    'forward':  (2e-5, 1.2e-5),
    'head':     (5e-6, 1e-5),
    'unit':     (2e-5, 7e-6),
    'wgrad':    (1.4e-5, 1e-4),
    'stem':     (7e-6, 1e-5),
    'maxpool':  (4e-6, 5e-6),
    'pool_sum': (8e-8, 6e-7),
}

CONFIGS = [
    # backbone, use_rnn, tensor_cores, batch, frozen blocks
    pytest.param('resnet50', True, True, 3, False, id='r50-lstm-tc-wgradtc-b3'),
    pytest.param('resnet50', True, False, 2, False, id='r50-lstm-fp32-b2'),
    pytest.param('resnet50', True, False, 1, False, id='r50-lstm-fp32-b1'),
    pytest.param('resnet50', True, True, 2, True, id='r50-lstm-tc-frozen-b2'),
    pytest.param('resnet50', False, True, 3, False, id='r50-mlp-tc-b3'),
    pytest.param('resnet18', True, True, 2, False, id='r18-lstm-tc-b2'),
    pytest.param('resnet18', False, False, 3, False, id='r18-mlp-fp32-b3'),
]


@pytest.fixture(scope='module')
def _built():
    import __graft_entry__ as entry
    entry.build()
    _lib.lib()


def slice_ratios(got, ref, keep=None, activation=True):
    """{slice: max |got - ref| / max |ref|} for the whole tensor and, for an NCHW activation, each image and the first /
    last column and row; each slice is normalised by its own max |ref| floored at 1e-3 of the tensor's.  keep: compare
    only where it is True."""
    err = (got - ref).abs()
    mag = ref.abs()
    if keep is not None:
        err, mag = err * keep, mag * keep
    top = float(mag.max())

    def r(e, m):
        e = float(e.max())
        den = max(float(m.max()), 1e-3 * top)
        return 0.0 if e == 0 else (e / den if den > 0 else float('inf'))
    out = {'all': r(err, mag)}
    if activation and ref.dim() == 4:
        for b in range(ref.shape[0]):
            out[f'image{b}'] = r(err[b], mag[b])
        for name, ix in (('col0', (Ellipsis, 0)), ('colW', (Ellipsis, -1)),
                         ('row0', (Ellipsis, 0, slice(None))), ('rowH', (Ellipsis, -1, slice(None)))):
            out[name] = r(err[ix], mag[ix])
    return out


class Judge:
    """Collects every comparison of one configuration: records it, keeps the worst ratio per section, lists violations."""

    def __init__(self, config, tensor_cores):
        self.config, self.tc = config, int(tensor_cores)
        self.worst, self.failures = {}, []

    def bound(self, section):
        return BOUND[section][self.tc]

    def __call__(self, section, unit, tensor, got, ref, keep=None, activation=True):
        assert got.shape == ref.shape, (section, unit, tensor, tuple(got.shape), tuple(ref.shape))
        ratios = slice_ratios(got.double(), ref, keep, activation)
        self.add(section, unit, tensor, ratios)

    def add(self, section, unit, tensor, ratios):
        gu.record('train_replay.jsonl', {'config': self.config, 'section': section, 'unit': unit, 'tensor': tensor,
                                         'ratios': ratios})
        sl, worst = max(ratios.items(), key=lambda kv: kv[1])
        if worst > self.worst.get(section, (-1.0,))[0]:
            self.worst[section] = (worst, unit, tensor, sl)
        bound = self.bound(section)
        if not worst <= bound:
            self.failures.append(f'{section}: {unit}: {tensor} [{sl}] {worst:.3e} > {bound:.0e}')

    def exact_zero(self, unit, tensor, got):
        if not bool((got == 0).all()):
            self.failures.append(f'unit: {unit}: {tensor} must be exactly 0, max |g| = {float(got.abs().max()):.3e}')


def judge_step(net, backbone, use_rnn, sd, x, bon, cor, r_bon, r_cor, frozen_bn, judge, device):
    """Every comparison of one training step of net (after its backward) with the fp64 replay of its tape."""
    B = x.shape[0]
    units, gout = tr.build_graph(backbone)
    assert [net.debug_train_unit(i, 0)[0] for i in range(len(units))] == [u.name for u in units]
    with pytest.raises(RuntimeError):
        net.debug_train_unit(len(units), 0)
    grads = {k: p.grad for k, p in net.named_parameters()}
    assert all(g is not None for g in grads.values())
    sd64 = _fp64(sd, device)
    masks = [None if m is None else m.double() for m in net.dropout_masks(net.last_dropout_seed, B, device)]
    dbon, dcor = r_bon.to(device, torch.float64), r_cor.to(device, torch.float64)

    def dev(i, what):
        return net.debug_train_unit(i, what)[1].double()

    image = tr.normalised_image(x)
    pooled = tr.pool(dev(0, 0))

    def act(k):
        return image if k == 'image' else pooled if k == 'pool' else dev(k, 0)

    # ---- the sequence adjoint and the head, from the device's four height-reduction outputs
    hidden_dev = None if use_rnn else net.debug_stage('mlp_hidden').double()
    rbon, rcor, rhidden, dgout, hgrads = tr.head_step([act(g) for g in gout], sd64, use_rnn, masks,
                                                      None if use_rnn else hidden_dev > 0, dbon, dcor)
    judge('head', 'head', 'bon', bon, rbon)
    judge('head', 'head', 'cor', cor, rcor)
    if not use_rnn:
        judge('head', 'head', 'mlp_hidden', hidden_dev, rhidden)
    for g, d in zip(gout, dgout):
        judge('head', units[g].name, 'd(y)', dev(g, 2), d)
    for k, g in hgrads.items():
        judge('head', k, 'grad', grads[k], g, activation=False)

    # ---- every conv unit, in the backward's order, driven by the device's own d(y)
    def report(kind, key, v):
        if kind == 'unit':
            u = units[key]
            judge('forward', u.name, 'z', dev(key, 1), v['z'])
            judge('forward', u.name, 'y', dev(key, 0), v['y'])
            section = 'stem' if key == 0 else 'unit'
            judge('stem' if key == 0 else 'wgrad', u.name, u.wkey, grads[u.wkey], v['weight'], activation=False)
            judge(section, u.name, 'gamma', grads[u.name + '.weight'], v['gamma'])
            judge(section, u.name, 'beta', grads[u.name + '.bias'], v['beta'])
            if u.bkey and u.name in frozen_bn:
                judge(section, u.name, u.bkey, grads[u.bkey], v['bias'], activation=False)
            elif u.bkey:                     # zeroed analytically: the batch mean subtracts the bias again
                judge.exact_zero(u.name, u.bkey, grads[u.bkey])
        elif kind == 'dy':
            judge('unit', units[key].name, 'd(y) from its consumers', dev(key, 2), v)
        else:
            dpool, dstem = v
            got = dev(0, 2)
            judge('maxpool', units[0].name, 'd(y) where y > 0', got, dstem, keep=act(0) > 0)
            # conservation per (image, channel): every d(pool) element lands on exactly one stem pixel, zeros included;
            # relative to sum |d pool|, the scale of the rounding of the sums
            scale = dpool.abs().sum((2, 3))
            cons = (got.sum((2, 3)) - dpool.sum((2, 3))).abs() / scale.clamp_min(1e-3 * float(scale.max()))
            judge.add('pool_sum', units[0].name, 'sum of d(y) - sum of d(pool)', {'all': float(cons.max())})

    tr.walk_backward(units, gout, sd64, frozen_bn, act, dgout, lambda i, acc: dev(i, 2), report)


@pytest.mark.gpu
@pytest.mark.parametrize('backbone,use_rnn,tensor_cores,batch,frozen', CONFIGS)
def test_training_step_matches_the_fp64_replay_of_its_tape(_built, request, backbone, use_rnn, tensor_cores, batch, frozen):
    """One net.train() step with dropout on and a linear loss (so d(bon), d(cor) are known exactly), then every step of
    its backward against the fp64 replay built from the device's own inputs to that step: each unit's forward (z, y),
    the sequence adjoint and the head, each conv unit's parameter gradients and the data gradient it sends to its
    producers, the max-pool routing and the stem."""
    config = request.node.callspec.id
    B = batch
    sd = synthetic_state_dict(11, 'random', use_rnn=use_rnn, backbone=backbone)
    net = HorizonNet(backbone, use_rnn)
    net.load_state_dict(sd, strict=True)
    net.use_tensor_cores(tensor_cores)
    net = net.to(DEV).train()
    if frozen:
        blocks = net.feature_extractor.list_blocks()
        for i in range(2):
            for m in blocks[i]:
                m.eval()
        net.get_submodule(FROZEN_GHC).eval()
    frozen_bn = {n for n, m in net.named_modules() if isinstance(m, torch.nn.BatchNorm2d) and not m.training}
    assert len(frozen_bn) == (12 if frozen else 0)
    assert frozen_bn == (_frozen_like_the_gpu_test(tr.build_graph(backbone)[0]) if frozen else set())
    x = synthetic_panoramas(B, seed=100 + B).to(DEV)
    gen = torch.Generator().manual_seed(17)
    r_bon = torch.randn(B, 2, 1024, generator=gen) / (B * 1024)
    r_cor = torch.randn(B, 1, 1024, generator=gen) / (B * 1024)
    torch.manual_seed(23)
    bon, cor = net(x)
    loss = (bon * r_bon.to(DEV)).sum() + (cor * r_cor.to(DEV)).sum()
    loss.backward()
    net.check()

    judge = Judge(config, tensor_cores)
    judge_step(net, backbone, use_rnn, sd, x, bon.detach(), cor.detach(), r_bon, r_cor, frozen_bn, judge, DEV)
    summary = {s: {'ratio': w[0], 'unit': w[1], 'tensor': w[2], 'slice': w[3], 'bound': judge.bound(s)}
               for s, w in judge.worst.items()}
    gu.record('train_replay_worst.jsonl', {'config': config, 'worst': summary})
    print(config, summary)
    assert set(judge.worst) == set(BOUND)
    assert not judge.failures, (f'{len(judge.failures)} comparisons out of bounds, first {judge.failures[0]}\n' +
                                '\n'.join(judge.failures[:25]))
