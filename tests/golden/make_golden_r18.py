"""Mint the golden fixtures of HorizonNet('resnet18', use_rnn) -- both heads -- by running the REAL reference (read-only,
/root/reference) on CPU.

Run in the build container only (the GPU box has no /root/reference):
    python tests/golden/make_golden_r18.py
Outputs (committed): state_dict_keys_r18{,_norn}.json, forward_r18_identity.npz (seed 0, identity BN, batch 2),
forward_r18_randombn.npz and forward_r18_norn_randombn.npz (seed 1, random BN, batch 1), train_r18.npz (train-mode
forward of the bi-LSTM model), train_backward_r18{,_norn}.npz (loss.backward()), reference_checkpoint_r18.json
(misc/utils.py save_model / load_trained_model with our class).  The sampling, the seeds and the mask replay are the ones
of make_golden.py / make_golden_norn.py, which this script imports.  One more shim: the reference passes ResNet50_Weights
to every ResNet builder (model.py:68), which current torchvision rejects for resnet18, so resnet18 is forced to
weights=None like resnet50 is.
"""
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg                     # noqa: E402  (shim 1: torchvision resnet50 with weights=None; reference model)
import make_golden_norn as mgn               # noqa: E402

import torchvision.models as tvm             # noqa: E402
_orig18 = tvm.resnet18
tvm.resnet18 = lambda *a, **k: _orig18(weights=None)     # shim 3: resnet18 without ImageNet weights (model.py:68)

from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas   # noqa: E402
from oracle import horizonnet_ref, horizonnet_r18_ref as oracle                  # noqa: E402

HERE = mg.HERE
N_PARAMS = {True: 142, False: 128}


def ref_net(use_rnn):
    return mg.ref_model.HorizonNet('resnet18', use_rnn)


def sfx(use_rnn):
    return '_r18' if use_rnn else '_r18_norn'


def masks_of(use_rnn, batch):
    """The dropout masks the reference consumes after torch.manual_seed(TRAIN_SEED), in the oracle's layout."""
    return mg.replay_dropout_masks(mg.TRAIN_SEED, batch) if use_rnn else mgn.replay_mask(mg.TRAIN_SEED, batch)


def golden_state_dict_keys(use_rnn):
    net = ref_net(use_rnn)
    keys = [[k, list(v.shape), str(v.dtype)] for k, v in net.state_dict().items()]
    json.dump(keys, open(os.path.join(HERE, f'state_dict_keys{sfx(use_rnn)}.json'), 'w'))
    n_bn = sum(isinstance(m, torch.nn.BatchNorm2d) for m in net.modules())
    print('state_dict keys', sfx(use_rnn), len(keys), 'parameter tensors:', len(list(net.parameters())),
          'parameters:', sum(p.numel() for p in net.parameters()), 'BatchNorm2d:', n_bn)


def golden_forward(name, seed, bn, batch, use_rnn):
    torch.manual_seed(0)
    net = ref_net(use_rnn).eval()
    sd = synthetic_state_dict(seed, bn, use_rnn=use_rnn, backbone='resnet18')
    net.load_state_dict(sd, strict=True)          # proves the key layout is the reference's
    x = synthetic_panoramas(batch, seed=100 + seed)
    stages = {}
    net.feature_extractor.register_forward_hook(
        lambda m, i, o: stages.update({f'layer{j + 1}': o[j] for j in range(4)}))
    net.reduce_height_module.register_forward_hook(lambda m, i, o: stages.update(feature=o))
    if use_rnn:
        net.bi_rnn.register_forward_hook(lambda m, i, o: stages.update(rnn_out=o[0]))
    else:
        net.linear[1].register_forward_hook(lambda m, i, o: stages.update(mlp_hidden=o.clone()))
    with torch.no_grad():
        bon, cor = net(x)
    out = dict(bon=bon.numpy(), cor=cor.numpy(), seed=seed, batch=batch, x_seed=100 + seed)
    for k, v in stages.items():
        s, mean_abs, max_abs = mg.sample(v)
        out[k + '_sample'] = s
        out[k + '_meanabs'] = mean_abs
        out[k + '_maxabs'] = max_abs
        out[k + '_shape'] = np.array(v.shape)
    fname = f'forward_r18_{name}.npz' if use_rnn else f'forward_r18_norn_{name}.npz'
    np.savez_compressed(os.path.join(HERE, fname), **out)
    print(fname, 'bon', float(bon.abs().max()), 'cor', float(cor.abs().max()),
          {k: float(v.abs().max()) for k, v in stages.items()})


def golden_train(batch=2, wseed=1):
    """net.train(); net(x) of the bi-LSTM model in fp32: outputs, moved running statistics and the two replayed dropout
    masks; asserts that the oracle fed with those masks reproduces the reference to 2e-5, which proves the replay."""
    net = ref_net(True)
    sd = synthetic_state_dict(wseed, 'random', backbone='resnet18')
    net.load_state_dict(sd, strict=True)
    net.train()
    x = synthetic_panoramas(batch, seed=200 + wseed)
    torch.manual_seed(mg.TRAIN_SEED)
    with torch.no_grad():
        bon, cor = net(x)
    after = net.state_dict()
    masks = masks_of(True, batch)
    tm = horizonnet_ref.TrainMode(masks=masks)
    with torch.no_grad():
        o_bon, o_cor = oracle.forward(sd, x, train=tm)
    err = max(float((o_bon - bon).abs().max()), float((o_cor - cor).abs().max()))
    assert err < 2e-5, f'mask replay / oracle restatement differs from the reference: {err}'
    bn_keys = [k for k in sd if k.endswith('running_mean') or k.endswith('running_var')]
    for k in bn_keys:
        assert not torch.equal(after[k], sd[k]), k
        assert torch.allclose(tm.running[k], after[k], rtol=1e-5, atol=1e-6), k
    nbt = [int(after[k]) for k in after if k.endswith('num_batches_tracked')]
    out = dict(bon=bon.numpy(), cor=cor.numpy(), wseed=wseed, x_seed=200 + wseed, batch=batch, train_seed=mg.TRAIN_SEED,
               momentum=np.float64(0.1), frozen=np.array([], dtype='U'),
               masks_bits=np.packbits(np.stack([(m > 0).numpy() for m in masks]).reshape(-1)),
               running=np.concatenate([after[k].numpy().reshape(-1) for k in bn_keys]).astype(np.float32),
               num_batches_tracked=np.array(nbt))
    np.savez_compressed(os.path.join(HERE, 'train_r18.npz'), **out)
    print('train_r18: oracle-vs-reference', err, 'bon', float(bon.abs().max()), 'cor', float(cor.abs().max()))


def golden_train_backward(use_rnn, batch=2, wseed=1, n=256):
    """loss.backward() as train.py drives it (:249, :52, :53-56 L1 + BCE-with-logits, :278), fp32: the loss and, per
    parameter, |grad| max, |grad| mean and n strided samples; asserts that torch.autograd through the oracle (same masks)
    reproduces them."""
    net = ref_net(use_rnn)
    sd = synthetic_state_dict(wseed, 'random', use_rnn=use_rnn, backbone='resnet18')
    net.load_state_dict(sd, strict=True)
    net.train()
    x = synthetic_panoramas(batch, seed=200 + wseed)
    g = torch.Generator().manual_seed(77)
    y_bon, y_cor = torch.rand(batch, 2, 1024, generator=g) - 0.5, torch.rand(batch, 1, 1024, generator=g)
    torch.manual_seed(mg.TRAIN_SEED)
    bon, cor = net(x)
    loss = F.l1_loss(bon, y_bon) + F.binary_cross_entropy_with_logits(cor, y_cor)
    loss.backward()
    names = [k for k, p in net.named_parameters() if p.requires_grad]
    grads = {k: p.grad for k, p in net.named_parameters()}
    assert len(names) == N_PARAMS[use_rnn] and all(v is not None for v in grads.values())
    masks = masks_of(use_rnn, batch)
    psd = {k: (v.clone().requires_grad_() if k in grads else v) for k, v in sd.items()}
    o_bon, o_cor = oracle.forward(psd, x, use_rnn=use_rnn, train=horizonnet_ref.TrainMode(masks=masks))
    o_loss = F.l1_loss(o_bon, y_bon) + F.binary_cross_entropy_with_logits(o_cor, y_cor)
    o_grads = dict(zip(names, torch.autograd.grad(o_loss, [psd[k] for k in names])))
    gmax = max(float(v.abs().max()) for v in grads.values())
    worst = max(float((o_grads[k] - grads[k]).abs().max()) / (float(grads[k].abs().max()) + 1e-4 * gmax) for k in names)
    assert abs(loss.item() - o_loss.item()) < 1e-6 and worst < 1e-3, (loss.item(), o_loss.item(), worst)

    def strided(t):
        flat = t.detach().reshape(-1)
        stride = max(1, flat.numel() // n)
        out = np.zeros(n, np.float32)
        v = flat[::stride][:n].numpy()
        out[:v.size] = v
        return out
    np.savez_compressed(os.path.join(HERE, f'train_backward{sfx(use_rnn)}.npz'), names=np.array(names, dtype='U'),
                        loss=np.float64(loss.item()), frozen=np.array([], dtype='U'),
                        absmax=np.array([float(grads[k].abs().max()) for k in names]),
                        absmean=np.array([float(grads[k].abs().double().mean()) for k in names]),
                        samples=np.stack([strided(grads[k]) for k in names]), n=n, wseed=wseed, x_seed=200 + wseed,
                        y_seed=77, batch=batch, train_seed=mg.TRAIN_SEED)
    print('train_backward', sfx(use_rnn), ': loss', loss.item(), 'parameters with a gradient:', len(names),
          'oracle autograd vs reference, worst tensor (rel. to its max):', worst)


def golden_checkpoint():
    """What the reference's misc/utils.py:49-65 save_model writes for our HorizonNet('resnet18', True) and whether its
    load_trained_model restores it."""
    from misc import utils as ref_utils
    from horizonnet_b200.model import HorizonNet
    sd = synthetic_state_dict(4, 'random', backbone='resnet18')
    net = HorizonNet('resnet18', True)
    net.load_state_dict(sd, strict=True)
    path = os.path.join(tempfile.mkdtemp(), 'ck.pth')
    ref_utils.save_model(net, path, types.SimpleNamespace(lr=1e-4))
    ck = torch.load(path, map_location='cpu')
    net2 = ref_utils.load_trained_model(HorizonNet, path)
    ok = list(net2.state_dict().keys()) == list(sd.keys()) and all(torch.equal(v, sd[k]) for k, v in net2.state_dict().items())
    out = {'what': "checkpoint written by the reference's misc/utils.py save_model(net, path, args(lr=1e-4)) for "
                   "HorizonNet('resnet18', True) loaded with synthetic_state_dict(4, 'random', backbone='resnet18'), and "
                   "whether its load_trained_model(HorizonNet, path) restored it",
           'top_level_keys': list(ck.keys()), 'args': ck['args'], 'kwargs': ck['kwargs'],
           'state_dict': [[k, list(v.shape), str(v.dtype), float(v.double().sum())] for k, v in ck['state_dict'].items()],
           'load_trained_model_restored_every_tensor': ok}
    json.dump(out, open(os.path.join(HERE, 'reference_checkpoint_r18.json'), 'w'), indent=0)
    print('checkpoint golden written, reference load restored every tensor:', ok)


if __name__ == '__main__':
    golden_state_dict_keys(True)
    golden_state_dict_keys(False)
    golden_forward('identity', seed=0, bn='identity', batch=2, use_rnn=True)
    golden_forward('randombn', seed=1, bn='random', batch=1, use_rnn=True)
    golden_forward('randombn', seed=1, bn='random', batch=1, use_rnn=False)
    golden_train()
    golden_train_backward(True)
    golden_train_backward(False)
    golden_checkpoint()
