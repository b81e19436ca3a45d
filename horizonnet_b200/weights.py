"""Deterministic synthetic checkpoints in the reference's 448-key layout (434 keys with the MLP head).

There is no network on any box, so no trained checkpoint exists; parity tests, smoke() and
bench.py all need *the same* random-init weights on the build container (where the real reference
is run to mint the golden outputs) and on the GPU box (where it is absent).  Weights are therefore
drawn with ``numpy.random.RandomState`` (bit-reproducible across machines) and follow the
distributions the reference's constructor uses (torchvision kaiming-normal fan_out for the encoder,
PyTorch defaults elsewhere, head bias per reference model.py:231-233).

``bn='identity'`` reproduces a fresh reference model (BN gamma=1, beta=0, mean=0, var=1);
``bn='random'`` draws non-trivial BN statistics so that BN folding is actually exercised.
"""
from collections import OrderedDict
import math
import numpy as np
import torch

from ._spec import state_dict_spec, HEAD_BIAS


def synthetic_state_dict(seed=0, bn='identity', use_rnn=True, backbone='resnet50'):
    """use_rnn=False: the MLP-head layout.  Its encoder and height-reduction tensors come first in the key order and are
    drawn identically, so they equal the bi-LSTM model's for the same seed; then linear.0 ~ U(+-1/sqrt(c_last)) (weight and
    bias, PyTorch's nn.Linear default), linear.3.weight ~ U(+-1/sqrt(512)), linear.3.bias = the reference's init.
    backbone: the key layout of that encoder (horizonnet_b200._spec.BACKBONES), drawn by the same rules."""
    rs = np.random.RandomState(seed)
    sd = OrderedDict()
    for key, (shape, kind) in state_dict_spec(use_rnn, backbone).items():
        if kind == 'enc_conv':
            co, ci, kh, kw = shape
            a = rs.standard_normal(shape) * math.sqrt(2.0 / (co * kh * kw))
        elif kind == 'ghc_conv':
            co, ci, kh, kw = shape
            bound = 1.0 / math.sqrt(ci * kh * kw)
            a = rs.uniform(-bound, bound, shape)
        elif kind == 'ghc_bias':
            # fan_in of the matching conv = 9 * Cin; Cin is recovered from the weight just drawn
            w = sd[key[:-len('bias')] + 'weight']
            bound = 1.0 / math.sqrt(w.shape[1] * 9)
            a = rs.uniform(-bound, bound, shape)
        elif kind == 'rnn':
            bound = 1.0 / math.sqrt(512)
            a = rs.uniform(-bound, bound, shape)
        elif kind == 'mlp_weight':
            bound = 1.0 / math.sqrt(shape[1])
            a = rs.uniform(-bound, bound, shape)
        elif kind == 'mlp_bias':
            bound = 1.0 / math.sqrt(sd[key[:-len('bias')] + 'weight'].shape[1])
            a = rs.uniform(-bound, bound, shape)
        elif kind == 'head_weight':
            bound = 1.0 / math.sqrt(shape[1])
            a = rs.uniform(-bound, bound, shape)
        elif kind == 'head_bias':
            a = np.asarray(HEAD_BIAS)
        elif kind == 'bn_weight':
            a = np.ones(shape) if bn == 'identity' else rs.uniform(0.5, 1.5, shape)
        elif kind == 'bn_bias':
            a = np.zeros(shape) if bn == 'identity' else rs.standard_normal(shape) * 0.1
        elif kind == 'bn_mean':
            a = np.zeros(shape) if bn == 'identity' else rs.standard_normal(shape) * 0.1
        elif kind == 'bn_var':
            a = np.ones(shape) if bn == 'identity' else rs.uniform(0.5, 1.5, shape)
        elif kind == 'bn_count':
            sd[key] = torch.zeros((), dtype=torch.int64)
            continue
        else:
            raise KeyError(kind)
        sd[key] = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    return sd


def synthetic_panoramas(batch, seed=1, channels=3):
    """x ~ U[0,1) in the reference's NCHW fp32 input format (inference.py:196-200)."""
    rs = np.random.RandomState(seed)
    return torch.from_numpy(rs.random_sample((batch, channels, 512, 1024)).astype(np.float32))
