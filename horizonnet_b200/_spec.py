"""Architecture spec of the model family on the hot path: a ResNet encoder (``resnet50`` or ``resnet18``) + bi-LSTM
head, or + per-column MLP head.

Everything here is derived from the *checkpoint layout* the reference writes
(reference misc/utils.py:49-58, model.py:189-246) -- resnet50: 448 keys with the bi-LSTM, 434 with the MLP head
(``use_rnn=False``); resnet18: 250 and 236 -- probed from the reference and pinned by tests/golden/state_dict_keys*.json.
The C library builds the same graph from the same key names (csrc/model.cu), so this file is the single Python-side
description of names + shapes.
"""
from collections import OrderedDict

# backbone -> (block kind, blocks per layer, planes per layer, expansion); torchvision resnet.py
BACKBONES = {
    'resnet50': ('bottleneck', (3, 4, 6, 3), (64, 128, 256, 512), 4),
    'resnet18': ('basic', (2, 2, 2, 2), (64, 128, 256, 512), 1),
}
PANO_H, PANO_W = 512, 1024          # reference model.py:255 hard-wires the input size
STEP_COLS = 4                        # model.py:194
SEQ_LEN = PANO_W // STEP_COLS        # 256 LSTM steps
RNN_HIDDEN = 512                     # model.py:195
OUT_SCALE = 8                        # model.py:193
HEAD_BIAS = [-1.0] * 4 + [-0.478] * 4 + [0.425] * 4   # model.py:231-233


def _bn(prefix, c, out):
    out[prefix + '.weight'] = ((c,), 'bn_weight')
    out[prefix + '.bias'] = ((c,), 'bn_bias')
    out[prefix + '.running_mean'] = ((c,), 'bn_mean')
    out[prefix + '.running_var'] = ((c,), 'bn_var')
    out[prefix + '.num_batches_tracked'] = ((), 'bn_count')


def state_dict_spec(use_rnn=True, backbone='resnet50'):
    """OrderedDict key -> (shape, kind) in the reference's own key order; use_rnn=False: the MLP head of
    model.py:234-243 (linear.0 = Linear(c_last, 512), linear.3 = Linear(512, 12)) instead of bi_rnn + linear."""
    kind, nblocks, planes_l, expansion = BACKBONES[backbone]
    out = OrderedDict()
    enc = 'feature_extractor.encoder.'
    out[enc + 'conv1.1.weight'] = ((64, 3, 7, 7), 'enc_conv')       # wrapped by LR_PAD -> '.1'
    _bn(enc + 'bn1', 64, out)
    inplanes = 64
    for li, (nblk, planes) in enumerate(zip(nblocks, planes_l), start=1):
        for b in range(nblk):
            p = f'{enc}layer{li}.{b}.'
            stride = 2 if (b == 0 and li > 1) else 1
            if kind == 'bottleneck':
                out[p + 'conv1.weight'] = ((planes, inplanes, 1, 1), 'enc_conv')
                _bn(p + 'bn1', planes, out)
                out[p + 'conv2.1.weight'] = ((planes, planes, 3, 3), 'enc_conv')   # wrapped 3x3
                _bn(p + 'bn2', planes, out)
                out[p + 'conv3.weight'] = ((planes * expansion, planes, 1, 1), 'enc_conv')
                _bn(p + 'bn3', planes * expansion, out)
            else:                                                    # BasicBlock: two wrapped 3x3, the stride on conv1
                out[p + 'conv1.1.weight'] = ((planes, inplanes, 3, 3), 'enc_conv')
                _bn(p + 'bn1', planes, out)
                out[p + 'conv2.1.weight'] = ((planes, planes, 3, 3), 'enc_conv')
                _bn(p + 'bn2', planes, out)
            if b == 0 and (stride != 1 or inplanes != planes * expansion):
                out[p + 'downsample.0.weight'] = ((planes * expansion, inplanes, 1, 1), 'enc_conv')
                _bn(p + 'downsample.1', planes * expansion, out)
            inplanes = planes * expansion
    for s, c in enumerate(encoder_channels(backbone)):
        chans = [c, c // 2, c // 2, c // 4, c // OUT_SCALE]
        for j in range(4):
            p = f'reduce_height_module.ghc_lst.{s}.layer.{j}.layers.'
            out[p + '0.1.weight'] = ((chans[j + 1], chans[j], 3, 3), 'ghc_conv')
            out[p + '0.1.bias'] = ((chans[j + 1],), 'ghc_bias')
            _bn(p + '1', chans[j + 1], out)
    width = c_last(backbone)
    if not use_rnn:
        out['linear.0.weight'] = ((RNN_HIDDEN, width), 'mlp_weight')
        out['linear.0.bias'] = ((RNN_HIDDEN,), 'mlp_bias')
        out['linear.3.weight'] = ((3 * STEP_COLS, RNN_HIDDEN), 'head_weight')
        out['linear.3.bias'] = ((3 * STEP_COLS,), 'head_bias')
        return out
    for layer in range(2):
        for suffix in ('', '_reverse'):
            in_sz = width if layer == 0 else 2 * RNN_HIDDEN
            out[f'bi_rnn.weight_ih_l{layer}{suffix}'] = ((4 * RNN_HIDDEN, in_sz), 'rnn')
            out[f'bi_rnn.weight_hh_l{layer}{suffix}'] = ((4 * RNN_HIDDEN, RNN_HIDDEN), 'rnn')
            out[f'bi_rnn.bias_ih_l{layer}{suffix}'] = ((4 * RNN_HIDDEN,), 'rnn')
            out[f'bi_rnn.bias_hh_l{layer}{suffix}'] = ((4 * RNN_HIDDEN,), 'rnn')
    out['linear.weight'] = ((3 * STEP_COLS, 2 * RNN_HIDDEN), 'head_weight')
    out['linear.bias'] = ((3 * STEP_COLS,), 'head_bias')
    return out


def encoder_channels(backbone='resnet50'):
    _, _, planes, expansion = BACKBONES[backbone]
    return tuple(p * expansion for p in planes)     # resnet50: 256, 512, 1024, 2048; resnet18: 64, 128, 256, 512


def c_last(backbone='resnet50'):
    """Width of the feature sequence (model.py:218): each scale ends with C/8 channels at H = 8, 4, 2, 1."""
    return sum(c * h for c, h in zip(encoder_channels(backbone), (8, 4, 2, 1))) // OUT_SCALE   # 1024 / 256
