"""TEST INFRASTRUCTURE ONLY -- CPU oracle for ``HorizonNet('resnet18', use_rnn)``, both heads.

The encoder is torchvision's resnet18 topology (reference model.py:66-68 builds it; torchvision/models/resnet.py
BasicBlock): two 3x3 convs per block, both wrapped by LR_PAD (model.py:42-55), the stride on conv1, a 1x1 downsample on
block 0 of layers 2-4.  Everything after the encoder -- the height reduction (model.py:148-156), the concat
(:175-178), the bi-LSTM head (:264-269) or the per-column MLP head (:270-275) -- is the one of oracle/horizonnet_ref.py and
oracle/horizonnet_norn_ref.py, with a feature sequence 256 wide instead of 1024 (64 + 128 + 256 + 512 channels / 8 at
H = 8, 4, 2, 1).

Pinned against the real reference by tests/golden/*_r18* (tests/golden/make_golden_r18.py); tests/test_resnet18.py
asserts this restatement reproduces them.  Train mode takes a ``horizonnet_ref.TrainMode`` (masks [256, B, 1024] for the
bi-LSTM head, (None, [B, 256, 512]) for the MLP head, as in those two oracles).
"""
import torch
import torch.nn.functional as F

from .horizonnet_ref import X_MEAN, X_STD, _bn, _circ_conv, _relu, bi_lstm, global_height_conv

BLOCKS = (2, 2, 2, 2)


def _basic_block(x, sd, p, stride, has_ds, tm=None):
    # torchvision resnet.py BasicBlock.forward
    out = _relu(_bn(_circ_conv(x, sd[p + 'conv1.1.weight'], None, stride, 1, 1), sd, p + 'bn1', tm), p + 'bn1', tm)
    out = _bn(_circ_conv(out, sd[p + 'conv2.1.weight'], None, 1, 1, 1), sd, p + 'bn2', tm)
    if has_ds:
        x = _bn(F.conv2d(x, sd[p + 'downsample.0.weight'], stride=stride), sd, p + 'downsample.1', tm)
    return _relu(out + x, p + 'bn2', tm)


def encoder(x, sd, tm=None):
    """model.py:71-82 with the resnet18 encoder: stem + layer1..4, returns the 4 feature maps (64..512 channels)."""
    e = 'feature_extractor.encoder.'
    x = _circ_conv(x, sd[e + 'conv1.1.weight'], None, 2, 3, 3)        # model.py:73 (7x7 s2, wrapped)
    x = _relu(_bn(x, sd, e + 'bn1', tm), e + 'bn1', tm)                # model.py:74-75
    x = F.max_pool2d(x, 3, 2, 1)                                       # model.py:76 (NOT wrapped)
    feats = []
    for li, nblk in zip((1, 2, 3, 4), BLOCKS):
        for b in range(nblk):
            stride = 2 if (b == 0 and li > 1) else 1
            x = _basic_block(x, sd, f'{e}layer{li}.{b}.', stride, b == 0 and li > 1, tm)
        feats.append(x)                                                # model.py:78-81
    return feats


def forward(sd, x, use_rnn=True, dtype=torch.float32, return_stages=False, train=None):
    """model.py:254-281 with backbone='resnet18'.  sd: the 250-key (use_rnn) or 236-key state_dict; x: [B, C>=3, 512, 1024]
    in [0,1].  Returns (bon [B,2,1024], cor [B,1,1024]); with return_stages also the NCHW stages 'layer1'..'layer4',
    'feature' ([B,256,256]) and 'rnn_out' ([256,B,1024]) or 'mlp_hidden' ([B,256,512])."""
    tm = train
    if x.shape[2] != 512 or x.shape[3] != 1024:
        raise NotImplementedError()                                    # model.py:255-256
    sd = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}
    x = x.to(dtype)
    mean = x.new_tensor(X_MEAN).view(1, 3, 1, 1)
    std = x.new_tensor(X_STD).view(1, 3, 1, 1)
    x = (x[:, :3] - mean) / std                                        # model.py:248-252
    feats = encoder(x, sd, tm)
    bs = x.shape[0]
    out_w = 1024 // 4                                                  # model.py:260
    red = [global_height_conv(f, sd, s, out_w, tm).reshape(bs, -1, out_w) for s, f in enumerate(feats)]
    feature = torch.cat(red, dim=1)                                    # model.py:175-178 -> [B,256,256]
    stages = {f'layer{i + 1}': f for i, f in enumerate(feats)}
    stages['feature'] = feature
    if use_rnn:
        seq = feature.permute(2, 0, 1)                                 # model.py:263
        rnn_out = bi_lstm(seq, sd, tm)                                 # model.py:264 (dropout = id in eval)
        head_in = rnn_out if tm is None else tm.dropout(rnn_out, 1)    # model.py:265 self.drop_out
        out = head_in @ sd['linear.weight'].t() + sd['linear.bias']    # model.py:266
        out = out.view(out.shape[0], out.shape[1], 3, 4).permute(1, 2, 0, 3)
        out = out.contiguous().view(out.shape[0], 3, -1)               # model.py:267-269
        stages['rnn_out'] = rnn_out
    else:
        col = feature.permute(0, 2, 1)                                 # model.py:271 [B, W, 256]
        hidden = _relu(col @ sd['linear.0.weight'].t() + sd['linear.0.bias'], 'linear.1', tm)     # linear[0], linear[1]
        head_in = hidden if tm is None else tm.dropout(hidden, 1)      # linear[2]
        out = head_in @ sd['linear.3.weight'].t() + sd['linear.3.bias']
        out = out.view(bs, out.shape[1], 3, 4).permute(0, 2, 1, 3)     # model.py:273-274
        out = out.contiguous().view(bs, 3, -1)                         # model.py:275
        stages['mlp_hidden'] = hidden
    cor, bon = out[:, :1], out[:, 1:]                                  # model.py:278-279
    if return_stages:
        return bon, cor, stages
    return bon, cor
