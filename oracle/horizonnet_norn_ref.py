"""TEST INFRASTRUCTURE ONLY -- CPU oracle for ``HorizonNet('resnet50', use_rnn=False).forward``, the per-column MLP head
the reference's ``train.py --no_rnn`` builds (reference model.py:234-243, forward :270-279).

The encoder and the height reduction are the ones of oracle/horizonnet_ref.py (model.py:71-82, 148-156, 175-178); only
the head differs: ``Linear(1024, 512) -> ReLU -> Dropout(0.5) -> Linear(512, 12)`` applied to every feature column.
It takes the reference's 434-key ``state_dict`` (``linear.0.*`` and ``linear.3.*`` instead of ``bi_rnn.*`` and
``linear.*``).  Pinned against the real reference by tests/golden/*_norn.* (tests/golden/make_golden_norn.py);
tests/test_no_rnn_head.py asserts this restatement reproduces them.

Train mode takes a ``horizonnet_ref.TrainMode``.  The model has one dropout, ``linear[2]`` on the post-ReLU hidden layer
(model.py:240, :272), so ``masks = (None, [B, 256, 512])`` in the reference's layout; masks=None draws it with F.dropout
from torch's generator, which is the one draw the reference makes.  ``relu_masks['linear.1']`` replaces the hidden
layer's ReLU decisions like the BatchNorm entries of ``relu_masks`` do for the encoder.
"""
import torch

from .horizonnet_ref import X_MEAN, X_STD, _relu, encoder, global_height_conv


def forward(sd, x, dtype=torch.float32, return_stages=False, train=None):
    """model.py:254-279 with use_rnn=False.  sd: the 434-key state_dict; x: [B, C>=3, 512, 1024] in [0,1].

    Returns (bon [B,2,1024], cor [B,1,1024]); with return_stages also the NCHW stages 'layer1'..'layer4', 'feature'
    ([B,1024,256]) and 'mlp_hidden' ([B,256,512], the output of linear[1]).  train: a horizonnet_ref.TrainMode, None = eval.
    """
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
    feature = torch.cat(red, dim=1)                                    # model.py:175-178 -> [B,1024,256]
    col = feature.permute(0, 2, 1)                                     # model.py:271 [B, W, 1024]
    hidden = _relu(col @ sd['linear.0.weight'].t() + sd['linear.0.bias'], 'linear.1', tm)     # linear[0], linear[1]
    head_in = hidden if tm is None else tm.dropout(hidden, 1)          # linear[2]
    out = head_in @ sd['linear.3.weight'].t() + sd['linear.3.bias']    # linear[3] -> [B, W, 12]
    out = out.view(bs, out.shape[1], 3, 4).permute(0, 2, 1, 3)         # model.py:273-274
    out = out.contiguous().view(bs, 3, -1)                             # model.py:275
    cor, bon = out[:, :1], out[:, 1:]                                  # model.py:278-279
    if return_stages:
        stages = {f'layer{i + 1}': f for i, f in enumerate(feats)}
        stages['feature'] = feature
        stages['mlp_hidden'] = hidden
        return bon, cor, stages
    return bon, cor
