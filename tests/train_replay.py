"""fp64 replay of the training step's graph, one backward step at a time (test helper for tests/test_train_replay.py).

The library's training step (csrc/train_step.cu) keeps every conv unit's raw output z, its activation y and, after the
backward, d(loss)/d(y) on a tape (``HorizonNet.debug_train_unit``).  This module describes the same graph in the same
unit order and recomputes each step of the backward in fp64 from the inputs that step actually had, so that a comparison
with the device carries the rounding of one step only:

  * ``build_graph``: the conv units in the order walk_forward lays them out (stem; per block conv1, downsample, conv2 and,
    for a Bottleneck, conv3; then ``ghc_lst.{s}.layer.{j}``), derived from ``_spec.BACKBONES`` and the state-dict shapes;
  * ``unit_step``: y = mask * (BN(conv_circ(in) + bias) + res) of one unit, and its autograd for a given dy;
  * ``head_step``: the four height-reduction outputs -> sequence -> bi-LSTM or MLP head -> (bon, cor), and its autograd;
  * ``walk_backward``: the units in reverse, each driven by a caller-supplied dy, accumulating the data gradients per
    producer tensor and handing each finished sum (and the max-pool's) to the caller.

ReLU decisions and dropout masks always come from the caller; nothing here re-decides a sign.
"""
from dataclasses import dataclass

import torch
import torch.nn.functional as F

from horizonnet_b200._spec import BACKBONES, state_dict_spec
from oracle import horizonnet_ref
from oracle.horizonnet_ref import BN_EPS, X_MEAN, X_STD, _circ_conv

SEQ_W = 256


@dataclass
class Unit:
    name: str           # BatchNorm2d prefix (what debug_train_unit names the unit)
    wkey: str
    bkey: object        # conv bias key or None
    k: int
    stride: tuple
    pad: int            # both axes; W is wrapped, H zero-padded
    src: object         # 'image', 'pool' or the index of the unit whose y is the input
    res: object         # None, 'pool' or a unit index: the identity added before the ReLU
    relu: bool


def build_graph(backbone):
    """(units, gout): the conv units in the library's order and the indices of the four ``ghc_lst.{s}.layer.3`` units."""
    kind, nblocks, _, _ = BACKBONES[backbone]
    spec = state_dict_spec(True, backbone)
    units = []

    def add(name, wkey, src, stride=(1, 1), res=None, relu=True, bkey=None):
        k = spec[wkey][0][-1]
        units.append(Unit(name, wkey, bkey, k, stride, k // 2, src, res, relu))
        return len(units) - 1

    e = 'feature_extractor.encoder.'
    add(e + 'bn1', e + 'conv1.1.weight', 'image', (2, 2))                 # model.py:73-75
    cur, feats = 'pool', []                                                 # model.py:76
    for li, nblk in enumerate(nblocks, start=1):
        for b in range(nblk):
            p = f'{e}layer{li}.{b}.'
            s = (2, 2) if (b == 0 and li > 1) else (1, 1)
            has_ds = p + 'downsample.0.weight' in spec

            def ds():
                return add(p + 'downsample.1', p + 'downsample.0.weight', cur, s, relu=False) if has_ds else cur
            if kind == 'bottleneck':                                        # v1.5: the stride on conv2
                t1 = add(p + 'bn1', p + 'conv1.weight', cur)
                idn = ds()
                t2 = add(p + 'bn2', p + 'conv2.1.weight', t1, s)
                cur = add(p + 'bn3', p + 'conv3.weight', t2, res=idn)
            else:                                                           # BasicBlock: the stride on conv1
                t1 = add(p + 'bn1', p + 'conv1.1.weight', cur, s)
                idn = ds()
                cur = add(p + 'bn2', p + 'conv2.1.weight', t1, res=idn)
        feats.append(cur)
    gout = []
    for s, g in enumerate(feats):                                           # model.py:148-151
        for j in range(4):
            p = f'reduce_height_module.ghc_lst.{s}.layer.{j}.layers.'
            g = add(p + '1', p + '0.1.weight', g, (2, 1), bkey=p + '0.1.bias')
        gout.append(g)
    return units, gout


def normalised_image(x, dtype=torch.float64):
    """model.py:248-252 on x [B, C>=3, 512, 1024]."""
    x = x[:, :3].to(dtype)
    return (x - x.new_tensor(X_MEAN).view(1, 3, 1, 1)) / x.new_tensor(X_STD).view(1, 3, 1, 1)


def pool(stem_y):
    return F.max_pool2d(stem_y, 3, 2, 1)                                    # model.py:76 (not wrapped)


def unit_forward(u, sd, x, res, mask, train):
    """(z, y) of one unit; mask None: ReLU decisions from this forward's own signs (tape-producing forward only)."""
    z = _circ_conv(x, sd[u.wkey], sd[u.bkey] if u.bkey else None, u.stride, u.pad, u.pad)
    if train:
        y = F.batch_norm(z, None, None, sd[u.name + '.weight'], sd[u.name + '.bias'], True, 0.0, BN_EPS)
    else:
        y = F.batch_norm(z, sd[u.name + '.running_mean'], sd[u.name + '.running_var'], sd[u.name + '.weight'],
                         sd[u.name + '.bias'], False, 0.0, BN_EPS)
    if res is not None:
        y = y + res
    if u.relu:
        y = y * ((y > 0) if mask is None else mask).to(y.dtype)
    return z, y


def forward_tape(units, sd, image, frozen):
    """Tape-producing forward through the graph, ReLU decisions from its own signs: ([z], [y]) in unit order."""
    zs, ys, pooled = [], [], None

    def act(k):
        return image if k == 'image' else pooled if k == 'pool' else ys[k]
    for i, u in enumerate(units):
        z, y = unit_forward(u, sd, act(u.src), act(u.res) if u.res is not None else None, None, u.name not in frozen)
        zs.append(z)
        ys.append(y)
        if i == 0:
            pooled = pool(y)
    return zs, ys


def unit_step(u, sd, x, res, mask, train, dy):
    """One unit replayed in fp64 from the given input, residual and ReLU mask, and backpropagated from dy.  Returns
    {'z', 'y', 'in' (None for the stem), 'res', 'weight', 'bias', 'gamma', 'beta'} (detached)."""
    leaf = {'weight': sd[u.wkey], 'gamma': sd[u.name + '.weight'], 'beta': sd[u.name + '.bias']}
    if u.bkey:
        leaf['bias'] = sd[u.bkey]
    if u.src != 'image':
        leaf['in'] = x
    if res is not None:
        leaf['res'] = res
    leaf = {k: v.detach().to(torch.float64).requires_grad_() for k, v in leaf.items()}
    p = dict(sd)
    p[u.wkey], p[u.name + '.weight'], p[u.name + '.bias'] = leaf['weight'], leaf['gamma'], leaf['beta']
    if u.bkey:
        p[u.bkey] = leaf['bias']
    z, y = unit_forward(u, p, leaf.get('in', x), leaf.get('res'), mask, train)
    names = list(leaf)
    grads = torch.autograd.grad(y, [leaf[k] for k in names], dy)
    out = dict.fromkeys(('in', 'res', 'bias'))
    out.update(zip(names, grads))
    out['z'], out['y'] = z.detach(), y.detach()
    return out


def to_sequence(gouts, out_w=SEQ_W):
    """model.py:152-155 (GlobalHeightConv's wrap pad, bilinear x f, crop) per scale, :175-178 concat -> [B, c_last, 256]."""
    red = []
    for x in gouts:
        factor = out_w // x.shape[3]
        x = torch.cat([x[..., -1:], x, x[..., :1]], 3)
        x = F.interpolate(x, size=(x.shape[2], out_w + 2 * factor), mode='bilinear', align_corners=False)
        red.append(x[..., factor:-factor].reshape(x.shape[0], -1, out_w))
    return torch.cat(red, dim=1)


def head_forward(gouts, sd, use_rnn, masks, hidden_mask=None):
    """(bon, cor, hidden) from the four height-reduction outputs.  masks: the library's dropout masks (bi-LSTM: two
    [256, B, 1024]; MLP: (None, [256, B, 512]) with rows t*B + b); hidden_mask: the MLP's ReLU decisions [B, 256, 512]
    (None: from this forward's own signs).  hidden is None for the bi-LSTM head."""
    feature = to_sequence(gouts)
    bs = feature.shape[0]
    dt = feature.dtype
    if use_rnn:
        tm = horizonnet_ref.TrainMode(masks=[m.to(dt) for m in masks])
        rnn_out = horizonnet_ref.bi_lstm(feature.permute(2, 0, 1), sd, tm)           # model.py:263-264
        out = tm.dropout(rnn_out, 1) @ sd['linear.weight'].t() + sd['linear.bias']    # model.py:265-266
        out = out.view(out.shape[0], out.shape[1], 3, 4).permute(1, 2, 0, 3).contiguous().view(bs, 3, -1)
        hidden = None
    else:
        pre = feature.permute(0, 2, 1) @ sd['linear.0.weight'].t() + sd['linear.0.bias']
        hidden = pre * ((pre > 0) if hidden_mask is None else hidden_mask).to(dt)     # linear[0], linear[1]
        head_in = hidden * masks[1].permute(1, 0, 2).to(dt)                           # linear[2]
        out = head_in @ sd['linear.3.weight'].t() + sd['linear.3.bias']
        out = out.view(bs, out.shape[1], 3, 4).permute(0, 2, 1, 3).contiguous().view(bs, 3, -1)   # model.py:273-275
    return out[:, 1:], out[:, :1], hidden                                            # model.py:278-279


def head_params(use_rnn, sd):
    return [k for k in sd if k.startswith(('bi_rnn.', 'linear'))]


def head_step(gouts, sd, use_rnn, masks, hidden_mask, dbon, dcor):
    """The head replayed in fp64 from the given height-reduction outputs and backpropagated from (dbon, dcor).
    Returns (bon, cor, hidden, [d gout[s]], {head parameter: gradient})."""
    leaves = [g.detach().to(torch.float64).requires_grad_() for g in gouts]
    keys = head_params(use_rnn, sd)
    p = dict(sd)
    for k in keys:
        p[k] = sd[k].detach().to(torch.float64).requires_grad_()
    bon, cor, hidden = head_forward(leaves, p, use_rnn, masks, hidden_mask)
    grads = torch.autograd.grad((bon, cor), leaves + [p[k] for k in keys], (dbon, dcor))
    return (bon.detach(), cor.detach(), None if hidden is None else hidden.detach(), list(grads[:4]),
            dict(zip(keys, grads[4:])))


def consumers(units):
    """producer ('pool' or unit index) -> indices of the units that read it as input or residual."""
    out = {}
    for i, u in enumerate(units):
        for p in (u.src, u.res):
            if p is not None and p != 'image':
                out.setdefault(p, []).append(i)
    return out


def walk_backward(units, gout, sd, frozen, act, dgout, dy_of, report):
    """The conv units in reverse, each replayed by unit_step from act(its input), act(its residual) and act(itself) > 0
    as the ReLU mask, driven by dy_of(i, accumulated d y of unit i).

    act(key): fp64 activation for 'image', 'pool' or a unit index.  dgout: d(loss)/d(gout[s]), the seed of the four last
    units' accumulators.  report(kind, key, value) is called with
      ('unit', i, unit_step result)             after each unit,
      ('dy', producer, accumulated d y)          once all consumers of a producer unit are done,
      ('pool', None, (d pool, d stem y))         d(pool output) and its max-pool adjoint onto the stem activation.
    Only the accumulators still waiting for a consumer are held."""
    cons = consumers(units)
    done_at = {p: min(c) for p, c in cons.items()}
    acc = {g: d for g, d in zip(gout, dgout)}
    for i in range(len(units) - 1, -1, -1):
        u = units[i]
        y = act(i)
        mask = (y > 0) if u.relu else None
        x = act(u.src)
        res = act(u.res) if u.res is not None else None
        r = unit_step(u, sd, x, res, mask, u.name not in frozen, dy_of(i, acc.pop(i)))
        del x, res, y, mask
        for p, d in ((u.src, r['in']), (u.res, r['res'])):
            if d is not None:
                acc[p] = acc[p] + d if p in acc else d
        report('unit', i, r)
        for p, last in done_at.items():
            if last != i:
                continue
            if p == 'pool':
                stem_y = act(0).detach().requires_grad_()
                dpool = acc.pop('pool')
                dstem, = torch.autograd.grad(pool(stem_y), stem_y, dpool)
                report('pool', None, (dpool, dstem))
                acc[0] = dstem
            else:
                report('dy', p, acc[p])
