"""Drop-in ``HorizonNet`` (reference model.py:185-281) backed by libhorizonnet_b200 (sm_90a CUDA).

Boundary kept from the reference (SURVEY 8b):
  * ``HorizonNet(backbone, use_rnn)`` is an ``nn.Module`` whose parameters/buffers carry exactly
    the reference's 448 ``state_dict`` keys (434 with ``use_rnn=False``), so ``misc/utils.py:49-65``
    (``save_model`` / ``load_trained_model``) work unchanged with this class;
  * ``forward(x[B, C>=3, 512, 1024]) -> (bon[B,2,1024], cor[B,1,1024])`` raw fp32 outputs,
    ``NotImplementedError`` for any other H x W (model.py:255-256);
  * ``.backbone``, ``.use_rnn``, ``.feature_extractor.list_blocks()``, ``.x_mean``, ``.x_std``.
Built: ``backbone='resnet50'`` with ``use_rnn=True`` (the path BASELINE.json names) or ``use_rnn=False`` (the
per-column MLP head of model.py:234-243, what the reference's ``train.py --no_rnn`` trains), and ``backbone='resnet18'``
(torchvision BasicBlocks, a 256-wide feature sequence) with either head; inference
(eval) forward -- plus the train-mode FORWARD (batch-statistics BatchNorm with running-stat updates,
LSTM / head dropout; train.py:52) and its backward (train.py:278 ``loss.backward()``): with autograd on,
``forward`` in train mode returns outputs whose grad_fn runs the library's backward pass and fills
``.grad`` of every parameter (row f1; one process per GPU, ``parallel.average_gradients`` in place of DataParallel).
The modules below are parameter containers with the reference's names; none of
their torch ``forward`` methods is ever called -- all arithmetic runs in the CUDA library, and there
is no CPU fallback: a CPU tensor or a missing library raises.
"""
import ctypes
import os
import threading

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from ._spec import BACKBONES, HEAD_BIAS, RNN_HIDDEN, STEP_COLS, PANO_H, PANO_W, c_last, encoder_channels, state_dict_spec


class CircularPadW(nn.Module):
    """Index-0 placeholder of the ``Sequential(LR_PAD, conv)`` pairs the reference creates in
    wrap_lr_pad (model.py:42-55); it is why wrapped convs are keyed ``...conv2.1.weight``.  The
    circular padding itself is realised by the halo columns of the device activation layout."""

    def __init__(self, padding):
        super().__init__()
        self.padding = padding

    def forward(self, x):
        raise RuntimeError('horizonnet_b200 modules are parameter containers; call HorizonNet.forward')


def _wrapped_conv(cin, cout, k, stride, bias):
    return nn.Sequential(CircularPadW(k // 2),
                         nn.Conv2d(cin, cout, k, stride=stride, padding=(k // 2, 0), bias=bias))


class _Bottleneck(nn.Module):
    def __init__(self, inplanes, planes, stride, downsample):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = _wrapped_conv(planes, planes, 3, stride, False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        if downsample:
            self.downsample = nn.Sequential(nn.Conv2d(inplanes, planes * 4, 1, stride=stride, bias=False),
                                            nn.BatchNorm2d(planes * 4))


class _BasicBlock(nn.Module):
    """torchvision resnet.py BasicBlock: two 3x3 convs (wrapped by LR_PAD, hence ``conv1.1`` / ``conv2.1``), the stride on
    conv1, the downsample on block 0 of layers 2-4 only."""

    def __init__(self, inplanes, planes, stride, downsample):
        super().__init__()
        self.conv1 = _wrapped_conv(inplanes, planes, 3, stride, False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = _wrapped_conv(planes, planes, 3, 1, False)
        self.bn2 = nn.BatchNorm2d(planes)
        if downsample:
            self.downsample = nn.Sequential(nn.Conv2d(inplanes, planes, 1, stride=stride, bias=False),
                                            nn.BatchNorm2d(planes))


class _ResNet(nn.Module):
    def __init__(self, backbone):
        super().__init__()
        kind, nblocks, planes_l, expansion = BACKBONES[backbone]
        block = _Bottleneck if kind == 'bottleneck' else _BasicBlock
        self.conv1 = _wrapped_conv(3, 64, 7, 2, False)
        self.bn1 = nn.BatchNorm2d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(3, 2, 1)
        inplanes = 64
        for li, (nblk, planes) in enumerate(zip(nblocks, planes_l), start=1):
            blocks = []
            for b in range(nblk):
                stride = 2 if (b == 0 and li > 1) else 1
                blocks.append(block(inplanes, planes, stride, b == 0 and (stride != 1 or inplanes != planes * expansion)))
                inplanes = planes * expansion
            setattr(self, f'layer{li}', nn.Sequential(*blocks))
        for m in self.modules():            # torchvision resnet.py:208-213 initialisation
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')


class _Encoder(nn.Module):
    def __init__(self, backbone):
        super().__init__()
        self.encoder = _ResNet(backbone)

    def list_blocks(self):
        """Same grouping as reference model.py:84-91 (used by train.py --freeze_earlier_blocks)."""
        lst = list(self.encoder.children())
        return lst[:4], lst[4:5], lst[5:6], lst[6:7], lst[7:8]


class _CompressH(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.layers = nn.Sequential(_wrapped_conv(cin, cout, 3, (2, 1), True), nn.BatchNorm2d(cout),
                                    nn.ReLU(inplace=True))


class _HeightConv(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.layer = nn.Sequential(_CompressH(cin, cin // 2), _CompressH(cin // 2, cin // 2),
                                   _CompressH(cin // 2, cin // 4), _CompressH(cin // 4, cout))


class _HeightStage(nn.Module):
    def __init__(self, cs, out_scale):
        super().__init__()
        self.cs = cs
        self.out_scale = out_scale
        self.ghc_lst = nn.ModuleList([_HeightConv(c, c // out_scale) for c in cs])


class _TrainStep(torch.autograd.Function):
    """forward = hn_train_forward (train-mode forward with a tape), backward = hn_train_backward.  The parameters are
    inputs only so that autograd routes their gradients; the arithmetic reads the device copies the handle holds."""

    @staticmethod
    def forward(ctx, net, x, *params):
        bon, cor = net._train_forward_impl(x)
        ctx.net, ctx.device = net, x.device
        ctx.wanted = [p.requires_grad for p in params]
        return bon, cor

    @staticmethod
    def backward(ctx, dbon, dcor):
        B = dbon.shape[0] if dbon is not None else dcor.shape[0]
        dbon = torch.zeros(B, 2, PANO_W, device=ctx.device) if dbon is None else dbon.to(torch.float32).contiguous()
        dcor = torch.zeros(B, 1, PANO_W, device=ctx.device) if dcor is None else dcor.to(torch.float32).contiguous()
        grads = ctx.net._train_backward_impl(ctx.device, dbon, dcor, ctx.wanted)
        return (None, None) + tuple(grads)


class HorizonNet(nn.Module):
    x_mean = torch.FloatTensor(np.array([0.485, 0.456, 0.406])[None, :, None, None])
    x_std = torch.FloatTensor(np.array([0.229, 0.224, 0.225])[None, :, None, None])

    def __init__(self, backbone, use_rnn):
        super().__init__()
        if backbone not in BACKBONES:
            raise NotImplementedError(
                f"horizonnet_b200 implements the {' and '.join(sorted(BACKBONES))} backbones (use_rnn=True or False), "
                f"not {backbone!r}")
        self.backbone = backbone
        self.use_rnn = use_rnn
        self.out_scale = 8
        self.step_cols = STEP_COLS
        self.rnn_hidden_size = RNN_HIDDEN
        self.feature_extractor = _Encoder(backbone)
        self.reduce_height_module = _HeightStage(encoder_channels(backbone), self.out_scale)
        width = c_last(backbone)                                      # feature sequence: 1024 (resnet50), 256 (resnet18)
        if use_rnn:
            self.bi_rnn = nn.LSTM(input_size=width, hidden_size=RNN_HIDDEN, num_layers=2, dropout=0.5,
                                  batch_first=False, bidirectional=True)
            self.drop_out = nn.Dropout(0.5)
            self.linear = nn.Linear(2 * RNN_HIDDEN, 3 * STEP_COLS)
            head = self.linear
        else:                                                         # model.py:234-243
            self.linear = nn.Sequential(nn.Linear(width, RNN_HIDDEN), nn.ReLU(inplace=True), nn.Dropout(0.5),
                                        nn.Linear(RNN_HIDDEN, 3 * STEP_COLS))
            head = self.linear[-1]
        with torch.no_grad():
            head.bias.copy_(torch.tensor(HEAD_BIAS))                  # model.py:231-233, :241-243
        # bypass nn.Module.__setattr__: runtime state must not become sub-modules / parameters
        object.__setattr__(self, '_handles', {})
        object.__setattr__(self, '_lock', threading.Lock())
        object.__setattr__(self, '_tensor_cores', 1)
        object.__setattr__(self, '_refresh_epoch', 0)
        object.__setattr__(self, 'last_dropout_seed', None)
        object.__setattr__(self, 'dropout_masks_override', None)    # test hook: (inter-layer, head) masks instead of Philox
        self._slots = None

    # ---- weights -> device library --------------------------------------------------------------
    def _state_tensors(self):
        if self._slots is None:
            slots = []
            spec = state_dict_spec(self.use_rnn, self.backbone)
            for key in spec:
                *path, leaf = key.split('.')
                mod = self
                for p in path:
                    mod = getattr(mod, p)
                slots.append((key, mod, leaf))
            self._slots = slots
        for key, mod, leaf in self._slots:
            t = mod._parameters.get(leaf)
            if t is None:
                t = mod._buffers[leaf]
            yield key, t

    def _weight_signature(self):
        """Identity of the current weights: (storage pointer, in-place version counter) of every tensor.  Edits made
        through ``param.data`` do not bump the version counter -- call refresh_weights() after such edits."""
        if self._slots is None:
            list(self._state_tensors())
        sig = [self._tensor_cores, self._refresh_epoch]
        for _, mod, leaf in self._slots:
            t = mod._parameters.get(leaf)
            if t is None:
                t = mod._buffers[leaf]
            sig.append(t.data_ptr())
            sig.append(t._version)
        return tuple(sig)

    def refresh_weights(self):
        """Force a re-upload of all weights on the next forward (needed after edits through ``.data`` / raw pointers,
        which PyTorch's version counter does not see)."""
        object.__setattr__(self, '_refresh_epoch', self._refresh_epoch + 1)
        return self

    def use_tensor_cores(self, enabled=True):
        """True (default): split-fp16 (hi+lo planes, 3 products) wgmma kernels where supported; False: exact fp32 kernels."""
        object.__setattr__(self, '_tensor_cores', 1 if enabled else 0)
        for h in self._handles.values():
            h['sig'] = None
        return self

    def _handle(self, device, batch):
        lib = _lib.lib()
        key = device.index if device.index is not None else torch.cuda.current_device()
        with self._lock:
            h = self._handles.get(key)
            if h is not None and h['max_batch'] < batch:
                if h.get('pending'):
                    raise RuntimeError('collect_host() the submitted batches before running a larger batch: the device '
                                       'workspace has to be re-created for it')
                lib.hn_model_destroy(h['ptr'])
                h = None
            if h is None:
                ptr = ctypes.c_void_p()
                max_batch = max(batch, 1)
                _lib.check(lib.hn_model_create_arch(key, max_batch, self.backbone.encode(), 1 if self.use_rnn else 0,
                                                    ctypes.byref(ptr)), 'hn_model_create_arch')
                h = {'ptr': ptr, 'max_batch': max_batch, 'sig': None}
                self._handles[key] = h
            sig = self._weight_signature()
            if h['sig'] != sig:
                for k, t in self._state_tensors():
                    if not t.is_floating_point():
                        _lib.check(lib.hn_model_set_tensor(h['ptr'], k.encode(), None, 1, 1), k)
                        continue
                    d = t.detach().to(device=device, dtype=torch.float32).contiguous()
                    _lib.check(lib.hn_model_set_tensor(h['ptr'], k.encode(), d.data_ptr(), d.numel(), 1), k)
                _lib.check(lib.hn_model_set_option(h['ptr'], b'tensor_cores', self._tensor_cores), 'set_option')
                _lib.check(lib.hn_model_finalize(h['ptr']), 'hn_model_finalize')
                h['sig'] = sig
        return h

    def _prepare_x(self, x):          # kept for API parity (model.py:248-252); fused into the stem kernel
        raise RuntimeError('input normalisation is fused into the stem kernel; call forward()')

    def forward(self, x):
        if self._train_mode_active():
            return self._forward_train(x)
        x, B, C, h, bon, cor, stream = self._forward_prologue(x)
        _lib.check(_lib.lib().hn_model_forward(h['ptr'], x.data_ptr(), B, C, bon.data_ptr(), cor.data_ptr(), stream),
                   'hn_model_forward')
        return bon, cor

    # ---- train-mode forward (train.py:52 under net.train()) ---------------------------------------
    def _train_mode_active(self):
        """True if any module that behaves differently in training mode is in training mode: a BatchNorm2d (batch
        statistics), the LSTM (inter-layer dropout) or the head dropout (linear[2] of the MLP head).  torch keeps the
        flag per module, and train.py:251-256 (--freeze_earlier_blocks) really does mix them."""
        rnn_p, head_p = self._dropout_ps(active_only=True)
        if rnn_p > 0 or head_p > 0:
            return True
        return any(m.training for m in self.modules() if isinstance(m, nn.BatchNorm2d))

    def _head_dropout(self):
        return self.drop_out if self.use_rnn else self.linear[2]

    def _dropout_ps(self, active_only):
        """(inter-layer LSTM dropout p, head dropout p); active_only: 0 for a module in eval mode.  The MLP head has no
        LSTM, so its first entry is always 0."""
        rnn_p = float(self.bi_rnn.dropout) if self.use_rnn and (self.bi_rnn.training or not active_only) else 0.0
        d = self._head_dropout()
        head_p = float(d.p) if (d.training or not active_only) else 0.0
        return rnn_p, head_p

    def _bn_modules(self, h):
        if 'bn' not in h:
            lib = _lib.lib()
            names = [lib.hn_model_bn_name(h['ptr'], i).decode() for i in range(lib.hn_model_num_bn(h['ptr']))]
            h['bn'] = [(n, self.get_submodule(n)) for n in names]
        return h['bn']

    def _forward_train(self, x):
        """Batch-statistics BN (+ running-stat update written back into the module buffers, num_batches_tracked
        incremented), LSTM inter-layer dropout and head dropout (MLP head: the dropout of linear[2]).  The dropout seed is drawn from torch's default
        generator (reproducible under torch.manual_seed) and kept in ``last_dropout_seed``; the masks are this
        library's Philox stream, not torch's.

        Every call runs the training step's forward (hn_train_forward, which keeps a tape; batch <= 64), so the
        outputs do not depend on whether autograd is on.  With autograd on and a parameter that requires grad they
        carry a grad_fn whose backward is hn_train_backward: the reference's ``loss.backward()`` (train.py:278) then
        fills ``.grad`` of every parameter."""
        params = [(k, p) for k, p in self.named_parameters()]
        if torch.is_grad_enabled() and any(p.requires_grad for _, p in params):
            return _TrainStep.apply(self, x, *[p for _, p in params])
        return self._train_forward_impl(x)

    def _train_forward_impl(self, x):
        x, B, C, h, bon, cor, stream = self._forward_prologue(x, train=True)
        lib = _lib.lib()
        bns = self._bn_modules(h)
        flags = (ctypes.c_ubyte * len(bns))(*[1 if m.training else 0 for _, m in bns])
        factors = (ctypes.c_double * len(bns))()
        for i, (_, m) in enumerate(bns):
            if not (m.training and m.track_running_stats):
                factors[i] = -1.0
            elif m.momentum is None:
                factors[i] = 1.0 / float(int(m.num_batches_tracked) + 1)        # cumulative moving average
            else:
                factors[i] = float(m.momentum)
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        object.__setattr__(self, 'last_dropout_seed', seed)
        rnn_p, head_p = self._dropout_ps(active_only=True)
        masks = [None, None]
        if getattr(self, 'dropout_masks_override', None) is not None:        # parity-test hook: torch-drawn masks
            masks = [t.to(device=x.device, dtype=torch.float32).contiguous() if t is not None else None
                     for t in self.dropout_masks_override]
            shapes = [(256, B, 2 * RNN_HIDDEN)] * 2 if self.use_rnn else [None, (256, B, RNN_HIDDEN)]
            assert all((t is None and s is None) or (t is not None and t.shape == s) for t, s in zip(masks, shapes))
        _lib.check(lib.hn_train_forward(h['ptr'], x.data_ptr(), B, C, bon.data_ptr(), cor.data_ptr(), flags, factors,
                                        len(bns), seed, rnn_p, head_p,
                                        masks[0].data_ptr() if masks[0] is not None else None,
                                        masks[1].data_ptr() if masks[1] is not None else None, stream),
                   'hn_train_forward')
        h['tape_keepalive'] = (x, masks)        # the backward reads the masks again
        with torch.no_grad():
            for i, (name, m) in enumerate(bns):
                if factors[i] < 0:
                    continue
                for leaf in ('running_mean', 'running_var'):
                    buf = getattr(m, leaf)
                    direct = buf.is_cuda and buf.device == x.device and buf.dtype == torch.float32 and buf.is_contiguous()
                    dst = buf if direct else torch.empty(buf.numel(), device=x.device, dtype=torch.float32)
                    _lib.check(lib.hn_model_get_tensor(h['ptr'], f'{name}.{leaf}'.encode(), dst.data_ptr(), buf.numel(), 1,
                                                       stream), 'hn_model_get_tensor')
                    if not direct:
                        buf.copy_(dst.view_as(buf))
                m.num_batches_tracked += 1
        h['sig'] = self._weight_signature()       # the device copies already hold what the buffers now hold
        for other in self._handles.values():
            if other is not h:
                other['sig'] = None
        return bon, cor

    def _train_backward_impl(self, device, dbon, dcor, wanted):
        """d(loss)/d(bon), d(loss)/d(cor) -> one gradient per named parameter (None where not wanted)."""
        lib = _lib.lib()
        key = device.index if device.index is not None else torch.cuda.current_device()
        h = self._handles[key]
        stream = torch.cuda.current_stream(device).cuda_stream
        with torch.cuda.device(device):
            _lib.check(lib.hn_train_backward(h['ptr'], dbon.data_ptr(), dcor.data_ptr(), stream), 'hn_train_backward')
            grads = []
            for (name, p), want in zip(self.named_parameters(), wanted):
                if not want:
                    grads.append(None)
                    continue
                g = torch.empty(p.shape, device=device, dtype=torch.float32)
                _lib.check(lib.hn_model_get_grad(h['ptr'], name.encode(), g.data_ptr(), g.numel(), stream), 'hn_model_get_grad')
                grads.append(g.to(device=p.device, dtype=p.dtype))
        h['tape_keepalive'] = None
        return grads

    def train_profile(self, device=None):
        """Device ms of the phases of the last backward: {'head', 'lstm', 'sequence', 'conv_units'}."""
        key = next(iter(self._handles)) if device is None else device
        ms = (ctypes.c_double * 4)()
        _lib.check(_lib.lib().hn_train_profile(self._handles[key]['ptr'], ms), 'hn_train_profile')
        out = dict(zip(('head', 'lstm', 'sequence', 'conv_units'), [round(v, 3) for v in ms]))
        if os.environ.get('HN_TRAIN_PROF', '0') not in ('', '0'):      # per-unit events were recorded: split the conv units
            us = (ctypes.c_double * 3)()
            if _lib.lib().hn_train_profile_units(self._handles[key]['ptr'], us) == 0:
                out.update(zip(('units_bn_backward', 'units_weight_gradient', 'units_data_gradient'), [round(v, 3) for v in us]))
        return out

    def debug_train_unit(self, i, what=0, device=None):
        """Tape of the last training-step forward (test hook): conv unit i in graph order (stem, blocks, height
        reduction) -> (BatchNorm2d prefix, NCHW tensor); what = 0 activation, 1 raw conv output, 2 its gradient."""
        lib = _lib.lib()
        key = next(iter(self._handles)) if device is None else device
        h = self._handles[key]
        dev = torch.device('cuda', key)
        cap = h['max_batch'] * 130 * 258 * 256
        out = torch.empty(cap, device=dev, dtype=torch.float32)
        dims = (ctypes.c_int * 4)()
        name = ctypes.create_string_buffer(256)
        with torch.cuda.device(dev):
            _lib.check(lib.hn_train_debug_unit(h['ptr'], i, what, out.data_ptr(), cap, dims, name, 256,
                                               torch.cuda.current_stream(dev).cuda_stream), 'hn_train_debug_unit')
        B, H, W, C = list(dims)
        t = out[:B * H * (W + 2) * C].view(B, H, W + 2, C)[:, :, 1:-1].permute(0, 3, 1, 2).contiguous()
        return name.value.decode(), t

    def dropout_masks(self, seed, batch, device):
        """The two multiplicative masks ([256, batch, 1024], values 0 or 1/(1-p)) a train forward with this seed applies:
        (between the LSTM layers, before the linear head).  MLP head: (None, [256, batch, 512]), the mask of linear[2] on
        the hidden layer, rows t*batch + b.  Test hook."""
        out = []
        dev = torch.device(device)
        rnn_p, head_p = self._dropout_ps(active_only=False)
        width = 2 * RNN_HIDDEN if self.use_rnn else RNN_HIDDEN
        for which, p in ((0, rnn_p), (1, head_p)):
            if which == 0 and not self.use_rnn:
                out.append(None)
                continue
            t = torch.empty(256, batch, width, device=dev, dtype=torch.float32)
            with torch.cuda.device(dev):
                _lib.check(_lib.lib().hn_dropout_mask(seed, which, p, t.data_ptr(), t.numel(),
                                                      torch.cuda.current_stream(dev).cuda_stream), 'hn_dropout_mask')
            out.append(t)
        return out

    def _refuse_train_mode(self):
        if self._train_mode_active():
            # the pipelined / host entry points run the eval graph only; in train mode that would diverge silently
            raise NotImplementedError('this entry point runs the inference graph: call .eval() first, or use forward() '
                                      'for the train-mode forward (backward is the "next" row f1)')

    def _forward_prologue(self, x, train=False):
        if x.shape[2] != PANO_H or x.shape[3] != PANO_W:
            raise NotImplementedError()                                   # model.py:255-256
        if not train:
            self._refuse_train_mode()
        if not x.is_cuda:
            raise RuntimeError('horizonnet_b200.HorizonNet has no CPU path: move the input to an H100 (cuda) device')
        if x.shape[1] < 3:
            raise RuntimeError('input needs at least 3 channels (model.py:252 reads x[:, :3])')
        x = x.detach().to(torch.float32).contiguous()
        B, C = x.shape[0], x.shape[1]
        h = self._handle(x.device, B)
        bon = torch.empty(B, 2, PANO_W, device=x.device, dtype=torch.float32)
        cor = torch.empty(B, 1, PANO_W, device=x.device, dtype=torch.float32)
        stream = torch.cuda.current_stream(x.device).cuda_stream
        return x, B, C, h, bon, cor, stream

    def forward_pipelined(self, x):
        """Throughput form of forward() for streams of batches (hn_model_forward_async): the encoder of this batch
        overlaps the bi-LSTM of the previous one on internal streams.  Returns (bon, cor) like forward(); in the order
        of the current CUDA stream they are complete after the NEXT forward_pipelined() call or after flush().
        Values are bit-identical to forward()."""
        x, B, C, h, bon, cor, stream = self._forward_prologue(x)
        _lib.check(_lib.lib().hn_model_forward_async(h['ptr'], x.data_ptr(), B, C, bon.data_ptr(), cor.data_ptr(), stream),
                   'hn_model_forward_async')
        # the caching allocator must not hand these buffers to another stream-ordered user before the internal
        # streams are done with them: keep them referenced until the next call / flush
        h['inflight'] = (h.get('inflight', ()) + ((x, bon, cor),))[-2:]
        return bon, cor

    def flush(self):
        """Make the current CUDA stream wait for every forward_pipelined() issued so far."""
        for key, h in self._handles.items():
            stream = torch.cuda.current_stream(torch.device('cuda', key)).cuda_stream
            _lib.check(_lib.lib().hn_model_flush(h['ptr'], stream), 'hn_model_flush')

    def forward_host(self, x_host, device=0):
        """End-to-end call on HOST arrays through the C ABI (H2D + forward + D2H inside the
        library): the equivalent of inference.py:78-79.  x_host: contiguous fp32 [B,C,512,1024]
        numpy array or CPU tensor (pinned memory makes the copies asynchronous-capable)."""
        xt = torch.as_tensor(x_host)
        if xt.is_cuda or xt.dtype != torch.float32 or not xt.is_contiguous():
            raise RuntimeError('forward_host expects a contiguous fp32 host array')
        if xt.shape[2] != PANO_H or xt.shape[3] != PANO_W:
            raise NotImplementedError()
        self._refuse_train_mode()
        B, C = xt.shape[0], xt.shape[1]
        dev = torch.device('cuda', device)
        h = self._handle(dev, B)
        bon = torch.empty(B, 2, PANO_W, dtype=torch.float32)
        cor = torch.empty(B, 1, PANO_W, dtype=torch.float32)
        _lib.check(_lib.lib().hn_model_forward_host(h['ptr'], xt.data_ptr(), B, C, bon.data_ptr(), cor.data_ptr()),
                   'hn_model_forward_host')
        return bon, cor

    def submit_host(self, x_host, device=0):
        """Pipelined host API (hn_model_submit_host): enqueue the upload of a batch; pair with collect_host()."""
        xt = torch.as_tensor(x_host)
        if xt.is_cuda or xt.dtype != torch.float32 or not xt.is_contiguous():
            raise RuntimeError('submit_host expects a contiguous fp32 host array')
        if xt.shape[2] != PANO_H or xt.shape[3] != PANO_W:
            raise NotImplementedError()
        self._refuse_train_mode()
        h = self._handle(torch.device('cuda', device), xt.shape[0])
        _lib.check(_lib.lib().hn_model_submit_host(h['ptr'], xt.data_ptr(), xt.shape[0], xt.shape[1]), 'hn_model_submit_host')
        h.setdefault('pending', []).append((xt, xt.shape[0]))        # keep the host buffer alive until collected

    def collect_host(self, device=0):
        """Forward + D2H of the oldest submitted batch -> (bon, cor) CPU tensors."""
        h = self._handles[device]
        _, B = h['pending'].pop(0)
        bon = torch.empty(B, 2, PANO_W, dtype=torch.float32)
        cor = torch.empty(B, 1, PANO_W, dtype=torch.float32)
        _lib.check(_lib.lib().hn_model_collect_host(h['ptr'], bon.data_ptr(), cor.data_ptr()), 'hn_model_collect_host')
        return bon, cor

    def set_option(self, name, value):
        """Library switch on every live handle (include/horizonnet_b200.h: hn_model_set_option)."""
        for h in self._handles.values():
            _lib.check(_lib.lib().hn_model_set_option(h['ptr'], name.encode(), int(value)), 'set_option')
        return self

    def debug_stage(self, name, device=None):
        """Intermediate result of the last forward in the reference's layout (test hook)."""
        lib = _lib.lib()
        key = next(iter(self._handles)) if device is None else device
        h = self._handles[key]
        dev = torch.device('cuda', key)
        dims = (ctypes.c_int * 4)()
        cap = h['max_batch'] * 256 * 128 * 256
        out = torch.empty(cap, device=dev, dtype=torch.float32)
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.hn_model_stage(h['ptr'], name.encode(), out.data_ptr(), cap, dims, stream), 'hn_model_stage')
        shape = [d for d in dims if d > 0]
        return out[:int(np.prod(shape))].view(*shape)

    PROFILE_CLASSES = ('stem', 'maxpool', 'encoder_convs', 'height_reduction_convs', 'upsample_concat',
                       'lstm_input_projection', 'lstm_recurrence', 'linear_head')

    def set_profile(self, enabled=True):
        """Per-launch CUDA-event timing inside the library (used by bench.py for the roofline)."""
        for h in self._handles.values():
            _lib.check(_lib.lib().hn_model_set_option(h['ptr'], b'profile', 1 if enabled else 0), 'set_option')

    def read_profile(self, reset=True):
        """{class: (device ms, algorithmic FLOPs, launches)} accumulated since the last reset."""
        out = {}
        for h in self._handles.values():
            ms = (ctypes.c_double * 8)()
            fl = (ctypes.c_double * 8)()
            n = (ctypes.c_longlong * 8)()
            _lib.check(_lib.lib().hn_model_profile_read(h['ptr'], ms, fl, n, 1 if reset else 0), 'profile_read')
            for i, name in enumerate(self.PROFILE_CLASSES):
                a = out.get(name, (0.0, 0.0, 0))
                out[name] = (a[0] + ms[i], a[1] + fl[i], a[2] + n[i])
        return out

    def check(self):
        """Synchronise and raise if an asynchronous forward failed on the device."""
        for h in self._handles.values():
            _lib.check(_lib.lib().hn_model_check(h['ptr']), 'hn_model_check')

    def __del__(self):
        try:
            for h in self._handles.values():
                _lib.lib().hn_model_destroy(h['ptr'])
            self._handles.clear()
        except Exception:
            pass
