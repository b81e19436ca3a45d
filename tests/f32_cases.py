"""fp32 CUDA-core convolution launches of the library and the code paths of conv_f32.cu / conv_wgrad_f32 they take (no GPU
needed).

* model_launches -- every conv_f32, conv_wgrad_f32 and conv_dgrad_f32 launch of a backbone, head, batch and tensor-core
                    setting: the eval forward (model.cu forward_encoder / forward_rnn / forward_mlp; fp32 only with
                    tensor_cores off), the training step's forward (train_step.cu walk_forward: the raw pass of every conv
                    unit, the LSTM input projections, the MLP hidden layer) and its backward (rnn_backward: gate recompute
                    accumulated in place, d(layer input) with the second direction accumulated in place, weight gradients;
                    mlp_backward: d(sequence), weight gradient; walk_backward: weight and data gradient of every unit).  With
                    tensor cores on, only what falls through to fp32: hn_conv_tc_plan / hn_wgrad_tc_plan return -1 for it,
                    or (forward convs) Cin is not a multiple of 64 so the layer has no weight planes;
* plan / variant_key -- hn_conv_f32_plan / hn_wgrad_f32_plan and the branches of the kernels a plan selects;
* CASES          -- the -m gpu unit cases of test_conv_f32_variants.py, each the cheapest stand-in for the model launch it is
                    named after; test_conv_f32_variants.py checks that they reach every key the model reaches.

A launch is a dict: op 'conv' (conv_f32 directly), 'wgrad' (conv_wgrad_f32) or 'dgrad' (conv_dgrad_f32: the transposed conv
of the unit on conv_f32 over dz, zero-dilated for a strided unit); B, H, W, Cin, Cout, k, stride, padding and halos describe
the forward convolution (for 'dgrad' the unit whose data gradient it is); kind = what the input operand holds ('act' a
post-ReLU activation, 'lstm' an LSTM state in (-1, 1), 'grad' a signed gradient); residual = 'none', 'separate' (another
tensor) or 'inplace' (the output buffer itself, accumulated into)."""
import ctypes

from horizonnet_b200 import _lib
from horizonnet_b200._spec import c_last

import tc_cases as T
import wgrad_cases as WG

PLAN_FIELDS = ('BM', 'BN', 'grid_m', 'grid_n')
WPLAN_FIELDS = ('kernel', 'gx', 'gy', 'slices', 'm_per_slice')
WGRAD_KERNELS = {2: 'wgrad128', 1: 'wgrad64_vec', 0: 'wgrad64_scalar'}
KEY_FIELDS = ('op', 'tile', 'ragged_m', 'partial_n', 'k', 'stride', 'in_halo', 'out_halo', 'residual', 'relu', 'dilated',
              'pad16', 'kind')
WGRAD_KEY_FIELDS = ('op', 'kernel', 'multi_slice', 'short_last_slice', 'ragged_tile', 'k', 'stride', 'in_halo')


def launch(name, op, B, H, W, Cin, Cout, k, stride, pad=None, in_halo=1, out_halo=1, kind='act', residual='none',
           relu=False):
    ph, pw = (k // 2, k // 2) if pad is None else pad
    return dict(name=name, op=op, B=B, H=H, W=W, Cin=Cin, Cout=Cout, k=k, stride=tuple(stride), ph=ph, pw=pw,
                in_halo=in_halo, out_halo=out_halo, kind=kind, residual=residual, relu=relu)


def out_hw(c):
    return (c['H'] + 2 * c['ph'] - c['k']) // c['stride'][0] + 1, (c['W'] + 2 * c['pw'] - c['k']) // c['stride'][1] + 1


def dgrad_conv(c):
    """The conv_f32 launch of conv_dgrad_f32 for a 'dgrad' launch: Cin <-> Cout (Cout padded to 16), padding k-1-p, stride
    1, in din's geometry (over dz itself for a stride-1 unit, over its dilated copy otherwise), halo 1 both sides."""
    co = -(-c['Cout'] // 16) * 16
    return launch(c['name'], 'conv', c['B'], c['H'], c['W'], co, c['Cin'], c['k'], (1, 1),
                  (c['k'] - 1 - c['ph'], c['k'] - 1 - c['pw']))


def conv_plan(c, sms=T.SMS):
    if c['op'] == 'dgrad':
        c = dgrad_conv(c)
    out = (ctypes.c_int * len(PLAN_FIELDS))()
    (sh, sw), k = c['stride'], c['k']
    rc = _lib.lib().hn_conv_f32_plan(c['B'], c['H'], c['W'], c['Cin'], c['in_halo'], c['Cout'], k, k, sh, sw, c['ph'],
                                     c['pw'], c['out_halo'], sms, out)
    return dict(zip(PLAN_FIELDS, out)) if rc == 0 else None


def wgrad_plan(c, sms=T.SMS):
    out = (ctypes.c_int * len(WPLAN_FIELDS))()
    (sh, sw), k = c['stride'], c['k']
    rc = _lib.lib().hn_wgrad_f32_plan(c['B'], c['H'], c['W'], c['Cin'], c['in_halo'], c['Cout'], k, k, sh, sw, c['ph'],
                                      c['pw'], c['out_halo'], sms, out)
    return dict(zip(WPLAN_FIELDS, out)) if rc == 0 else None


def plan(c, sms=T.SMS):
    return wgrad_plan(c, sms) if c['op'] == 'wgrad' else conv_plan(c, sms)


def pixels(c):
    Ho, Wo = (c['H'], c['W']) if c['op'] == 'dgrad' else out_hw(c)
    return c['B'] * Ho * Wo


def check_plan(c, p):
    """The plan covers the output once: conv -- grid_m tiles of BM pixels and grid_n of BN channels, the last of each
    partly used at most; wgrad -- grid tiles over K = k*k*Cin and Cout, pixel slices of m_per_slice (a multiple of 16)
    with only the last one short."""
    M, name = pixels(c), c['name']
    if c['op'] == 'wgrad':
        tile = 128 if p['kernel'] == 2 else 64
        K = c['k'] ** 2 * c['Cin']
        assert p['kernel'] == (2 if c['Cin'] % 4 == 0 and c['Cout'] >= 128 and K >= 128 else 1 if c['Cin'] % 4 == 0 else 0), name
        assert p['gx'] == -(-K // tile) and p['gy'] == -(-c['Cout'] // tile), name
        assert p['m_per_slice'] % 16 == 0 and p['m_per_slice'] > 0, name
        assert (p['slices'] - 1) * p['m_per_slice'] < M <= p['slices'] * p['m_per_slice'], name
        assert 1 <= p['slices'] <= 64, name
        return
    Cout = c['Cin'] if c['op'] == 'dgrad' else c['Cout']
    assert (p['BM'], p['BN']) in ((128, 128), (128, 64), (64, 64)), name
    assert (p['grid_m'] - 1) * p['BM'] < M <= p['grid_m'] * p['BM'], name
    assert (p['grid_n'] - 1) * p['BN'] < Cout <= p['grid_n'] * p['BN'], name


def variant_key(c, p):
    """The branches of the kernel this launch takes, and what its input operand holds."""
    sh, sw = c['stride']
    M = pixels(c)
    if c['op'] == 'wgrad':
        tile = 128 if p['kernel'] == 2 else 64
        K = c['k'] ** 2 * c['Cin']
        return ('wgrad', WGRAD_KERNELS[p['kernel']],
                p['slices'] > 1,                                       # several pixel slices, reduced with atomics
                M % p['m_per_slice'] != 0,                             # the last slice is short
                K % tile != 0 or c['Cout'] % tile != 0,                # a ragged K or Cout tile
                c['k'], (sh, sw), c['in_halo'], c['kind'])
    Cout = c['Cin'] if c['op'] == 'dgrad' else c['Cout']
    dgrad = c['op'] == 'dgrad'
    return (c['op'], f"{p['BM']}x{p['BN']}",
            M % p['BM'] != 0,                                          # ragged last pixel tile
            Cout % p['BN'] != 0,                                       # Cout below, or not a multiple of, BN
            c['k'], (sh, sw), c['in_halo'], c['out_halo'],
            'inplace' if dgrad else c['residual'], c['relu'],
            (sh, sw) != (1, 1) if dgrad else None,                     # dz zero-dilated to din's geometry
            c['Cout'] % 16 != 0 if dgrad else None,                    # Cout padded to 16 with zero rows
            'grad' if dgrad else c['kind'])


def key_dict(k):
    return dict(zip((WGRAD_KEY_FIELDS + ('kind',)) if k[0] == 'wgrad' else KEY_FIELDS, k))


def _unit_raw_on_tc(c):
    """The training step's raw pass of this unit runs on the tensor cores (train_step.cu unit_forward: the layer has weight
    planes, Cin % 64 == 0, and conv_tc_supported takes the fp32-output conv)."""
    if c['Cin'] % 64:
        return False
    return T.plan(T.launch(c['name'], c['B'], c['H'], c['W'], c['Cin'], c['Cout'], c['k'], c['stride'], out_f32=True)) \
        is not None


def model_launches(backbone, use_rnn, B, tensor_cores):
    out = []
    rows, cl = 256 * B, c_last(backbone)
    units = T.conv_units(backbone)
    # ---- eval forward (forward_encoder): folded BN, ReLU except a downsample, the block's identity before the ReLU
    if not tensor_cores:
        for name, H, W, Ci, Co, k, st in units:
            res = 'separate' if T.has_residual(backbone, name) else 'none'
            out.append(launch(name, 'conv', B, H, W, Ci, Co, k, st, residual=res, relu=not name.endswith('downsample')))
    # ---- training step forward: raw pass z = conv + bias of every unit, then the head's GEMM rows
    for name, H, W, Ci, Co, k, st in units:
        c = launch(name + ':raw', 'conv', B, H, W, Ci, Co, k, st)
        if not tensor_cores or not _unit_raw_on_tc(c):
            out.append(c)
    if use_rnn:
        for layer in range(2):
            out.append(launch(f'bi_rnn.xproj_l{layer}', 'conv', 1, 1, rows, cl if layer == 0 else 1024, 4096, 1, (1, 1),
                              in_halo=0, out_halo=0, kind='act' if layer == 0 else 'lstm'))
    else:
        out.append(launch('linear.0', 'conv', 1, 1, rows, cl, 512, 1, (1, 1), in_halo=0, out_halo=0, relu=True))
    # ---- training step backward, head
    if use_rnn:
        for layer in (1, 0):
            K = cl if layer == 0 else 1024
            out.append(launch(f'bi_rnn.gates_l{layer}', 'conv', 1, 1, rows, 512, 2048, 1, (1, 1), in_halo=0, out_halo=0,
                              kind='lstm', residual='inplace'))
            for w, ci, kind in ((f'weight_ih_l{layer}', K, 'act' if layer == 0 else 'lstm'), (f'weight_hh_l{layer}', 512, 'lstm')):
                c = launch('bi_rnn.' + w, 'wgrad', 1, 1, rows, ci, 2048, 1, (1, 1), in_halo=0, out_halo=0, kind=kind)
                if not tensor_cores or WG.plan(WG.launch(c['name'], 1, 1, rows, ci, 2048, 1, (1, 1))) is None:
                    out.append(c)
            for d, res in ((0, 'none'), (1, 'inplace')):
                out.append(launch(f'bi_rnn.dx_l{layer}_dir{d}', 'conv', 1, 1, rows, 2048, K, 1, (1, 1), in_halo=0,
                                  out_halo=0, kind='grad', residual=res))
    else:
        c = launch('linear.0.weight', 'wgrad', 1, 1, rows, cl, 512, 1, (1, 1), in_halo=0, out_halo=0)
        if not tensor_cores or WG.plan(WG.launch(c['name'], 1, 1, rows, cl, 512, 1, (1, 1))) is None:
            out.append(c)
        out.append(launch('linear.0:dseq', 'conv', 1, 1, rows, 512, cl, 1, (1, 1), in_halo=0, out_halo=0, kind='grad'))
    # ---- training step backward, conv units (walk_backward): weight gradient, data gradient (not of the stem)
    for name, H, W, Ci, Co, k, st in units:
        if not tensor_cores or WG.plan(WG.launch(name, B, H, W, Ci, Co, k, st)) is None:
            out.append(launch(name + ':wgrad', 'wgrad', B, H, W, Ci, Co, k, st))
        if not tensor_cores or T.plan(T.dgrad_launch(name, B, H, W, Ci, Co, k, st)) is None:
            out.append(launch(name + ':dgrad', 'dgrad', B, H, W, Ci, Co, k, st, kind='grad'))
    # the stem's weight gradient (stem_tc / stem_f32 compute the forward; conv_wgrad_f32 its weight gradient on both paths):
    # the NHWC copy of the input with a circular halo of 3
    out.append(launch('stem:wgrad', 'wgrad', B, 512, 1024, 3, 64, 7, (2, 2), in_halo=3))
    return out


# GPU unit cases.  Each stands for the model launch it is named after (backbone prefix r50 / r18, head mlp for the MLP head,
# suffix: batch, tc / f32 for the tensor_cores setting where it matters) at the same variant key on a 132-SM H100 SXM and /
# or a 114-SM H100 PCIe, with batch, height, width of a GEMM row and channels cut as far as the key allows.
CASES = [
    launch('r18.bi_rnn.dx_l0_dir0_b1_tc', 'conv', 1, 1, 64, 64, 256, 1, (1, 1), in_halo=0, out_halo=0, kind='grad'),
    launch('r18.bi_rnn.dx_l0_dir0_b64_tc', 'conv', 1, 1, 8448, 64, 256, 1, (1, 1), in_halo=0, out_halo=0, kind='grad'),
    launch('r18.bi_rnn.dx_l0_dir1_b1_tc', 'conv', 1, 1, 64, 64, 256, 1, (1, 1), in_halo=0, out_halo=0, kind='grad', residual='inplace'),
    launch('r18.bi_rnn.dx_l0_dir1_b64_tc', 'conv', 1, 1, 8448, 64, 256, 1, (1, 1), in_halo=0, out_halo=0, kind='grad', residual='inplace'),
    launch('r18.ghc0.0:dgrad_b1_tc', 'dgrad', 1, 66, 256, 64, 32, 3, (2, 1), kind='grad'),
    launch('r18.ghc0.2:dgrad_b1_tc', 'dgrad', 1, 2, 32, 32, 16, 3, (2, 1), kind='grad'),
    launch('r18.ghc0.2:dgrad_b3_tc', 'dgrad', 3, 22, 256, 32, 16, 3, (2, 1), kind='grad'),
    launch('r18.ghc0.2:wgrad_b1_tc', 'wgrad', 1, 8, 256, 32, 16, 3, (2, 1)),
    launch('r18.ghc0.3:dgrad_b1_tc', 'dgrad', 1, 2, 32, 16, 8, 3, (2, 1), kind='grad'),
    launch('r18.ghc0.3:dgrad_b8_tc', 'dgrad', 5, 14, 256, 16, 8, 3, (2, 1), kind='grad'),
    launch('r18.ghc0.3:raw_b16_tc', 'conv', 14, 10, 256, 16, 8, 3, (2, 1)),
    launch('r18.ghc0.3:raw_b1_tc', 'conv', 1, 2, 64, 16, 8, 3, (2, 1)),
    launch('r18.ghc0.3:wgrad_b1_tc', 'wgrad', 1, 8, 256, 16, 8, 3, (2, 1)),
    launch('r18.ghc0.3_b16_f32', 'conv', 14, 10, 256, 16, 8, 3, (2, 1), relu=True),
    launch('r18.ghc0.3_b1_f32', 'conv', 1, 2, 64, 16, 8, 3, (2, 1), relu=True),
    launch('r18.ghc1.0:wgrad_b2_f32', 'wgrad', 1, 62, 16, 64, 64, 3, (2, 1)),
    launch('r18.ghc1.3:wgrad_b1_tc', 'wgrad', 1, 2, 16, 32, 16, 3, (2, 1)),
    launch('r18.ghc2.0:wgrad_b1_f32', 'wgrad', 1, 10, 64, 128, 128, 3, (2, 1)),
    launch('r18.ghc2.2:wgrad_b1_f32', 'wgrad', 1, 2, 16, 64, 64, 3, (2, 1)),
    launch('r18.ghc3.3:raw_b1_f32', 'conv', 1, 2, 16, 64, 64, 3, (2, 1)),
    launch('r18.ghc3.3:wgrad_b16_f32', 'wgrad', 9, 2, 32, 64, 64, 3, (2, 1)),
    launch('r18.ghc3.3_b1_f32', 'conv', 1, 2, 16, 64, 64, 3, (2, 1), relu=True),
    launch('r18.layer1.0.conv2_b1_f32', 'conv', 1, 66, 256, 64, 64, 3, (1, 1), residual='separate', relu=True),
    launch('r18.layer2.0.conv1:dgrad_b1_f32', 'dgrad', 1, 66, 256, 64, 64, 3, (2, 2), kind='grad'),
    launch('r18.layer2.0.conv1:wgrad_b1_f32', 'wgrad', 1, 6, 256, 32, 128, 3, (2, 2)),
    launch('r18.layer2.0.conv1:wgrad_b2_f32', 'wgrad', 1, 122, 16, 32, 128, 3, (2, 2)),
    launch('r18.layer2.0.conv2_b1_f32', 'conv', 1, 1, 64, 64, 128, 3, (1, 1), residual='separate', relu=True),
    launch('r18.layer2.0.conv2_b3_f32', 'conv', 3, 44, 128, 64, 128, 3, (1, 1), residual='separate', relu=True),
    launch('r18.layer2.0.downsample:dgrad_b1_f32', 'dgrad', 1, 66, 256, 64, 64, 1, (2, 2), kind='grad'),
    launch('r18.layer2.0.downsample:wgrad_b1_f32', 'wgrad', 1, 32, 256, 64, 128, 1, (2, 2)),
    launch('r18.layer2.0.downsample_b1_f32', 'conv', 1, 2, 128, 64, 128, 1, (2, 2)),
    launch('r18.layer3.0.conv1:dgrad_b1_f32', 'dgrad', 1, 2, 32, 128, 64, 3, (2, 2), kind='grad'),
    launch('r18.layer3.0.conv1:wgrad_b1_f32', 'wgrad', 1, 10, 128, 128, 256, 3, (2, 2)),
    launch('r18.layer3.0.downsample:dgrad_b1_f32', 'dgrad', 1, 2, 32, 128, 64, 1, (2, 2), kind='grad'),
    launch('r18.layer3.0.downsample:dgrad_b3_f32', 'dgrad', 3, 44, 128, 128, 64, 1, (2, 2), kind='grad'),
    launch('r18.layer4.0.downsample:wgrad_b1_f32', 'wgrad', 1, 18, 64, 128, 512, 1, (2, 2)),
    launch('r18.layer4.0.downsample:wgrad_b64_f32', 'wgrad', 3, 18, 32, 128, 512, 1, (2, 2)),
    launch('r50.bi_rnn.gates_l1_b1_tc', 'conv', 1, 1, 64, 64, 2048, 1, (1, 1), in_halo=0, out_halo=0, kind='lstm', residual='inplace'),
    launch('r50.bi_rnn.gates_l1_b8_tc', 'conv', 1, 1, 1280, 64, 2048, 1, (1, 1), in_halo=0, out_halo=0, kind='lstm', residual='inplace'),
    launch('r50.bi_rnn.weight_ih_l1_b1_f32', 'wgrad', 1, 1, 16, 128, 2048, 1, (1, 1), in_halo=0, out_halo=0, kind='lstm'),
    launch('r50.bi_rnn.weight_ih_l1_b3_f32', 'wgrad', 1, 1, 384, 128, 2048, 1, (1, 1), in_halo=0, out_halo=0, kind='lstm'),
    launch('r50.bi_rnn.weight_ih_l1_b8_f32', 'wgrad', 1, 1, 1024, 512, 2048, 1, (1, 1), in_halo=0, out_halo=0, kind='lstm'),
    launch('r50.bi_rnn.xproj_l0_b1_tc', 'conv', 1, 1, 64, 64, 4096, 1, (1, 1), in_halo=0, out_halo=0),
    launch('r50.bi_rnn.xproj_l0_b3_tc', 'conv', 1, 1, 768, 64, 4096, 1, (1, 1), in_halo=0, out_halo=0),
    launch('r50.bi_rnn.xproj_l1_b1_tc', 'conv', 1, 1, 64, 64, 4096, 1, (1, 1), in_halo=0, out_halo=0, kind='lstm'),
    launch('r50.bi_rnn.xproj_l1_b3_tc', 'conv', 1, 1, 768, 64, 4096, 1, (1, 1), in_halo=0, out_halo=0, kind='lstm'),
    launch('r50.ghc0.1:wgrad_b1_f32', 'wgrad', 1, 62, 16, 128, 128, 3, (2, 1)),
    launch('r50.ghc0.2:raw_b1_f32', 'conv', 1, 2, 64, 64, 64, 3, (2, 1)),
    launch('r50.ghc0.2_b1_f32', 'conv', 1, 2, 64, 64, 64, 3, (2, 1), relu=True),
    launch('r50.ghc0.3:dgrad_b1_tc', 'dgrad', 1, 2, 32, 64, 32, 3, (2, 1), kind='grad'),
    launch('r50.ghc0.3:wgrad_b8_tc', 'wgrad', 1, 14, 256, 32, 32, 3, (2, 1)),
    launch('r50.ghc1.0:raw_b3_f32', 'conv', 3, 44, 128, 64, 256, 3, (2, 1)),
    launch('r50.ghc1.0_b3_f32', 'conv', 3, 44, 128, 64, 256, 3, (2, 1), relu=True),
    launch('r50.ghc1.3:raw_b64_f32', 'conv', 44, 6, 128, 64, 64, 3, (2, 1)),
    launch('r50.ghc1.3_b64_f32', 'conv', 44, 6, 128, 64, 64, 3, (2, 1), relu=True),
    launch('r50.ghc2.2:dgrad_b16_f32', 'dgrad', 11, 6, 64, 512, 64, 3, (2, 1), kind='grad'),
    launch('r50.ghc2.3:wgrad_b1_f32', 'wgrad', 1, 2, 16, 128, 128, 3, (2, 1)),
    launch('r50.layer1.0.conv1:dgrad_b1_f32', 'dgrad', 1, 66, 256, 64, 64, 1, (1, 1), kind='grad'),
    launch('r50.layer1.0.conv1:raw_b1_f32', 'conv', 1, 66, 256, 64, 64, 1, (1, 1)),
    launch('r50.layer1.0.conv1:wgrad_b1_f32', 'wgrad', 1, 12, 256, 64, 64, 1, (1, 1)),
    launch('r50.layer1.0.conv1_b1_f32', 'conv', 1, 66, 256, 64, 64, 1, (1, 1), relu=True),
    launch('r50.layer1.0.conv2:dgrad_b1_f32', 'dgrad', 1, 66, 256, 64, 64, 3, (1, 1), kind='grad'),
    launch('r50.layer1.0.conv2:raw_b1_f32', 'conv', 1, 66, 256, 64, 64, 3, (1, 1)),
    launch('r50.layer1.0.conv2:wgrad_b1_f32', 'wgrad', 1, 64, 256, 64, 64, 3, (1, 1)),
    launch('r50.layer1.0.conv2_b1_f32', 'conv', 1, 66, 256, 64, 64, 3, (1, 1), relu=True),
    launch('r50.layer2.0.conv2:raw_b1_f32', 'conv', 1, 2, 128, 64, 128, 3, (2, 2)),
    launch('r50.layer2.0.conv2:raw_b3_f32', 'conv', 3, 88, 256, 64, 128, 3, (2, 2)),
    launch('r50.layer2.0.conv2_b1_f32', 'conv', 1, 2, 128, 64, 128, 3, (2, 2), relu=True),
    launch('r50.layer2.0.conv2_b3_f32', 'conv', 3, 88, 256, 64, 128, 3, (2, 2), relu=True),
    launch('r50.layer2.0.conv3:dgrad_b1_f32', 'dgrad', 1, 1, 64, 128, 64, 1, (1, 1), kind='grad'),
    launch('r50.layer2.0.conv3:raw_b1_f32', 'conv', 1, 33, 128, 64, 512, 1, (1, 1)),
    launch('r50.layer2.0.conv3_b1_f32', 'conv', 1, 33, 128, 64, 512, 1, (1, 1), residual='separate', relu=True),
    launch('r50.layer2.0.downsample_b1_f32', 'conv', 1, 66, 256, 64, 512, 1, (2, 2)),
    launch('r50.layer2.1.conv1:dgrad_b1_f32', 'dgrad', 1, 33, 128, 512, 64, 1, (1, 1), kind='grad'),
    launch('r50.layer2.1.conv1:raw_b1_f32', 'conv', 1, 1, 64, 64, 128, 1, (1, 1)),
    launch('r50.layer2.1.conv1_b1_f32', 'conv', 1, 1, 64, 64, 128, 1, (1, 1), relu=True),
    launch('r50.layer2.1.conv2:dgrad_b1_f32', 'dgrad', 1, 1, 64, 128, 64, 3, (1, 1), kind='grad'),
    launch('r50.layer2.1.conv2:dgrad_b3_f32', 'dgrad', 3, 44, 128, 128, 64, 3, (1, 1), kind='grad'),
    launch('r50.layer2.1.conv2:raw_b1_f32', 'conv', 1, 1, 64, 64, 128, 3, (1, 1)),
    launch('r50.layer2.1.conv2:raw_b3_f32', 'conv', 3, 44, 128, 64, 128, 3, (1, 1)),
    launch('r50.layer2.1.conv2_b1_f32', 'conv', 1, 1, 64, 64, 128, 3, (1, 1), relu=True),
    launch('r50.layer2.1.conv2_b3_f32', 'conv', 3, 44, 128, 64, 128, 3, (1, 1), relu=True),
    launch('r50.layer3.0.conv1_b2_f32', 'conv', 2, 33, 128, 64, 256, 1, (1, 1), relu=True),
    launch('r50.layer3.0.conv2:wgrad_b1_f32', 'wgrad', 1, 62, 32, 128, 256, 3, (2, 2)),
    launch('r50.layer3.0.conv3_b1_f32', 'conv', 1, 1, 64, 64, 1024, 1, (1, 1), residual='separate', relu=True),
    launch('r50.layer3.1.conv1:wgrad_b16_f32', 'wgrad', 9, 3, 16, 256, 256, 1, (1, 1)),
    launch('r50.layer3.1.conv2:wgrad_b1_f32', 'wgrad', 1, 31, 16, 128, 256, 3, (1, 1)),
    launch('r50.layer4.0.conv2:dgrad_b3_f32', 'dgrad', 3, 22, 64, 512, 64, 3, (2, 2), kind='grad'),
    launch('r50.layer4.0.conv2:wgrad_b1_f32', 'wgrad', 1, 2, 32, 128, 512, 3, (2, 2)),
    launch('r50.layer4.0.downsample:wgrad_b1_f32', 'wgrad', 1, 2, 32, 128, 2048, 1, (2, 2)),
    launch('r50.layer4.1.conv1:wgrad_b1_f32', 'wgrad', 1, 9, 32, 128, 512, 1, (1, 1)),
    launch('r50.layer4.1.conv2:wgrad_b1_f32', 'wgrad', 1, 1, 16, 128, 512, 3, (1, 1)),
    launch('r50.layer4.1.conv2:wgrad_b3_f32', 'wgrad', 3, 3, 32, 128, 512, 3, (1, 1)),
    launch('r50.mlp.linear.0.weight_b1_f32', 'wgrad', 1, 1, 16, 128, 512, 1, (1, 1), in_halo=0, out_halo=0),
    launch('r50.mlp.linear.0.weight_b3_f32', 'wgrad', 1, 1, 384, 128, 512, 1, (1, 1), in_halo=0, out_halo=0),
    launch('r50.mlp.linear.0.weight_b8_f32', 'wgrad', 1, 1, 268, 128, 512, 1, (1, 1), in_halo=0, out_halo=0),
    launch('r50.mlp.linear.0_b1_tc', 'conv', 1, 1, 64, 64, 512, 1, (1, 1), in_halo=0, out_halo=0, relu=True),
    launch('r50.mlp.linear.0_b32_tc', 'conv', 1, 1, 4352, 64, 512, 1, (1, 1), in_halo=0, out_halo=0, relu=True),
    launch('r50.stem:wgrad_b1_tc', 'wgrad', 1, 4, 1024, 3, 64, 7, (2, 2), in_halo=3),
    # batches between those above and past 64 (132 SMs, then 114 SMs)
    launch('r18.layer2.0.downsample:wgrad_b15_f32', 'wgrad', 1, 24, 256, 64, 128, 1, (2, 2)),
    launch('r50.bi_rnn.weight_ih_l1_b35_f32', 'wgrad', 1, 1, 272, 128, 2048, 1, (1, 1), in_halo=0, out_halo=0, kind='lstm'),
    launch('r50.layer1.0.conv1:wgrad_b55_f32', 'wgrad', 1, 11, 256, 64, 64, 1, (1, 1)),
    launch('r50.ghc3.2_b65_f32', 'conv', 65, 4, 32, 16, 512, 3, (2, 1), relu=True),
    launch('r50.ghc3.2:raw_b65_f32', 'conv', 65, 4, 32, 16, 512, 3, (2, 1)),
    launch('r50.ghc3.3:dgrad_b65_f32', 'dgrad', 65, 2, 32, 512, 256, 3, (2, 1), kind='grad'),
    launch('r18.ghc3.3_b525_f32', 'conv', 525, 2, 32, 16, 64, 3, (2, 1), relu=True),
    launch('r18.ghc3.3:raw_b525_f32', 'conv', 525, 2, 32, 16, 64, 3, (2, 1)),
    launch('r18.layer2.0.downsample:wgrad_b15_f32_h20', 'wgrad', 1, 20, 256, 64, 128, 1, (2, 2)),
    launch('r50.layer1.0.conv1:wgrad_b15_f32', 'wgrad', 1, 10, 256, 64, 64, 1, (1, 1)),
    launch('r50.layer1.0.conv2:wgrad_b25_f32', 'wgrad', 1, 2, 256, 64, 64, 3, (1, 1)),
    launch('r50.ghc3.2_b57_f32', 'conv', 57, 4, 32, 16, 512, 3, (2, 1), relu=True),
    launch('r50.ghc3.2:raw_b57_f32', 'conv', 57, 4, 32, 16, 512, 3, (2, 1)),
    launch('r50.ghc3.3:dgrad_b57_f32', 'dgrad', 57, 2, 32, 512, 256, 3, (2, 1), kind='grad'),
    launch('r18.ghc3.3_b453_f32', 'conv', 453, 2, 32, 16, 64, 3, (2, 1), relu=True),
    launch('r18.ghc3.3:raw_b453_f32', 'conv', 453, 2, 32, 16, 64, 3, (2, 1)),
]
