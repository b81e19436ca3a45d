"""Weight-gradient launches of the training step and the code paths of the tensor-core weight-gradient kernel they take
(wgrad_tc.cu; no GPU needed).

* model_launches -- every conv_wgrad_tc shape the training step of a backbone passes at a batch (train_step.cu): the
                    weight gradient of every conv unit behind the stem (walk_backward), the bi-LSTM's W_ih / W_hh
                    (rnn_backward: 1x1 "convolutions" over one row of 256 * B pixels, Cout = 2048) and the MLP head's
                    first layer (mlp_backward, Cout = 512).  The training step hands the LSTM and head rows over with halo
                    0; hn_conv2d_wgrad_tc and hn_wgrad_tc_plan take halo 1, which leaves the plan unchanged (the pixel
                    tiling depends on dz's geometry only);
* plan / variant_key -- hn_wgrad_tc_plan and the branches of wgrad_tc.cu a plan selects;
* CASES          -- the -m gpu unit cases of test_wgrad_tc_variants.py, each the cheapest stand-in (batch, height or
                    channels cut where the key stays the same) for the model launch it is named after;
                    test_wgrad_tc_variants.py checks that they reach every key the model reaches."""
import ctypes

from horizonnet_b200 import _lib
from horizonnet_b200._spec import c_last

import tc_cases as T

KT = 64                       # pixels per K tile
PLAN_FIELDS = ('tw', 'rpt', 'wsegs', 'box_rows', 'imgs', 'num_kt', 'kt_per_slice', 'slices', 'items', 'ctas')
KEY_FIELDS = ('operand', 'k', 'sh', 'parity', 'tw', 'row_box', 'whole_images', 'strided_rows', 'ragged_last_tile',
              'cin_atoms', 'cout_atoms', 'multi_slice', 'short_last_slice')


def launch(name, B, H, W, Cin, Cout, k, stride, kind='conv'):
    """kind: what the input operand holds in the training step -- 'conv' a post-ReLU activation, 'seq' the feature
    sequence (post-ReLU), 'lstm' H_prev or the first LSTM layer's output (inside (-1, 1))."""
    return dict(name=name, B=B, H=H, W=W, Cin=Cin, Cout=Cout, k=k, stride=tuple(stride), kind=kind)


def model_launches(backbone, B):
    out = [launch(name, B, H, W, Ci, Co, k, st) for name, H, W, Ci, Co, k, st in T.conv_units(backbone)]
    rows = 256 * B
    out.append(launch('bi_rnn.weight_ih_l0', 1, 1, rows, c_last(backbone), 2048, 1, (1, 1), 'seq'))
    out.append(launch('bi_rnn.weight_ih_l1', 1, 1, rows, 1024, 2048, 1, (1, 1), 'lstm'))
    for layer in range(2):
        out.append(launch(f'bi_rnn.weight_hh_l{layer}', 1, 1, rows, 512, 2048, 1, (1, 1), 'lstm'))
    out.append(launch('linear.0.weight', 1, 1, rows, c_last(backbone), 512, 1, (1, 1), 'seq'))
    return out


def plan(c, sms=T.SMS):
    out = (ctypes.c_int * len(PLAN_FIELDS))()
    k, (sh, sw) = c['k'], c['stride']
    rc = _lib.lib().hn_wgrad_tc_plan(c['B'], c['H'], c['W'], c['Cin'], c['Cout'], k, k, sh, sw, k // 2, k // 2, sms, out)
    return dict(zip(PLAN_FIELDS, out)) if rc == 0 else None


def check_plan(c, p):
    """The plan tiles the output pixels (dz's geometry) exactly once: 64-pixel tiles of rows of one image or of whole
    images, at most 64 tiles (256 accumulation steps) per slice, one CTA per work item and slice."""
    name, k, (sh, sw), B = c['name'], c['k'], c['stride'], c['B']
    Ho, Wo = (c['H'] + 2 * (k // 2) - k) // sh + 1, (c['W'] + 2 * (k // 2) - k) // sw + 1
    assert p['tw'] * p['rpt'] == KT and p['wsegs'] * p['tw'] == Wo, name
    assert p['box_rows'] * p['imgs'] == p['rpt'], name                 # rows of one image, or whole images
    assert (p['imgs'] == 1 and Ho % p['rpt'] == 0) or (p['box_rows'] == Ho), name
    rows = B * Ho
    assert p['num_kt'] == -(-rows // p['rpt']) * p['wsegs'] and p['num_kt'] * KT >= rows * Wo, name
    assert 1 <= p['kt_per_slice'] <= 64, name                          # <= 256 accumulation steps per register accumulator
    assert (p['slices'] - 1) * p['kt_per_slice'] < p['num_kt'] <= p['slices'] * p['kt_per_slice'], name
    assert p['items'] == -(-c['Cout'] // 128) * -(-c['Cin'] // 128) * k * k and p['ctas'] == p['items'] * p['slices'], name


def atoms(C):
    """64-channel atoms per 128-channel tile along a channel axis (wgrad_tc_kernel: n_atoms / m_atoms; one atom = the
    wgrad_consume<1> instantiation along Cin, one active consumer warpgroup along Cout)."""
    return tuple(sorted({min(2, (C - c0) // 64) for c0 in range(0, C, 128)}))


def variant_key(c, p):
    """The branches of wgrad_tc.cu this launch takes, and what its input operand holds (an LSTM state has a subnormal lo
    plane everywhere)."""
    sh, sw = c['stride']
    Ho = (c['H'] + 2 * (c['k'] // 2) - c['k']) // sh + 1
    return (c['kind'], c['k'], sh, sw == 2, p['tw'], p['box_rows'] > 1, p['imgs'] > 1,
            sh == 2 and p['box_rows'] * p['imgs'] > 1,                      # input box of every second row (TMA stride)
            (c['B'] * Ho) % p['rpt'] != 0,                                  # the last tile reaches past the last image
            atoms(c['Cin']), atoms(c['Cout']),
            p['slices'] > 1,                                                # pixel slices reduced with red.global.add
            p['num_kt'] % p['kt_per_slice'] != 0)                           # the last slice is short


def key_dict(k):
    return dict(zip(KEY_FIELDS, k))


# GPU unit cases (input geometry, k x k kernel, padding k // 2, halo 1).  Each stands for the model launch it is named after
# (backbone prefix r50 / r18, batch suffix) at the same variant key on a 132-SM H100 SXM and / or a 114-SM H100 PCIe, with
# batch, height and channels cut as far as the key allows.
CASES = [
    launch('r18.ghc1.1_b1', 1, 16, 128, 64, 64, 3, (2, 1)),
    launch('r18.ghc1.1_b16', 13, 2, 128, 64, 64, 3, (2, 1)),
    launch('r18.ghc2.2_b1', 1, 2, 64, 128, 64, 3, (2, 1)),
    launch('r18.ghc2.2_b32', 17, 2, 64, 128, 64, 3, (2, 1)),
    launch('r18.ghc3.3_b1', 1, 2, 32, 128, 64, 3, (2, 1)),
    launch('r18.ghc3.3_b2', 2, 2, 32, 128, 64, 3, (2, 1)),
    launch('r18.ghc3.3_b32', 32, 2, 32, 128, 64, 3, (2, 1)),
    launch('r18.layer2.0.conv1_b1', 1, 16, 256, 64, 128, 3, (2, 2)),
    launch('r18.layer2.0.conv1_b16', 13, 2, 256, 64, 128, 3, (2, 2)),
    launch('r18.layer2.0.downsample_b16', 13, 2, 256, 64, 128, 1, (2, 2)),
    launch('r18.layer2.0.downsample_b3', 3, 8, 256, 64, 128, 1, (2, 2)),
    launch('r50.ghc0.0_b1', 1, 8, 256, 128, 128, 3, (2, 1)),
    launch('r50.ghc0.2_b1', 1, 8, 256, 128, 64, 3, (2, 1)),
    launch('r50.ghc2.0_b1', 1, 2, 64, 128, 128, 3, (2, 1)),
    launch('r50.ghc2.0_b32', 17, 2, 64, 128, 128, 3, (2, 1)),
    launch('r50.ghc3.0_b1', 1, 4, 32, 128, 128, 3, (2, 1)),
    launch('r50.ghc3.0_b1_h2', 1, 2, 32, 128, 128, 3, (2, 1)),
    launch('r50.ghc3.0_b2', 2, 2, 32, 128, 128, 3, (2, 1)),
    launch('r50.ghc3.0_b32', 17, 4, 32, 128, 128, 3, (2, 1)),
    launch('r50.ghc3.0_b64', 34, 2, 32, 128, 128, 3, (2, 1)),
    launch('r50.ghc3.0_b8', 4, 16, 32, 128, 128, 3, (2, 1)),
    launch('r50.layer1.0.conv1_b1', 1, 8, 256, 64, 64, 1, (1, 1)),
    launch('r50.layer1.0.conv1_b3', 3, 2, 256, 64, 64, 1, (1, 1)),
    launch('r50.layer1.0.conv2_b1', 1, 32, 256, 64, 64, 3, (1, 1)),
    launch('r50.layer1.0.conv2_b1_h4', 1, 4, 256, 64, 64, 3, (1, 1)),
    launch('r50.layer1.0.downsample_b1', 1, 8, 256, 64, 128, 1, (1, 1)),
    launch('r50.layer1.0.downsample_b3', 3, 2, 256, 64, 128, 1, (1, 1)),
    launch('r50.layer1.1.conv1_b1', 1, 8, 256, 128, 64, 1, (1, 1)),
    launch('r50.layer1.1.conv1_b3', 3, 2, 256, 128, 64, 1, (1, 1)),
    launch('r50.layer2.0.conv1_b3', 3, 2, 256, 128, 128, 1, (1, 1)),
    launch('r50.layer2.0.conv2_b1', 1, 16, 256, 128, 128, 3, (2, 2)),
    launch('r50.layer2.0.downsample_b3', 3, 8, 256, 128, 128, 1, (2, 2)),
    launch('r50.layer2.1.conv2_b1', 1, 8, 128, 128, 128, 3, (1, 1)),
    launch('r50.layer3.0.conv2_b32', 17, 2, 128, 128, 128, 3, (2, 2)),
    launch('r50.layer3.0.conv3_b16', 13, 2, 64, 128, 128, 1, (1, 1)),
    launch('r50.layer3.0.downsample_b32', 25, 2, 128, 128, 128, 1, (2, 2)),
    launch('r50.layer3.1.conv2_b16', 13, 2, 64, 128, 128, 3, (1, 1)),
    launch('r50.layer4.0.conv2_b1', 1, 4, 64, 128, 128, 3, (2, 2)),
    launch('r50.layer4.0.conv2_b2', 2, 32, 64, 128, 128, 3, (2, 2)),
    launch('r50.layer4.0.conv2_b32', 17, 4, 64, 128, 128, 3, (2, 2)),
    launch('r50.layer4.0.conv3_b1', 1, 2, 32, 128, 128, 1, (1, 1)),
    launch('r50.layer4.0.conv3_b3', 3, 16, 32, 128, 128, 1, (1, 1)),
    launch('r50.layer4.0.conv3_b32', 25, 2, 32, 128, 128, 1, (1, 1)),
    launch('r50.layer4.0.downsample_b1', 1, 4, 64, 128, 128, 1, (2, 2)),
    launch('r50.layer4.0.downsample_b3', 3, 32, 64, 128, 128, 1, (2, 2)),
    launch('r50.layer4.0.downsample_b32', 25, 4, 64, 128, 128, 1, (2, 2)),
    launch('r50.layer4.1.conv2_b1', 1, 2, 32, 128, 128, 3, (1, 1)),
    launch('r50.layer4.1.conv2_b2', 2, 16, 32, 128, 128, 3, (1, 1)),
    launch('r50.layer4.1.conv2_b32', 17, 2, 32, 128, 128, 3, (1, 1)),
    launch('r50.bi_rnn.weight_ih_l0_b1', 1, 1, 256, 128, 128, 1, (1, 1), 'seq'),
    launch('r50.bi_rnn.weight_ih_l0_b8', 1, 1, 1792, 128, 128, 1, (1, 1), 'seq'),
    launch('r50.bi_rnn.weight_ih_l0_b8_w1536', 1, 1, 1536, 128, 128, 1, (1, 1), 'seq'),
    launch('r50.bi_rnn.weight_ih_l1_b1', 1, 1, 256, 128, 128, 1, (1, 1), 'lstm'),
    launch('r50.bi_rnn.weight_ih_l1_b8', 1, 1, 1792, 128, 128, 1, (1, 1), 'lstm'),
    launch('r50.bi_rnn.weight_ih_l1_b8_w1536', 1, 1, 1536, 128, 128, 1, (1, 1), 'lstm'),
    # batches between those above (none past 64 adds a key)
    launch('r18.ghc3.3_b31', 31, 2, 32, 128, 64, 3, (2, 1)),
    launch('r18.ghc3.3_b33', 33, 2, 32, 128, 64, 3, (2, 1)),
    launch('r18.ghc3.3_b34', 34, 2, 32, 128, 64, 3, (2, 1)),
    launch('r50.ghc3.3_b47', 31, 2, 32, 128, 128, 3, (2, 1)),
    launch('r50.ghc3.3_b48', 32, 2, 32, 128, 128, 3, (2, 1)),
    launch('r50.ghc3.3_b49', 33, 2, 32, 128, 128, 3, (2, 1)),
]
