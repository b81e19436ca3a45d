"""Shapes of HorizonNet('resnet50' / 'resnet18', rnn) and launch plans of the tensor-core convolution (no GPU needed).

* conv_units         -- every conv unit behind the stem of a backbone (resnet50_rnn_convs: resnet50's, shared with
                        test_wgrad_plan.py and profiles/conv_launches.py);
* model_launches     -- every conv_tc_planes launch the library makes for a backbone and a batch: eval forward, train-mode
                        forward (batch statistics pass and real pass), the fp32 raw pass of the training step, the LSTM
                        input projections and the data gradient of every unit (train_step.cu: the transposed conv as a
                        stride-1 conv);
* plan / variant_key -- hn_conv_tc_plan and the code paths of conv_tc.cu a plan selects;
* CASES              -- the unit cases of test_tc_kernels.py; test_conv_tc_plan.py checks that they reach every variant
                        key the model reaches at every batch in ACCEPTED_BATCHES."""
import ctypes

from horizonnet_b200 import _lib
from horizonnet_b200._spec import BACKBONES, c_last

SMS = 132                     # H100 SXM
SM_COUNTS = (132, 114)        # H100 SXM, H100 PCIe
BATCHES = (1, 2, 3, 8, 16, 32, 64)          # the batches the -m gpu tests run the model at
ACCEPTED_BATCHES = range(1, 1025)           # every max_batch hn_model_create_arch accepts: the host censuses plan them all
PLAN_FIELDS = ('gemm_kernel', 'BN', 'mode', 'M', 'tw', 'rows_per_tile', 'wsegs', 'rowbox', 'box_rows', 'box_imgs', 'dxr',
               'parity', 'num_kc', 'seg', 'pf', 'n_tiles', 'num_tiles', 'grid')


def conv_units(backbone):
    """(name, H, W, Cin, Cout, k, stride) of every conv unit behind the stem, input geometry at 512 x 1024, in the order
    of the forward: per block conv1, downsample, conv2 (and conv3 of a Bottleneck), then ghc{s}.{j}."""
    kind, nblk, planes, expansion = BACKBONES[backbone]
    out = []
    H, W, inpl = 128, 256, 64
    for l in range(4):
        p = planes[l]
        for b in range(nblk[l]):
            s = 2 if (b == 0 and l > 0) else 1
            n = f'layer{l + 1}.{b}'
            ds = b == 0 and (s != 1 or inpl != p * expansion)
            if kind == 'bottleneck':                  # v1.5: the stride on conv2
                out.append((n + '.conv1', H, W, inpl, p, 1, (1, 1)))
                if ds:
                    out.append((n + '.downsample', H, W, inpl, p * expansion, 1, (s, s)))
                out.append((n + '.conv2', H, W, p, p, 3, (s, s)))
                out.append((n + '.conv3', H // s, W // s, p, p * expansion, 1, (1, 1)))
            else:                                     # BasicBlock: the stride on conv1
                out.append((n + '.conv1', H, W, inpl, p, 3, (s, s)))
                if ds:
                    out.append((n + '.downsample', H, W, inpl, p, 1, (s, s)))
                out.append((n + '.conv2', H // s, W // s, p, p, 3, (1, 1)))
            inpl, H, W = p * expansion, H // s, W // s
    for s in range(4):
        c = planes[s] * expansion
        ch = (c, c // 2, c // 2, c // 4, c // 8)
        h, w = 128 >> s, 256 >> s
        for j in range(4):
            out.append((f'ghc{s}.{j}', h, w, ch[j], ch[j + 1], 3, (2, 1)))
            h //= 2
    return out


def resnet50_rnn_convs():
    return conv_units('resnet50')


def has_residual(backbone, name):
    """The unit adds the block's identity before its ReLU: a Bottleneck's conv3, a BasicBlock's conv2."""
    last = 'conv3' if BACKBONES[backbone][0] == 'bottleneck' else 'conv2'
    return name.startswith('layer') and name.endswith(last)


def launch(name, B, H, W, Cin, Cout, k, stride, in_halo=1, out_halo=1, out_f32=False, residual=False, pad=None):
    ph, pw = (k // 2, k // 2) if pad is None else pad
    return dict(name=name, B=B, H=H, W=W, Cin=Cin, Cout=Cout, k=k, stride=tuple(stride), ph=ph, pw=pw, in_halo=in_halo,
                out_halo=out_halo, out_f32=out_f32, residual=residual)


def dgrad_launch(name, B, H, W, Cin, Cout, k, stride):
    """The data gradient of a conv unit as train_step.cu launches it: Cin <-> Cout, padding k-1-p, stride 1, over dz or (a
    strided unit) over its zero-dilated copy in the input geometry; fp32 output in the input geometry."""
    p = k // 2
    return launch(name + ':dgrad', B, H, W, Cout, Cin, k, (1, 1), out_f32=True, pad=(k - 1 - p, k - 1 - p))


def model_launches(backbone, B):
    out = []
    for name, H, W, Ci, Co, k, st in conv_units(backbone):
        res = has_residual(backbone, name)
        out.append(launch(name, B, H, W, Ci, Co, k, st, residual=res))                       # eval; train real pass
        out.append(launch(name + ':stats', B, H, W, Ci, Co, k, st))                          # train batch-statistics pass
        out.append(launch(name + ':raw', B, H, W, Ci, Co, k, st, out_f32=True))              # training step raw pass
        out.append(dgrad_launch(name, B, H, W, Ci, Co, k, st))
    for layer in range(2):                                                                   # LSTM input projections
        out.append(launch(f'xproj{layer}', 1, 1, 256 * B, c_last(backbone) if layer == 0 else 1024, 4096, 1, (1, 1), 0, 0,
                          out_f32=True))
    return out


def plan(c, sms=SMS):
    out = (ctypes.c_int * len(PLAN_FIELDS))()
    rc = _lib.lib().hn_conv_tc_plan(c['B'], c['H'], c['W'], c['Cin'], c['in_halo'], c['Cout'], c['k'], c['k'],
                                    c['stride'][0], c['stride'][1], c['ph'], c['pw'], c['out_halo'], int(c['out_f32']),
                                    int(c['residual']), sms, out)
    return dict(zip(PLAN_FIELDS, out)) if rc == 0 else None


def variant_key(c, p):
    """The code paths of conv_tc.cu this launch takes."""
    return (('gemm_tc' if p['gemm_kernel'] else 'conv_tc'), p['BN'], p['mode'], p['dxr'], p['box_rows'] > 1, p['box_imgs'] > 1,
            p['parity'], c['stride'][0], bool(c['out_f32']), bool(c['residual']),
            p['pf'] > 0 and p['num_tiles'] > p['pf'] * p['grid'],              # the L2 prefetch branch is live
            p['num_kc'] % p['seg'] != 0,                                         # last accumulation segment is short
            p['num_tiles'] > p['grid'])                                          # a CTA runs more than one tile


KEY_FIELDS = ('kernel', 'BN', 'mode', 'dxr', 'multi_row_box', 'whole_images', 'parity', 'sh', 'out_f32', 'residual', 'prefetch',
              'short_segment', 'multi_tile')


def case(name, B, H, W, Cin, Cout, k, stride, residual=False, out_f32=False, in_halo=1, out_halo=1, relu=True):
    c = launch(name, B, H, W, Cin, Cout, k, stride, in_halo, out_halo, out_f32, residual)
    c['relu'] = relu and not out_f32
    return c


# Forward unit cases of test_tc_kernels.py (input geometry; k x k kernel, padding k // 2).  Each reaches one or more variant
# keys of the model at 132 SMs; comments name the model layer whose path it stands for.
CASES = [
    # gemm_tc_kernel (1x1, K <= 256, plane output)
    case('gemm_k64_res_pf', 3, 56, 256, 64, 256, 1, (1, 1), residual=True),       # layer1.x.conv3: prefetch, ragged M tile
    case('gemm_k64_pf', 4, 56, 256, 64, 64, 1, (1, 1)),                           # layer1.0.conv1: no residual
    case('gemm_k64_few', 1, 8, 64, 64, 256, 1, (1, 1), residual=True),            # one tile per CTA
    case('gemm_k256', 3, 267, 62, 256, 64, 1, (1, 1)),                            # layer1.1/2.conv1
    case('gemm_k256_res', 3, 67, 62, 256, 256, 1, (1, 1), residual=True),
    case('gemm_k128_res', 3, 33, 62, 128, 512, 1, (1, 1), residual=True),         # layer2.x.conv3
    case('gemm_cout1024', 3, 17, 62, 256, 1024, 1, (1, 1), residual=True),        # layer3.x.conv3: MAX_COUT constants
    # conv_tc_kernel mode 0 (1x1 with K > 256, or fp32 output)
    case('mode0_k512', 2, 16, 64, 512, 128, 1, (1, 1)),                           # layer2/3 conv1
    case('mode0_k1024', 2, 16, 32, 1024, 256, 1, (1, 1)),                         # layer3/4 conv1
    case('mode0_k2048', 2, 8, 32, 2048, 512, 1, (1, 1)),                          # layer4.x.conv1
    case('mode0_k512_res', 2, 8, 32, 512, 2048, 1, (1, 1), residual=True),        # layer4.x.conv3
    case('mode0_bn128', 2, 24, 256, 512, 256, 1, (1, 1)),
    # conv rows: 3x3 stride 1, dx reuse (W >= 128, one output row per tile)
    case('dxr_bn128_w1', 2, 100, 128, 64, 256, 3, (1, 1)),                        # layer2 conv2 (BN = 128, wsegs 1)
    case('dxr_bn64_w2', 2, 16, 256, 64, 64, 3, (1, 1)),                           # layer1 conv2 (wsegs 2)
    case('dxr_bn128_w2', 2, 64, 256, 64, 128, 3, (1, 1)),
    case('dxr_bn64_w1', 1, 16, 128, 128, 128, 3, (1, 1)),
    # conv rows: one box of several rows of one image, and of whole images
    case('rowbox_s1', 2, 16, 32, 256, 256, 3, (1, 1)),                            # layer3 conv2: 4 rows per tile
    case('rowbox_s1_bn128', 8, 16, 32, 256, 256, 3, (1, 1)),
    case('rowbox_s1_k2304', 2, 8, 16, 512, 512, 3, (1, 1)),                       # layer4 conv2: 8 rows per tile
    case('images_s1', 5, 2, 32, 256, 128, 3, (1, 1)),                             # whole images, ragged last tile
    # stride 2 (first blocks of layers 2-4): parity along W, a box of every second input row along H
    case('s2_parity_rowbox2', 2, 32, 64, 128, 128, 3, (2, 2)),                    # layer3.0.conv2 shape family
    case('s2_parity_bn128', 8, 32, 64, 128, 128, 3, (2, 2)),
    case('s2_parity_norowbox', 2, 64, 256, 64, 128, 3, (2, 2)),                   # layer2.0.conv2: 128-wide rows
    case('s2_parity_1x1', 2, 32, 64, 256, 512, 1, (2, 2)),                        # downsample
    case('s2_parity_1x1_bn128', 2, 64, 256, 256, 512, 1, (2, 2)),                 # layer2.0.downsample
    case('s2_parity_images', 3, 8, 32, 512, 256, 3, (2, 2)),                      # layer4.0.conv2: whole images
    # stride (2, 1): height-reduction convs
    case('h2_bn32_w256', 2, 16, 256, 64, 32, 3, (2, 1)),                          # ghc0.3
    case('h2_w256_bn64', 2, 32, 256, 128, 64, 3, (2, 1)),
    case('h2_w256_bn128', 3, 64, 256, 256, 128, 3, (2, 1)),                       # ghc0.0 at small batch
    case('h2_rowbox2', 3, 16, 64, 256, 128, 3, (2, 1)),                           # two rows per tile
    case('h2_images', 3, 4, 32, 512, 256, 3, (2, 1)),                             # H 4 -> 2, whole images, ragged
    case('h2_images_bn128', 8, 2, 32, 1024, 512, 3, (2, 1)),                      # H 2 -> 1
    case('h2_k18432', 2, 2, 32, 2048, 1024, 3, (2, 1)),                           # ghc3.0: K = 18432
]

# fp32-output mode (hn_conv2d impl = 2): the LSTM projections, the raw pass of the training step, the data gradient
F32_CASES = [
    case('xproj_b2', 1, 1, 512, 1024, 4096, 1, (1, 1), out_f32=True, in_halo=0, out_halo=0),
    case('xproj_b9', 1, 1, 2304, 1024, 4096, 1, (1, 1), out_f32=True, in_halo=0, out_halo=0),
    case('f32_1x1_halo1', 3, 13, 62, 64, 256, 1, (1, 1), out_f32=True),           # M = 3*13*64 = 2496: ragged last tile
    case('f32_1x1_halo1_bn128', 2, 56, 256, 64, 256, 1, (1, 1), out_f32=True),
    case('f32_3x3', 2, 16, 128, 128, 128, 3, (1, 1), out_f32=True),
    case('f32_3x3_rowbox', 2, 16, 32, 256, 256, 3, (1, 1), out_f32=True),
    case('f32_3x3_bn128', 2, 48, 128, 128, 256, 3, (1, 1), out_f32=True),
    case('f32_s21', 3, 16, 64, 256, 128, 3, (2, 1), out_f32=True),
    case('f32_s22', 2, 32, 64, 128, 128, 3, (2, 2), out_f32=True),
]

# The cheapest launch of the model (batch 1 .. 1024; input channels cut where the plan stays the same) for each variant key
# the cases above leave out at 132 or 114 SMs, named after the layer.  out_f32 = the training step's raw pass, its data gradients
# (":dgrad": the transposed conv of train_step.cu) and the LSTM projections, all run here through hn_conv2d impl = 2.
MODEL_CASES = [
    case('ghc0.0_b1', 1, 128, 256, 256, 128, 3, (2, 1)),
    case('ghc0.0_raw_b1', 1, 128, 256, 256, 128, 3, (2, 1), out_f32=True),
    case('ghc0.1_b2', 2, 64, 256, 64, 128, 3, (2, 1)),
    case('ghc0.1_b3', 3, 64, 256, 64, 128, 3, (2, 1)),
    case('ghc0.1_dgrad_b1', 1, 64, 256, 64, 128, 3, (1, 1), out_f32=True),
    case('ghc0.1_raw_b2', 2, 64, 256, 64, 128, 3, (2, 1), out_f32=True),
    case('ghc0.1_raw_b3', 3, 64, 256, 64, 128, 3, (2, 1), out_f32=True),
    case('ghc0.2_b8', 8, 32, 256, 64, 64, 3, (2, 1)),
    case('ghc0.2_raw_b8', 8, 32, 256, 64, 64, 3, (2, 1), out_f32=True),
    case('ghc0.3_b32', 32, 16, 256, 64, 32, 3, (2, 1)),
    case('ghc0.3_raw_b1', 1, 16, 256, 64, 32, 3, (2, 1), out_f32=True),
    case('ghc0.3_raw_b32', 32, 16, 256, 64, 32, 3, (2, 1), out_f32=True),
    case('ghc1.0_raw_b3', 3, 64, 128, 256, 256, 3, (2, 1), out_f32=True),
    case('ghc1.1_b3', 3, 32, 128, 256, 256, 3, (2, 1)),
    case('ghc1.1_dgrad_b3', 3, 32, 128, 256, 256, 3, (1, 1), out_f32=True),
    case('ghc1.1_dgrad_b1', 1, 32, 128, 256, 256, 3, (1, 1), out_f32=True),
    case('ghc1.1_raw_b3', 3, 32, 128, 256, 256, 3, (2, 1), out_f32=True),
    case('ghc1.2_b1', 1, 16, 128, 256, 128, 3, (2, 1)),
    case('ghc1.2_dgrad_b3', 3, 16, 128, 64, 256, 3, (1, 1), out_f32=True),
    case('ghc1.2_raw_b1', 1, 16, 128, 256, 128, 3, (2, 1), out_f32=True),
    case('ghc1.3_raw_b1', 1, 8, 128, 64, 64, 3, (2, 1), out_f32=True),
    case('ghc2.0_b3', 3, 32, 64, 256, 512, 3, (2, 1)),
    case('ghc2.0_b8', 8, 32, 64, 256, 512, 3, (2, 1)),
    case('ghc2.0_dgrad_b1', 1, 32, 64, 256, 1024, 3, (1, 1), out_f32=True),
    case('ghc2.0_raw_b3', 3, 32, 64, 256, 512, 3, (2, 1), out_f32=True),
    case('ghc2.0_raw_b8', 8, 32, 64, 256, 512, 3, (2, 1), out_f32=True),
    case('ghc2.1_b8', 8, 16, 64, 256, 512, 3, (2, 1)),
    case('ghc2.1_raw_b8', 8, 16, 64, 256, 512, 3, (2, 1), out_f32=True),
    case('ghc2.3_dgrad_b1', 1, 4, 64, 64, 256, 3, (1, 1), out_f32=True),
    case('ghc2.3_dgrad_b32', 32, 4, 64, 64, 256, 3, (1, 1), out_f32=True),
    case('ghc3.2_raw_b1', 1, 4, 32, 256, 512, 3, (2, 1), out_f32=True),
    case('ghc3.3_dgrad_b1', 1, 2, 32, 256, 512, 3, (1, 1), out_f32=True),
    case('ghc3.3_raw_b1', 1, 2, 32, 256, 256, 3, (2, 1), out_f32=True),
    case('layer1.0.conv1_b1', 1, 128, 256, 64, 64, 1, (1, 1)),
    case('layer1.0.conv1_raw_b1', 1, 128, 256, 64, 64, 1, (1, 1), out_f32=True),
    case('layer1.0.conv2_b1', 1, 128, 256, 64, 64, 3, (1, 1)),
    case('layer2.0.conv2_b2', 2, 128, 256, 64, 128, 3, (2, 2)),
    case('layer2.0.conv2_b3', 3, 128, 256, 64, 128, 3, (2, 2)),
    case('layer2.0.conv2_raw_b1', 1, 128, 256, 64, 128, 3, (2, 2), out_f32=True),
    case('layer2.0.conv2_raw_b2', 2, 128, 256, 64, 128, 3, (2, 2), out_f32=True),
    case('layer2.0.conv2_raw_b3', 3, 128, 256, 64, 128, 3, (2, 2), out_f32=True),
    case('layer2.0.downsample_raw_b1', 1, 128, 256, 256, 512, 1, (2, 2), out_f32=True),
    case('layer2.1.conv2_b2', 2, 64, 128, 64, 128, 3, (1, 1)),
    case('layer3.0.conv1_b1', 1, 64, 128, 512, 256, 1, (1, 1)),
    case('layer3.0.conv2_b3', 3, 64, 128, 256, 256, 3, (2, 2)),
    case('layer3.0.conv2_dgrad_b1', 1, 64, 128, 256, 256, 3, (1, 1), out_f32=True),
    case('layer3.0.conv2_raw_b3', 3, 64, 128, 256, 256, 3, (2, 2), out_f32=True),
    case('layer3.0.downsample_b1', 1, 64, 128, 256, 1024, 1, (2, 2)),
    case('layer3.0.downsample_raw_b1', 1, 64, 128, 256, 1024, 1, (2, 2), out_f32=True),
    case('layer3.1.conv2_b3', 3, 32, 64, 256, 256, 3, (1, 1)),
    case('layer3.1.conv2_b8', 8, 32, 64, 256, 256, 3, (1, 1)),
    case('layer3.1.conv2_raw_b3', 3, 32, 64, 256, 256, 3, (1, 1), out_f32=True),
    case('layer4.0.conv1_raw_b1', 1, 32, 64, 256, 512, 1, (1, 1), out_f32=True),
    case('layer4.0.conv2_dgrad_b3', 3, 32, 64, 256, 512, 3, (1, 1), out_f32=True),
    case('layer4.0.conv3_b2', 2, 16, 32, 256, 2048, 1, (1, 1), residual=True),
    case('layer4.0.conv3_dgrad_b1', 1, 16, 32, 256, 512, 1, (1, 1), out_f32=True),
    case('layer4.0.conv3_stats_b1', 1, 16, 32, 256, 2048, 1, (1, 1)),
    case('layer4.0.downsample_b3', 3, 32, 64, 256, 2048, 1, (2, 2)),
    case('layer4.0.downsample_raw_b1', 1, 32, 64, 256, 2048, 1, (2, 2), out_f32=True),
    case('layer4.0.downsample_raw_b3', 3, 32, 64, 256, 2048, 1, (2, 2), out_f32=True),
    case('layer4.1.conv2_b8', 8, 16, 32, 256, 512, 3, (1, 1)),
    # batches 16 and 64, a 114-SM H100 PCIe and resnet18 (prefix r18.): batch and input channels cut where the key stays
    case('ghc2.2_b32', 29, 8, 64, 64, 256, 3, (2, 1)),
    case('ghc2.2_raw_b32', 29, 8, 64, 64, 256, 3, (2, 1), out_f32=True),
    case('ghc2.3_b1', 1, 4, 64, 64, 128, 3, (2, 1)),
    case('ghc2.3_b64', 58, 4, 64, 64, 128, 3, (2, 1)),
    case('ghc2.3_dgrad_b32_cut17', 17, 4, 64, 64, 256, 3, (1, 1), out_f32=True),   # batch cut to 17
    case('ghc2.3_raw_b1', 1, 4, 64, 64, 128, 3, (2, 1), out_f32=True),
    case('ghc2.3_raw_b64', 58, 4, 64, 64, 128, 3, (2, 1), out_f32=True),
    case('ghc3.1_b32', 17, 8, 32, 64, 1024, 3, (2, 1)),
    case('ghc3.1_raw_b32', 17, 8, 32, 64, 1024, 3, (2, 1), out_f32=True),
    case('ghc3.2_b32', 29, 4, 32, 256, 512, 3, (2, 1)),
    case('ghc3.2_b64', 57, 4, 32, 256, 512, 3, (2, 1)),
    case('ghc3.2_dgrad_b32', 17, 4, 32, 64, 1024, 3, (1, 1), out_f32=True),
    case('ghc3.2_raw_b32', 29, 4, 32, 256, 512, 3, (2, 1), out_f32=True),
    case('ghc3.2_raw_b64', 57, 4, 32, 256, 512, 3, (2, 1), out_f32=True),
    case('ghc3.3_dgrad_b32', 29, 2, 32, 256, 512, 3, (1, 1), out_f32=True),
    case('ghc3.3_dgrad_b64', 57, 2, 32, 256, 512, 3, (1, 1), out_f32=True),
    case('layer2.1.conv1_b1', 1, 64, 128, 64, 128, 1, (1, 1)),
    case('r18.ghc2.3_b1', 1, 4, 64, 64, 32, 3, (2, 1)),
    case('r18.ghc2.3_raw_b1', 1, 4, 64, 64, 32, 3, (2, 1), out_f32=True),
    case('r18.ghc3.3_b1', 1, 2, 32, 64, 64, 3, (2, 1)),
    case('r18.ghc3.3_dgrad_b1', 1, 2, 32, 64, 128, 3, (1, 1), out_f32=True),
    case('r18.ghc3.3_raw_b1', 1, 2, 32, 64, 64, 3, (2, 1), out_f32=True),
    case('r18.layer1.0.conv2_b1', 1, 128, 256, 64, 64, 3, (1, 1), residual=True),
    case('r18.layer2.0.conv2_b1', 1, 64, 128, 64, 128, 3, (1, 1), residual=True),
    case('r18.layer2.0.conv2_b2', 2, 64, 128, 64, 128, 3, (1, 1), residual=True),
    case('r18.layer2.0.conv2_b3', 3, 64, 128, 64, 128, 3, (1, 1), residual=True),
    case('r18.layer3.0.conv2_b8', 4, 32, 64, 256, 256, 3, (1, 1), residual=True),
    case('r18.layer4.0.conv2_b1', 1, 16, 32, 256, 512, 3, (1, 1), residual=True),
    case('r18.layer4.0.conv2_b16', 9, 16, 32, 256, 512, 3, (1, 1), residual=True),
    case('r18.layer4.0.conv2_b8', 5, 16, 32, 256, 512, 3, (1, 1), residual=True),
    case('r18.layer4.0.downsample_b16', 9, 32, 64, 64, 512, 1, (2, 2)),
    case('r18.layer4.0.downsample_b8', 5, 32, 64, 64, 512, 1, (2, 2)),
    case('r18.layer4.0.downsample_raw_b1', 1, 32, 64, 256, 512, 1, (2, 2), out_f32=True),
    case('r18.layer4.0.downsample_raw_b16', 9, 32, 64, 64, 512, 1, (2, 2), out_f32=True),
    case('r18.layer4.0.downsample_raw_b8', 5, 32, 64, 64, 512, 1, (2, 2), out_f32=True),
    # batches between those above and past 64, each named after the first batch that reaches its key; input channels cut
    # where the key stays.  Past 64 only the small height-reduction convs (ghc2.3, ghc3.2, ghc3.3) change their path:
    # more tiles than CTAs (multi_tile), and BN 128 once the 64-channel tiles alone would fill the grid.
    # 132 SMs
    case('ghc3.2_b33', 33, 4, 32, 256, 512, 3, (2, 1)),
    case('ghc3.2_raw_b33', 33, 4, 32, 256, 512, 3, (2, 1), out_f32=True),
    case('ghc3.3_dgrad_b33', 33, 2, 32, 256, 512, 3, (1, 1), out_f32=True),
    case('ghc3.2_b67', 67, 4, 32, 256, 512, 3, (2, 1)),
    case('ghc3.2_raw_b67', 67, 4, 32, 256, 512, 3, (2, 1), out_f32=True),
    case('ghc3.3_dgrad_b67', 67, 2, 32, 256, 512, 3, (1, 1), out_f32=True),
    case('ghc3.3_b133', 133, 2, 32, 256, 256, 3, (2, 1)),
    case('ghc3.3_raw_b133', 133, 2, 32, 256, 256, 3, (2, 1), out_f32=True),
    case('ghc3.3_b217', 217, 2, 32, 256, 256, 3, (2, 1)),
    case('ghc3.3_raw_b217', 217, 2, 32, 256, 256, 3, (2, 1), out_f32=True),
    case('ghc3.3_b265', 265, 2, 32, 256, 256, 3, (2, 1)),
    case('ghc3.3_raw_b265', 265, 2, 32, 256, 256, 3, (2, 1), out_f32=True),
    case('r18.layer3.0.conv1_b4', 4, 64, 128, 64, 256, 3, (2, 2)),
    case('r18.layer3.0.conv1_raw_b4', 4, 64, 128, 64, 256, 3, (2, 2), out_f32=True),
    case('r18.ghc2.1_b17', 17, 16, 64, 64, 128, 3, (2, 1)),
    case('r18.ghc2.1_raw_b17', 17, 16, 64, 64, 128, 3, (2, 1), out_f32=True),
    case('r18.ghc2.3_b133', 133, 4, 64, 64, 32, 3, (2, 1)),
    case('r18.ghc2.3_raw_b133', 133, 4, 64, 64, 32, 3, (2, 1), out_f32=True),
    case('r18.ghc3.3_dgrad_b133', 133, 2, 32, 64, 128, 3, (1, 1), out_f32=True),
    case('r18.ghc3.3_dgrad_b219', 219, 2, 32, 64, 128, 3, (1, 1), out_f32=True),
    case('r18.ghc3.3_dgrad_b265', 265, 2, 32, 64, 128, 3, (1, 1), out_f32=True),
    case('r18.ghc3.3_b529', 529, 2, 32, 64, 64, 3, (2, 1)),
    case('r18.ghc3.3_raw_b529', 529, 2, 32, 64, 64, 3, (2, 1), out_f32=True),
    # 114 SMs
    case('ghc1.2_b14', 14, 16, 128, 256, 128, 3, (2, 1)),
    case('ghc1.2_raw_b14', 14, 16, 128, 256, 128, 3, (2, 1), out_f32=True),
    case('ghc1.3_dgrad_b14', 14, 8, 128, 64, 128, 3, (1, 1), out_f32=True),
    case('ghc2.1_b7', 7, 16, 64, 256, 512, 3, (2, 1)),
    case('ghc2.1_raw_b7', 7, 16, 64, 256, 512, 3, (2, 1), out_f32=True),
    case('ghc2.3_dgrad_b28', 28, 4, 64, 64, 256, 3, (1, 1), out_f32=True),
    case('ghc3.2_b55', 55, 4, 32, 256, 512, 3, (2, 1)),
    case('ghc3.2_raw_b55', 55, 4, 32, 256, 512, 3, (2, 1), out_f32=True),
    case('ghc3.3_dgrad_b55', 55, 2, 32, 256, 512, 3, (1, 1), out_f32=True),
    case('ghc3.3_b113', 113, 2, 32, 256, 256, 3, (2, 1)),
    case('ghc3.3_raw_b113', 113, 2, 32, 256, 256, 3, (2, 1), out_f32=True),
    case('ghc3.3_b229', 229, 2, 32, 256, 256, 3, (2, 1)),
    case('ghc3.3_raw_b229', 229, 2, 32, 256, 256, 3, (2, 1), out_f32=True),
    case('layer4.0.conv2_b7', 7, 32, 64, 256, 512, 3, (2, 2)),
    case('layer4.0.conv2_raw_b7', 7, 32, 64, 256, 512, 3, (2, 2), out_f32=True),
    case('layer4.1.conv2_b7', 7, 16, 32, 256, 512, 3, (1, 1)),
    case('layer4.1.conv2_raw_b7', 7, 16, 32, 256, 512, 3, (1, 1), out_f32=True),
    case('r18.ghc2.1_b28', 28, 16, 64, 64, 128, 3, (2, 1)),
    case('r18.ghc2.1_raw_b28', 28, 16, 64, 64, 128, 3, (2, 1), out_f32=True),
    case('r18.ghc2.3_b115', 115, 4, 64, 64, 32, 3, (2, 1)),
    case('r18.ghc2.3_raw_b115', 115, 4, 64, 64, 32, 3, (2, 1), out_f32=True),
    case('r18.ghc3.3_dgrad_b115', 115, 2, 32, 64, 128, 3, (1, 1), out_f32=True),
    case('r18.ghc3.3_dgrad_b229', 229, 2, 32, 64, 128, 3, (1, 1), out_f32=True),
    case('r18.ghc3.3_b457', 457, 2, 32, 64, 64, 3, (2, 1)),
    case('r18.ghc3.3_raw_b457', 457, 2, 32, 64, 64, 3, (2, 1), out_f32=True),
    case('r18.layer4.0.conv2_b7', 7, 16, 32, 256, 512, 3, (1, 1), residual=True),
]

ALL_CASES = CASES + F32_CASES + MODEL_CASES

# Data gradients of the training step through hn_conv2d_dgrad_tc (test_tc_kernels.py): B, Cin, H, W, Cout, k, stride of the
# unit.  Together they cover every data-gradient unit kind (dgrad_kind) of resnet50 and resnet18; the first four are
# also run accumulating into a prefilled din.
DGRAD_CASES = [
    (2, 64, 32, 128, 64, 3, (1, 1)),          # 3x3 stride 1 (layer1 conv2): dx reuse
    (2, 128, 32, 64, 128, 3, (2, 2)),         # 3x3 stride 2 (layer2-4 .0.conv2): dilated dz
    (2, 256, 32, 64, 512, 1, (2, 2)),         # 1x1 stride 2 (downsample)
    (3, 256, 16, 64, 128, 3, (2, 1)),         # 3x3 stride (2, 1) (height reduction)
    (2, 512, 16, 32, 128, 1, (1, 1)),         # 1x1 stride 1, Cin > 256 (conv1 of layer3)
    (2, 256, 8, 64, 1024, 1, (1, 1)),         # layer3.x.conv3
    (1, 64, 8, 256, 256, 1, (1, 1)),          # layer1.0.conv3, layer1.0.downsample: W = 256
    (1, 512, 8, 128, 128, 1, (1, 1)),         # layer2.x.conv1: Cin > 256, W = 128
    (1, 64, 16, 256, 128, 1, (2, 2)),         # resnet18 layer2.0.downsample
    (2, 1024, 8, 64, 2048, 1, (2, 2)),        # layer4.0.downsample
    (1, 512, 8, 128, 1024, 1, (2, 2)),        # layer3.0.downsample
    (2, 256, 8, 64, 256, 3, (1, 1)),          # layer3.x.conv2: W = 64
    (2, 512, 4, 32, 512, 3, (1, 1)),          # layer4.x.conv2 (both backbones): W = 32
    (2, 64, 16, 256, 128, 3, (2, 2)),         # resnet18 layer2.0.conv1: 3x3 stride 2, 64 -> 128
    (2, 512, 8, 64, 512, 3, (2, 2)),          # layer4.0.conv2
    (2, 128, 8, 256, 64, 3, (2, 1)),          # ghc0.2: W = 256
    (1, 512, 8, 128, 256, 3, (2, 1)),         # ghc1.0: Cin > 256, W = 128
    (2, 512, 8, 64, 512, 3, (2, 1)),          # ghc2.1
]


def dgrad_kind(k, stride, Cin, W):
    """The unit kinds of the data gradient: kernel size, stride, Cin above 256 (the transposed conv's Cout: two or more
    output-channel tiles of 128) and input rows of 128 or more pixels (one conv row per tile, dx reuse)."""
    return k, tuple(stride), Cin > 256, W >= 128
