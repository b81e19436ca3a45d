"""Host plan of the tensor-core convolution (hn_conv_tc_plan = what conv_tc_planes launches), no GPU needed:
* every conv_tc_planes launch of the model (tc_cases.model_launches: eval and train forwards, the training step's raw pass
  and data gradients, the LSTM projections) has a plan whose tiles cover the output exactly once;
* coverage guard: every variant key (tc_cases.variant_key) resnet50 or resnet18 reaches at any batch the library accepts
  (tc_cases.ACCEPTED_BATCHES, 1 .. 1024) on a 132-SM H100 SXM or a 114-SM H100 PCIe is reached by a case of the -m gpu
  table (tc_cases.ALL_CASES) planned for the same SM count.  A heuristic change that sends the model into a new variant
  fails here, naming the key and the first launch and batch that reach it, until a unit case for it is added."""
import pytest

import __graft_entry__ as entry
from horizonnet_b200 import _lib
import tc_cases as T

BM = 128


@pytest.fixture(scope='module', autouse=True)
def _built():
    entry.build()


def _check(c, p, sms):
    name = c['name']
    k, (sh, sw), B = c['k'], c['stride'], c['B']
    Ho, Wo = (c['H'] + 2 * c['ph'] - k) // sh + 1, (c['W'] + 2 * c['pw'] - k) // sw + 1
    assert p['n_tiles'] * p['BN'] == c['Cout'], name
    assert p['num_kc'] == k * k * c['Cin'] // 64 and p['seg'] >= 1, name
    if p['mode'] == 0:                            # GEMM rows: every halo-NHWC pixel once
        assert k == 1 and (sh, sw) == (1, 1) and c['in_halo'] == c['out_halo'], name
        assert p['M'] == B * c['H'] * (c['W'] + 2 * c['in_halo']), name
        assert not p['rowbox'] and p['box_rows'] == p['box_imgs'] == 1, name
        m_tiles = -(-p['M'] // BM)
    else:                                         # conv rows: B*Ho rows x Wo columns once
        assert p['M'] == B * Ho and p['tw'] * p['rows_per_tile'] == BM and p['wsegs'] * p['tw'] == Wo, name
        m_tiles = -(-p['M'] // p['rows_per_tile']) * p['wsegs']
        assert (m_tiles // p['wsegs'] - 1) * p['rows_per_tile'] < p['M'] <= m_tiles // p['wsegs'] * p['rows_per_tile'], name
        assert p['parity'] == (sw == 2), name
        assert p['box_rows'] * p['box_imgs'] == p['rows_per_tile'], name     # one TMA box per plane covers the tile
        assert p['rowbox'] == (p['rows_per_tile'] > 1), name
        assert (p['box_imgs'] == 1 and Ho % p['rows_per_tile'] == 0) or p['box_rows'] == Ho, name
        if p['dxr']:                              # the 130-pixel input row of the last tile stays inside Wp
            Wp = c['W'] + 2 * c['in_halo']
            assert p['rows_per_tile'] == 1 and k == 3 and sw == 1, name
            assert p['wsegs'] * BM + (c['in_halo'] - c['pw']) + 2 <= Wp, name
    assert p['num_tiles'] == m_tiles * p['n_tiles'], name
    assert p['grid'] == min(p['num_tiles'], sms), name
    if p['gemm_kernel']:
        assert p['BN'] == 64 and not c['out_f32'] and c['Cin'] <= 256, name
    if c['out_f32']:
        assert not p['gemm_kernel'], name


@pytest.mark.parametrize('sms', T.SM_COUNTS)                 # H100 SXM, H100 PCIe
@pytest.mark.parametrize('B', T.ACCEPTED_BATCHES)
def test_every_model_launch_has_a_plan_covering_its_output_once(B, sms):
    launches = T.model_launches('resnet50', B)
    assert len(launches) == 4 * 68 + 2
    for c in launches:
        p = T.plan(c, sms)
        if c['Cin'] % 64:
            assert p is None, c['name']           # ghc0.3's data gradient (32 channels in) stays on conv_dgrad_f32
            continue
        assert p is not None, (c['name'], _lib.lib().hn_last_error())
        _check(c, p, sms)


@pytest.mark.parametrize('sms', T.SM_COUNTS)
@pytest.mark.parametrize('B', T.ACCEPTED_BATCHES)
def test_every_resnet18_launch_has_a_plan_covering_its_output_once(B, sms):
    launches = T.model_launches('resnet18', B)
    assert len(launches) == 4 * 35 + 2
    planned = 0
    for c in launches:
        p = T.plan(c, sms)
        if c['Cin'] % 64:
            # the narrow height-reduction convs (16 / 32 channels in) run on conv_narrow, their data gradients (and
            # ghc0.0's, 32 channels in) on conv_dgrad_f32
            assert p is None, c['name']
            continue
        assert p is not None, (c['name'], _lib.lib().hn_last_error())
        _check(c, p, sms)
        planned += 1
    # not planned: eval, statistics and raw pass of ghc0.1-3 and ghc1.3 (32 / 16 channels in), the data gradients of
    # ghc0.0-3, ghc1.2-3 and ghc2.3 (32 / 16 / 8 channels out)
    assert planned == 4 * 35 + 2 - 3 * 4 - 7


def test_unit_cases_have_consistent_plans():
    names = [c['name'] for c in T.ALL_CASES]
    assert len(set(names)) == len(names), sorted({n for n in names if names.count(n) > 1})     # the -m gpu test ids
    for sms in T.SM_COUNTS:
        for c in T.ALL_CASES:
            p = T.plan(c, sms)
            assert p is not None, (c['name'], _lib.lib().hn_last_error())
            _check(c, p, sms)


def test_unit_cases_reach_every_variant_key_of_the_model():
    """At each SM count the unit cases, planned for that count, reach every key the model reaches there."""
    report = []
    for sms in T.SM_COUNTS:
        model = {}
        for B in T.ACCEPTED_BATCHES:                      # batch outermost: a failure names the first batch of a key
            for backbone in ('resnet50', 'resnet18'):
                for c in T.model_launches(backbone, B):
                    p = T.plan(c, sms)
                    if p is not None:
                        model.setdefault(T.variant_key(c, p), f"{backbone} {c['name']} @ B={B}")
        cases = {T.variant_key(c, T.plan(c, sms)) for c in T.ALL_CASES}
        missing = {k: v for k, v in model.items() if k not in cases}
        assert not missing, f'{len(missing)} variant key(s) at {sms} SMs without a unit case:\n' + \
            '\n'.join(f'{dict(zip(T.KEY_FIELDS, k))}  (e.g. {v})' for k, v in missing.items())
        report.append(f'{len(model)} at {sms} SMs')
    print(f"forward: variant keys of the model {', '.join(report)}, all reached by the {len(T.ALL_CASES)} unit cases")


def test_dgrad_cases_cover_every_data_gradient_kind_of_the_model():
    model = {}
    for backbone in ('resnet50', 'resnet18'):
        for name, H, W, Ci, Co, k, st in T.conv_units(backbone):
            if T.plan(T.dgrad_launch(name, 1, H, W, Ci, Co, k, st)) is not None:
                model.setdefault(T.dgrad_kind(k, st, Ci, W), f'{backbone} {name}')
    cases = set()
    for B, Ci, H, W, Co, k, st in T.DGRAD_CASES:
        assert T.plan(T.dgrad_launch('case', B, H, W, Ci, Co, k, st)) is not None, (B, Ci, H, W, Co, k, st)
        cases.add(T.dgrad_kind(k, st, Ci, W))
    missing = {kd: v for kd, v in model.items() if kd not in cases}
    assert not missing, '\n'.join(f'k, stride, Cin > 256, W >= 128 = {kd}  (e.g. {v})' for kd, v in missing.items())
    print(f'data gradient: {len(model)} unit kinds of the model, all reached by the {len(T.DGRAD_CASES)} cases')


def test_unit_cases_include_the_named_variants():
    plans = {c['name']: (c, T.plan(c)) for c in T.ALL_CASES}

    def has(pred):
        return any(pred(c, p) for c, p in plans.values())
    tiles_per_cta = lambda p: p['num_tiles'] / p['grid']
    ragged = lambda p: p['mode'] == 0 and p['M'] % BM != 0
    assert has(lambda c, p: p['BN'] == 128 and tiles_per_cta(p) >= 3)
    for res in (False, True):                     # K = 64 with a live L2 prefetch, 3+ tiles per CTA, ragged last M tile
        assert has(lambda c, p: p['gemm_kernel'] and p['num_kc'] == 1 and p['pf'] and c['residual'] == res and
                   tiles_per_cta(p) >= 3 and ragged(p))
    assert has(lambda c, p: p['gemm_kernel'] and p['num_kc'] == 4 and tiles_per_cta(p) >= 3 and ragged(p))
    assert has(lambda c, p: p['gemm_kernel'] and c['Cout'] == 1024 and tiles_per_cta(p) >= 3 and ragged(p))
    for kc in (8, 16, 32):                        # conv_tc_kernel mode 0 at K = 512, 1024, 2048
        assert has(lambda c, p: not p['gemm_kernel'] and p['mode'] == 0 and p['num_kc'] == kc)
    for bn in (64, 128):
        for ws in (1, 2):
            assert has(lambda c, p: p['dxr'] and p['BN'] == bn and p['wsegs'] == ws)
    assert has(lambda c, p: p['BN'] == 32 and c['stride'] == (2, 1) and c['W'] == 256)
    assert has(lambda c, p: p['parity'] and p['box_rows'] > 1 and c['stride'][0] == 2)
    assert has(lambda c, p: p['parity'] and p['box_rows'] == 1)
    assert has(lambda c, p: p['box_imgs'] > 1 and c['B'] in (3, 5) and p['M'] % p['rows_per_tile'] != 0)
    assert has(lambda c, p: p['num_kc'] * 64 == 18432)
    for B in (2, 9):                              # LSTM projection shape, fp32 output
        assert has(lambda c, p: c['out_f32'] and c['in_halo'] == 0 and c['W'] == 256 * B and c['Cin'] == 1024 and
                   c['Cout'] == 4096)


def test_plan_rejects_what_the_kernel_does_not_take():
    bad = [T.launch('cin48', 2, 16, 32, 48, 64, 3, (1, 1)),                       # Cin % 64
           T.launch('cout96', 2, 16, 32, 64, 96, 3, (1, 1)),                      # Cout > 64, not a multiple of 128
           T.launch('w24', 2, 16, 24, 64, 64, 3, (1, 1)),                         # W = 24: not a power-of-two tile width
           T.launch('h3_w32', 2, 3, 32, 64, 64, 3, (1, 1)),                       # Ho = 3, 4 rows per tile: not one box
           T.launch('sh3_w128', 1, 12, 128, 64, 64, 3, (3, 1)),                   # stride 3 along H
           T.launch('f32res', 2, 16, 32, 64, 64, 1, (1, 1), out_f32=True, residual=True)]
    for c in bad:
        assert T.plan(c) is None, c['name']
    assert b'residual' in _lib.lib().hn_last_error()
    assert T.plan(T.launch('ok', 2, 16, 32, 64, 64, 3, (1, 1))) is not None
