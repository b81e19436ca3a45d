"""profiles/conv_launches.py maps the convolution kernels of one forward to layers by launch order; check that order
against the model's conv units and the committed H100 tables (no GPU needed)."""
import json
import os
import sys

import pytest

import tc_cases as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'profiles'))
import conv_launches as C  # noqa: E402

TABLES = ('h100_conv_launches_b32.json', 'h100_conv_launches_b32_pdl0.json', 'h100_conv_launches_b32_pdl0_dxr0.json')


def test_expected_launches_follow_the_forward():
    exp = C.expected_launches()
    units = [u[0] for u in T.resnet50_rnn_convs()]
    fused = [n for n in units if n.startswith('layer1') and n.endswith(('conv2', 'conv3'))]
    assert len(exp) == len(units) - len(fused) // 2 + 2
    assert [n for n, _ in exp[-2:]] == ['xproj0', 'xproj1']
    for name, c in exp:
        if c is None:
            assert name.startswith('layer1') and name.endswith('conv2+conv3')
        else:
            assert T.plan(c) is not None, name


@pytest.mark.parametrize('table', TABLES)
def test_committed_table_matches_the_plans(table):
    d = json.load(open(os.path.join(ROOT, 'profiles', table)))
    exp = C.expected_launches()
    assert [r['name'] for r in d['launches']] == [n for n, _ in exp]
    assert 'H100' in d['card']
    dxr_off = d['env'].get('HN_TC_DXR') == '0'
    for r, (name, c) in zip(d['launches'], exp):
        if c is None:
            assert r['kernel'] == 'bott_tc_kernel'
            continue
        p = T.plan(c)
        assert r['kernel'] == ('gemm_tc_kernel' if p['gemm_kernel'] else f'conv_tc_kernel<{p["BN"]}>')
        assert r['num_tiles'] == p['num_tiles'] and r['grid'] == p['grid']
        assert r['dxr'] == (0 if dxr_off else p['dxr'])
