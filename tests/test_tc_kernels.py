"""-m gpu: every launch variant of the tensor-core convolution kernels (conv_tc.cu) against fp64, elementwise.

* forward cases of tests/tc_cases.py through hn_conv2d impl 1 (split-plane output) and impl 2 (fp32 output: the epilogue of
  the LSTM projections, of the training step's raw pass and of its data gradients), with the error bound of
  gpu_utils.run_tc_case: NaN-filled output that must be written everywhere, circular halo columns, a canary behind the
  output;
* the tensor-core data gradient of the training step (hn_conv2d_dgrad_tc) against torch.autograd in fp64.
Worst err / bound per case and variant key go to $HN_TEST_RECORD_DIR/tc_errors.jsonl when that variable is set
(gpu_utils.record)."""
import pytest
import torch

import __graft_entry__ as entry
from horizonnet_b200 import _lib
import gpu_utils as gu
import tc_cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    entry.build()
    _lib.lib()


def _key(c):
    return dict(zip(tc_cases.KEY_FIELDS, tc_cases.variant_key(c, tc_cases.plan(c, gu.device_sms()))))


@pytest.mark.parametrize('c', tc_cases.ALL_CASES, ids=lambda c: c['name'])
def test_conv_tc_variant_vs_fp64(c):
    ratio = gu.run_tc_case(c)
    gu.record('tc_errors.jsonl', {'test': 'conv', 'case': c['name'], 'ratio': ratio, 'key': _key(c)})
    assert ratio <= 1.0, ratio


def test_fp32_output_rejects_a_residual():
    x = torch.zeros(1, 1, 8, 66 * 64, device='cuda:0')
    w = torch.zeros(64 * 64, device='cuda:0')
    v = torch.ones(64, device='cuda:0')
    out = torch.zeros(1, 8, 66, 64, device='cuda:0')
    rc = _lib.lib().hn_conv2d(x.data_ptr(), 1, 8, 64, 64, 1, w.data_ptr(), v.data_ptr(), v.data_ptr(), out.data_ptr(), 64,
                              1, 1, 1, 1, 0, 0, 0, out.data_ptr(), 1, 2, None)
    assert rc != 0 and b'residual' in _lib.lib().hn_last_error()


DGRAD_CASES = tc_cases.DGRAD_CASES


@pytest.mark.parametrize('dz_scale', [1.0, 1e-6, 1e-12])
@pytest.mark.parametrize('case', DGRAD_CASES, ids=str)
def test_dgrad_tc_vs_autograd(case, dz_scale):
    B, Ci, H, W, Co, k, st = case
    ratio = gu.run_dgrad_case(B, Ci, H, W, Co, k, st, dz_scale=dz_scale, seed=hash(case) % 1000)
    gu.record('tc_errors.jsonl', {'test': 'dgrad', 'case': list(case[:6]) + list(st), 'dz_scale': dz_scale, 'ratio': ratio})
    assert ratio <= 1.0, ratio


@pytest.mark.parametrize('case', DGRAD_CASES[:4], ids=str)
def test_dgrad_tc_accumulates_into_din(case):
    B, Ci, H, W, Co, k, st = case
    ratio = gu.run_dgrad_case(B, Ci, H, W, Co, k, st, prefill=True, seed=7)
    gu.record('tc_errors.jsonl', {'test': 'dgrad_prefill', 'case': list(case[:6]) + list(st), 'ratio': ratio})
    assert ratio <= 1.0, ratio
    assert gu.run_dgrad_case(B, Ci, H, W, Co, k, st, prefill=True, zero=True, seed=8) == 0.0


def test_dgrad_tc_rejects_shapes_the_kernel_does_not_take():
    z = torch.zeros(1 << 16, device='cuda:0')
    # ghc0.3 (64 -> 32): the transposed conv has 32 input channels
    assert _lib.lib().hn_conv2d_dgrad_tc(1, 4, 16, 64, z.data_ptr(), z.data_ptr(), 32, 3, 3, 2, 1, 1, 1, z.data_ptr(),
                                         None) != 0
    assert b'not supported' in _lib.lib().hn_last_error()
