"""Every weight-gradient launch of the training step on the tensor-core kernel (wgrad_tc.cu), by variant key.

CPU (no GPU needed):
* coverage guard: every variant key (wgrad_cases.variant_key) the training step of resnet50 or resnet18 reaches, with either
  head, at any batch the library accepts (tc_cases.ACCEPTED_BATCHES, 1 .. 1024) on a 132-SM H100 SXM or a 114-SM H100
  PCIe, is reached by a unit case of wgrad_cases.CASES planned for the same SM count.  A plan change that sends the model
  into a new variant fails here until a unit case for it is added;
* every unit case and every model launch has a plan that covers its pixels once (test_wgrad_plan.py's invariants).
-m gpu:
* each unit case through hn_conv2d_wgrad_tc against fp64, elementwise, with the bound of gpu_utils.run_wgrad_case; worst
  err / bound per case and variant key go to $HN_TEST_RECORD_DIR/wgrad_errors.jsonl when that variable is set;
* an all-zero dz gives dW = 0 exactly; the fp32 CUDA-core kernel (hn_conv2d_backward) meets the same bound on the same
  inputs."""
import pytest

import __graft_entry__ as entry
from horizonnet_b200 import _lib
import gpu_utils as gu
import tc_cases as T
import wgrad_cases as W

BACKBONES = ('resnet50', 'resnet18')


@pytest.fixture(scope='module', autouse=True)
def _built():
    entry.build()


def _model_keys(sms):
    keys = {}
    for B in T.ACCEPTED_BATCHES:                          # batch outermost: a failure names the first batch of a key
        for backbone in BACKBONES:
            for c in W.model_launches(backbone, B):
                p = W.plan(c, sms)
                if p is not None:
                    keys.setdefault(W.variant_key(c, p), f"{backbone} {c['name']} @ B={B}")
    return keys


@pytest.mark.parametrize('sms', T.SM_COUNTS)
def test_unit_cases_reach_every_variant_key_of_the_model(sms):
    model = _model_keys(sms)
    cases = {W.variant_key(c, W.plan(c, sms)) for c in W.CASES}
    missing = {k: v for k, v in model.items() if k not in cases}
    assert not missing, f'{len(missing)} variant key(s) at {sms} SMs without a unit case:\n' + \
        '\n'.join(f'{W.key_dict(k)}  (e.g. {v})' for k, v in missing.items())
    print(f'weight gradient: {len(model)} variant keys of the model at {sms} SMs, all reached by the {len(W.CASES)} unit cases')


@pytest.mark.parametrize('sms', T.SM_COUNTS)
def test_unit_cases_have_consistent_plans(sms):
    assert len({c['name'] for c in W.CASES}) == len(W.CASES)
    for c in W.CASES:
        p = W.plan(c, sms)
        assert p is not None, (c['name'], _lib.lib().hn_last_error())
        W.check_plan(c, p)


@pytest.mark.parametrize('sms', T.SM_COUNTS)
@pytest.mark.parametrize('backbone', BACKBONES)
def test_every_weight_gradient_launch_of_the_model_has_a_plan(backbone, sms):
    # conv units the kernel does not take: Cout or Cin not a multiple of 64 (resnet50's ghc0.3; resnet18's narrow
    # height-reduction convs) -- their weight gradients stay on conv_wgrad_f32
    on_tc = {'resnet50': 67 + 5, 'resnet18': 28 + 5}[backbone]                  # conv units + LSTM and MLP rows
    for B in T.ACCEPTED_BATCHES:
        n = 0
        for c in W.model_launches(backbone, B):
            p = W.plan(c, sms)
            if c['Cin'] % 64 or c['Cout'] % 64:
                assert p is None, c['name']
                continue
            assert p is not None, (c['name'], B, _lib.lib().hn_last_error())
            W.check_plan(c, p)
            n += 1
        assert n == on_tc, (B, n)


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize('c', W.CASES, ids=lambda c: c['name'])
def test_wgrad_tc_variant_vs_fp64(c):
    ratio = gu.run_wgrad_case(c)
    key = W.key_dict(W.variant_key(c, W.plan(c, gu.device_sms())))
    gu.record('wgrad_errors.jsonl', {'test': 'wgrad', 'case': c['name'], 'sms': gu.device_sms(), 'ratio': ratio,
                                     'key': {k: list(v) if isinstance(v, tuple) else v for k, v in key.items()}})
    assert ratio <= 1.0, ratio


ZERO_DZ_CASES = ('r50.layer1.0.conv1_b1', 'r50.layer4.0.conv2_b32', 'r50.bi_rnn.weight_ih_l1_b8')


@pytest.mark.gpu
@pytest.mark.parametrize('name', ZERO_DZ_CASES)
def test_wgrad_tc_of_a_zero_dz_is_exactly_zero(name):
    assert gu.run_wgrad_case(next(c for c in W.CASES if c['name'] == name), zero_dz=True) == 0.0


@pytest.mark.gpu
def test_wgrad_tc_and_the_fp32_kernel_meet_the_same_bound():
    c = next(c for c in W.CASES if c['name'] == 'r50.layer2.0.conv2_b1')
    ratio, ratio32 = gu.run_wgrad_case(c, with_fp32=True)
    gu.record('wgrad_errors.jsonl', {'test': 'wgrad_vs_fp32', 'case': c['name'], 'ratio': ratio, 'ratio_fp32': ratio32})
    assert ratio <= 1.0 and ratio32 <= 1.0, (ratio, ratio32)
