"""Every launch layout of the bi-LSTM recurrence (lstm_cluster.cu: lstm_cluster_kernel), by variant key, against a
teacher-forced fp64 replay.

CPU (no GPU needed):
* census: every key (lstm_cases.variant_key) that the model's recurrence launches (eval forward, training forward, TTA;
  both layers, T = 256, every batch in tc_cases.ACCEPTED_BATCHES, 1 .. 1024) or hn_lstm_layer at T = 1, 2, 3 reach on a
  device with 2 .. 8 co-resident clusters is a unit case of lstm_cases.CASES, and batch_for finds its batch there.  A
  failure names the missing key and the first launch and batch that reach it;
* every plan owns each column once, and takes two groups per cluster exactly when one each would not fit in one wave;
* hn_lstm_plan rejects T < 1, B < 1 and fewer than 2 co-resident clusters;
* the bound of gpu_utils.lstm_bound holds for a CPU emulation of the kernel's arithmetic, and fails it with a cross
  product dropped or with h_{t-2} fed in where h_{t-1} belongs.
-m gpu, on the device's own cluster count (hn_lstm_plan with max_clusters = -1):
* each unit case through hn_lstm_layer with the init inputs: its plan has the key it is named after, the output is fully
  written, finite and nothing is written past it, every element is within the bound; worst err / bound per case go to
  $HN_TEST_RECORD_DIR/lstm_errors.jsonl when that variable is set;
* the trained, saturated and small inputs at the model's T = 256 and B = 32 (the benchmark) and 64 (the training step's
  largest batch);
* each column equals the same column run alone at B = 1, bit for bit;
* direction mirror: xproj reversed in time with its direction halves swapped and W_hh of the two directions swapped gives
  the output reversed in time with its halves swapped, bit for bit."""
import ctypes

import pytest
import torch

import __graft_entry__ as entry
from horizonnet_b200 import _lib
import gpu_utils as gu
import lstm_cases as L

DEV = 'cuda:0'


@pytest.fixture(scope='module', autouse=True)
def _built():
    entry.build()


def _census(max_clusters):
    """{key: a launch that reaches it} of the model and the ABI's short sequences on max_clusters clusters."""
    keys = {}
    for B in L.ACCEPTED_BATCHES:
        for c in L.model_launches(B) + L.abi_launches(B):
            p = L.plan(c['T'], c['B'], max_clusters)
            assert p is not None, (c, _lib.lib().hn_last_error())
            L.check_plan(c['T'], c['B'], p)
            keys.setdefault(L.variant_key(c['T'], p), f"{c['name']} @ B={B}")
    return keys


@pytest.mark.parametrize('max_clusters', L.MAX_CLUSTERS)
def test_unit_cases_reach_every_variant_key_of_the_model(max_clusters):
    census = _census(max_clusters)
    missing = {k: v for k, v in census.items() if L.key_name(k) not in L.CASES or L.batch_for(k, max_clusters) is None}
    assert not missing, f'{len(missing)} variant key(s) at {max_clusters} clusters without a unit case:\n' + \
        '\n'.join(f'{L.key_dict(k)}  (e.g. {v})' for k, v in missing.items())
    for name in L.CASES:
        key = L.CASE_KEYS[name]
        B = L.batch_for(key, max_clusters)
        if B is not None:
            T = L.T_FOR_CLASS[key[5]]
            assert L.variant_key(T, L.plan(T, B, max_clusters)) == key
    print(f'lstm: {len(census)} variant keys at {max_clusters} clusters, all reached by the unit cases')


def test_the_census_reaches_the_h100_sxm_layouts():
    """On the 7 clusters of an H100 SXM: the benchmark's batch 32 runs on 4 two-group clusters in one wave, B = 33 .. 39
    ends on a one-group cluster with a partial group, and every batch from 49 (7 groups of 8 columns: 4 cluster pairs,
    one more than 7 clusters hold) to the largest the library accepts needs a second wave or more."""
    assert L.plan(256, 32, 7) == dict(max_clusters=7, ngroups=4, gpc=2, clusters=4, last_cluster_groups=2,
                                      last_group_cols=8, waves=1)
    for B in range(33, 40):
        k = L.key_dict(L.variant_key(256, L.plan(256, B, 7)))
        assert k['gpc'] == 2 and k['last_cluster_one_group'] and k['partial_group'] and not k['second_wave'], B
    plans = {B: L.plan(256, B, 7) for B in L.ACCEPTED_BATCHES}
    first = min(B for B, p in plans.items() if p['clusters'] > p['max_clusters'])
    assert first == 49 and plans[first]['clusters'] == 8
    assert [B for B, p in plans.items() if p['waves'] > 1] == list(range(first, L.ACCEPTED_BATCHES[-1] + 1))
    assert len(L.CASES) == len(set(L.CASES)) == len(L.CASE_KEYS)


@pytest.mark.parametrize('max_clusters', L.MAX_CLUSTERS + (9, 16, 132))
def test_two_groups_per_cluster_exactly_when_one_each_would_not_fit(max_clusters):
    for T in (1, 2, 3, 256):
        for B in L.ACCEPTED_BATCHES:
            p = L.plan(T, B, max_clusters)
            L.check_plan(T, B, p)
            assert (p['gpc'] == 1) == (2 * p['ngroups'] <= max_clusters), (T, B, p)
            assert p['max_clusters'] == max_clusters


def test_hn_lstm_plan_rejects_bad_arguments():
    lib = _lib.lib()
    out = (ctypes.c_int * 7)()
    for T, B, mc in ((0, 1, 7), (-3, 8, 7), (256, 0, 7), (256, -1, 7), (256, 8, 1)):
        assert lib.hn_lstm_plan(T, B, mc, out) == -1, (T, B, mc)
        assert lib.hn_last_error(), (T, B, mc)
    lib.hn_lstm_plan(256, 8, 1, out)
    assert b'2 are needed' in lib.hn_last_error()
    assert lib.hn_lstm_plan(256, 8, 2, None) == -1


# ---- the bound against a CPU emulation of the kernel's arithmetic
def _row_scale(absmax):
    """lstm_cluster.cu row_scale: the power of two that puts max|w| of a row into (2^13, 2^14] (1 for a zero row)."""
    e = torch.frexp(16384.0 / absmax.clamp_min(1e-30))[1]
    return torch.where(absmax > 0, torch.ldexp(torch.ones_like(absmax), e - 1), torch.ones_like(absmax))


def _split(v):
    hi = v.half().float()
    return hi, (v - hi).half().float()


def _emulate(xp, W, mutation=None):
    """One direction in step order, as lstm_cluster_kernel computes it: fp16 hi / lo of the row-scaled W and of 256 h, the
    three products hi*hi + hi*lo + lo*hi with fp32 sums, fmaf(sum, unscale, xp), the cell in fp32.  mutation: 'hl' or 'lh'
    drops that product, 'stale' feeds h_{t-2} into step t."""
    T, B, _ = xp.shape
    sc = _row_scale(W.abs().amax(1))
    whi, wlo = _split(W * sc[:, None])
    unscale = 1.0 / (sc * 256.0)
    h = hold = c = torch.zeros(B, 512)
    out = torch.empty(T, B, 512)
    for t in range(T):
        hh, hl = _split((hold if mutation == 'stale' else h) * 256.0)
        s = hh @ whi.t()
        if mutation != 'hl':
            s = s + hl @ whi.t()
        if mutation != 'lh':
            s = s + hh @ wlo.t()
        pre = torch.addcmul(xp[t], s, unscale[None])
        i, f, g, o = pre.chunk(4, 1)
        sig = lambda x: 1.0 / (1.0 + torch.exp(-x))
        c = sig(f) * c + sig(i) * torch.tanh(g)
        hold, h = h, sig(o) * torch.tanh(c)
        out[t] = h
    return out


def _emulated_ratio(kind, mutation):
    xproj, W = gu.lstm_inputs(kind, 64, 4, 7)
    xp = xproj[..., :2048]
    h = _emulate(xp, W[0], mutation)
    ref, bound = gu.lstm_bound(h, xp, W[0])
    return gu._worst_ratio(h.double() - ref, bound)


@pytest.mark.parametrize('kind', gu.LSTM_KINDS)
def test_bound_holds_for_an_emulation_of_the_kernel(kind):
    r = _emulated_ratio(kind, None)
    print(f'{kind}: emulated err / bound {r:.3f}')
    assert r < 0.5, r


@pytest.mark.parametrize('mutation', ['hl', 'lh', 'stale'])
@pytest.mark.parametrize('kind', ['init', 'trained'])
def test_bound_catches_an_emulation_with_a_lost_product_or_a_stale_h(kind, mutation):
    r = _emulated_ratio(kind, mutation)
    print(f'{kind} {mutation}: emulated err / bound {r:.1f}')
    assert r > 1.0, r


# ------------------------------------------------------------------------------------------------------------------ GPU
def _device_clusters():
    p = L.plan(1, 1, -1)
    assert p is not None, _lib.lib().hn_last_error()
    return p['max_clusters']


def _case(name):
    """(T, B, plan) of a unit case on this device; skips a key no batch reaches here."""
    mc = _device_clusters()
    key = L.CASE_KEYS[name]
    B = L.batch_for(key, mc)
    if B is None:
        pytest.skip(f'no batch of the model takes layout {name} on a device with {mc} co-resident clusters')
    T = L.T_FOR_CLASS[key[5]]
    p = L.plan(T, B, mc)
    assert L.variant_key(T, p) == key, (name, p)
    return T, B, p


def _to_dev(xproj, W):
    return xproj.to(DEV), [w.to(DEV) for w in W]


def _check_bound(name, kind, T, B, p, seed):
    xproj, W = _to_dev(*gu.lstm_inputs(kind, T, B, seed))
    out = gu.lstm_run(xproj, W)
    ratio, where = gu.lstm_ratio(out, xproj, W)
    gu.record('lstm_errors.jsonl', {'test': 'lstm_variant', 'case': name, 'kind': kind, 'T': T, 'B': B, 'plan': p,
                                    'ratio': ratio, 'where': where})
    assert ratio <= 1.0, (ratio, where)


@pytest.mark.gpu
@pytest.mark.parametrize('name', L.CASES)
def test_lstm_variant_vs_fp64(name):
    T, B, p = _case(name)
    _check_bound(name, 'init', T, B, p, seed=T * 1000 + B)


@pytest.mark.gpu
@pytest.mark.parametrize('B', [32, 64])
@pytest.mark.parametrize('kind', ['trained', 'saturated', 'small'])
def test_lstm_model_layouts_with_checkpoint_like_inputs_vs_fp64(kind, B):
    T = L.MODEL_T
    p = L.plan(T, B, _device_clusters())
    _check_bound(L.key_name(L.variant_key(T, p)), kind, T, B, p, seed=B + 10 * gu.LSTM_KINDS.index(kind))


@pytest.mark.gpu
@pytest.mark.parametrize('name', L.CASES)
def test_lstm_columns_match_batch_one(name):
    T, B, _ = _case(name)
    xproj, W = _to_dev(*gu.lstm_inputs('init', T, B, T * 1000 + B))
    out = gu.lstm_run(xproj, W)
    for b in range(B):
        one = gu.lstm_run(xproj[:, b:b + 1].contiguous(), W)
        assert torch.equal(out[:, b:b + 1], one), f'{name}: column {b} of B = {B} differs from the same column alone'


def _mirror(x, half):
    return torch.cat([x[..., half:], x[..., :half]], dim=-1).flip(0).contiguous()


@pytest.mark.gpu
@pytest.mark.parametrize('name', L.CASES)
def test_lstm_direction_mirror(name):
    T, B, _ = _case(name)
    xproj, W = _to_dev(*gu.lstm_inputs('init', T, B, T * 1000 + B + 1))
    out = gu.lstm_run(xproj, W)
    mirrored = gu.lstm_run(_mirror(xproj, 2048), [W[1], W[0]])
    assert torch.equal(mirrored, _mirror(out, 512)), f'{name}: the mirrored launch is not the mirrored output'
