"""-m gpu: the layout post-processing kernel (csrc/layout.cu, hn_layout_postproc) and infer_layout against
oracle/layout_ref.py, which tests/test_layout_oracle.py pins to the real reference.

Discrete results (status, peaks, corner counts, fallbacks) must be identical; cor_id within 1e-5 (normalised units) and
z1 within 1e-5 relative."""
import ctypes
import os

import numpy as np
import pytest
import torch

import __graft_entry__ as entry
from horizonnet_b200 import _lib
from horizonnet_b200.inference import infer_layout, post_process, tta_forward, MAX_ROWS
from horizonnet_b200.model import HorizonNet
from horizonnet_b200.weights import synthetic_state_dict, synthetic_panoramas
from oracle import layout_ref as L

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
G = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'layout.npz'))
NAMES = [str(n) for n in G['names']]
R_PX = int(G['r_px'])
MODES = {'general': (False, False, 0.05), 'cuboid': (True, False, 0.0), 'raw': (False, True, 0.05)}


@pytest.fixture(scope='module', autouse=True)
def _built():
    entry.build()
    _lib.lib()


def _run(yb, yc, force_cuboid, force_raw, min_v, max_rows=MAX_ROWS, r_px=R_PX):
    """hn_layout_postproc on [B][2][1024] / [B][1024] host arrays; returns host numpy outputs."""
    B = yb.shape[0]
    ybd = torch.from_numpy(np.ascontiguousarray(yb, np.float32)).to(DEV)
    ycd = torch.from_numpy(np.ascontiguousarray(yc, np.float32)).to(DEV)
    cor = torch.full((B, max_rows, 2), np.nan, device=DEV)
    n_rows = torch.empty(B, dtype=torch.int32, device=DEV)
    z0 = torch.empty(B, device=DEV)
    z1 = torch.empty(B, device=DEV)
    st = torch.empty(B, dtype=torch.int32, device=DEV)
    pk = torch.empty(B, 1024, dtype=torch.int32, device=DEV)
    npk = torch.empty(B, dtype=torch.int32, device=DEV)
    _lib.check(_lib.lib().hn_layout_postproc(ybd.data_ptr(), ycd.data_ptr(), B, r_px, float(min_v), int(force_cuboid),
                                             int(force_raw), max_rows, cor.data_ptr(), n_rows.data_ptr(), z0.data_ptr(),
                                             z1.data_ptr(), st.data_ptr(), pk.data_ptr(), npk.data_ptr(), None),
               'hn_layout_postproc')
    torch.cuda.synchronize()
    return dict(cor_id=cor.cpu().numpy(), n_rows=n_rows.cpu().numpy(), z0=z0.cpu().numpy(), z1=z1.cpu().numpy(),
                status=st.cpu().numpy(), peaks=pk.cpu().numpy(), n_peaks=npk.cpu().numpy())


def _inputs(names):
    return (np.stack([G[n + '/y_bon'] for n in names]), np.stack([G[n + '/y_cor'] for n in names]))


def _oracle_peaks(yb, yc, z1, force_cuboid, force_raw, min_v, o):
    if force_raw:
        return np.zeros(0, np.int64)
    if o['status'] == L.FALLBACK:
        return L.find_peaks(yc, R_PX, 0, 4)
    return L.find_peaks(yc, R_PX, min_v, 4 if force_cuboid else None)


def _check(name, b, out, yb, yc, force_cuboid, force_raw, min_v, max_rows=MAX_ROWS):
    o = L.post_process(yb, yc, R_PX, min_v=min_v, force_cuboid=force_cuboid, force_raw=force_raw, max_rows=max_rows)
    st = int(out['status'][b])
    assert st == o['status'], (name, L.STATUS_NAMES[st], L.STATUS_NAMES[o['status']], o.get('error'))
    assert abs(float(out['z1'][b]) - float(o['z1'])) <= 1e-5 * abs(float(o['z1'])), name
    assert out['z0'][b] == 50
    if st in (L.OK, L.FALLBACK, L.ERR_GROUPS, L.ERR_VOTE, L.ERR_RING):
        want = _oracle_peaks(yb, yc, o['z1'], force_cuboid, force_raw, min_v, o)
        got = out['peaks'][b][:out['n_peaks'][b]]
        assert np.array_equal(got, want), (name, got, want)
    if o['cor_id'] is None:
        assert out['n_rows'][b] == 0
        return
    n = len(o['cor_id'])
    assert out['n_rows'][b] == n, (name, out['n_rows'][b], n)
    np.testing.assert_allclose(out['cor_id'][b, :n], o['cor_id'], rtol=0, atol=1e-5, err_msg=name)
    assert not out['cor_id'][b, n:].any()


@pytest.mark.parametrize('mode', list(MODES))
def test_golden_inputs_match_the_oracle(mode):
    force_cuboid, force_raw, min_v = MODES[mode]
    yb, yc = _inputs(NAMES)
    out = _run(yb, yc, force_cuboid, force_raw, min_v)
    for b, name in enumerate(NAMES):
        _check(name, b, out, yb[b], yc[b], force_cuboid, force_raw, min_v)
    if mode == 'general':
        assert {L.OK, L.FALLBACK, L.ERR_GROUPS, L.ERR_VOTE, L.ERR_RING} <= set(out['status'].tolist())


def test_cuboid_without_four_peaks_is_a_group_error():
    yb, yc = _inputs(['three_peaks', 'two_peaks'])
    out = _run(yb, yc, True, False, 0.5)
    for b, name in enumerate(['three_peaks', 'two_peaks']):
        _check(name, b, out, yb[b], yc[b], True, False, 0.5)
    assert (out['status'] == L.ERR_GROUPS).all()


@pytest.mark.parametrize('batch', [1, 7, 32])
def test_batches_match_one_at_a_time(batch):
    names = (NAMES * 2)[:batch]
    yb, yc = _inputs(names)
    for mode in ('general', 'cuboid'):
        force_cuboid, force_raw, min_v = MODES[mode]
        full = _run(yb, yc, force_cuboid, force_raw, min_v)
        for b in range(batch):
            one = _run(yb[b:b + 1], yc[b:b + 1], force_cuboid, force_raw, min_v)
            for k in full:
                assert np.array_equal(full[k][b], one[k][0], equal_nan=True), (names[b], mode, k)


def test_plateau_ties_go_to_the_lower_column():
    yb, _ = _inputs(['room0_4c_clean'])
    flat = np.full((1, 1024), 1.0, np.float32)           # saturated sigmoid everywhere
    out = _run(yb, flat, True, False, 0.0)
    assert out['status'][0] == L.OK
    assert out['peaks'][0][:out['n_peaks'][0]].tolist() == [0, 1, 2, 3]
    sig = np.full((1, 1024), 0.01, np.float32)
    sig[0, [50, 300, 700]] = 0.9
    out = _run(yb, sig, True, False, 0.0)
    assert out['peaks'][0][:4].tolist() == [0, 50, 300, 700]
    _check('plateau', 0, out, yb[0], sig[0], True, False, 0.0)


def test_overflow_returns_its_status():
    names = ['room2_6c_clean', 'plateau']
    yb, yc = _inputs(names)
    out = _run(yb, yc, False, False, 0.05, max_rows=8)
    for b, name in enumerate(names):
        _check(name, b, out, yb[b], yc[b], False, False, 0.05, max_rows=8)
    assert (out['status'] == L.ERR_OVERFLOW).all() and (out['n_rows'] == 0).all()
    out = _run(yb[:1], yc[:1], False, True, 0.05, max_rows=2047)
    assert out['status'][0] == L.ERR_OVERFLOW


def test_post_process_raises_like_the_reference():
    yb, yc = _inputs(['no_peaks'])
    with pytest.raises(AssertionError, match='panorama 0'):
        post_process(yb[0], yc[0])
    yb, yc = _inputs(['two_peaks'])
    with pytest.raises(ValueError, match='panorama 0'):
        post_process(yb[0], yc[0])
    res, st = post_process(yb, yc, return_status=True)
    assert st.tolist() == [L.ERR_RING] and res[0][0] is None
    cor_id, z0, z1 = post_process(yb[0], yc[0], force_cuboid=True)
    o = L.post_process(yb[0], yc[0], R_PX, force_cuboid=True)
    np.testing.assert_allclose(cor_id, o['cor_id'], rtol=0, atol=1e-5)


@pytest.mark.parametrize('backbone,use_rnn', [('resnet50', True), ('resnet50', False), ('resnet18', True),
                                              ('resnet18', False)])
def test_infer_layout_matches_the_oracle_on_tta_outputs(backbone, use_rnn):
    net = HorizonNet(backbone, use_rnn).eval()
    net.load_state_dict(synthetic_state_dict(2, 'random', use_rnn=use_rnn, backbone=backbone), strict=True)
    net = net.to(DEV)
    x = synthetic_panoramas(3, seed=102)
    flip, rotate = True, [0.25, 0.333]
    for force_cuboid in (False, True):
        res, status = infer_layout(net, x, flip=flip, rotate=rotate, force_cuboid=force_cuboid, return_status=True)
        assert len(res) == 3
        for b in range(3):
            yb, yc = tta_forward(net, x[b:b + 1], flip=flip, rotate=rotate)
            o = L.post_process(yb, yc, R_PX, force_cuboid=force_cuboid)
            assert int(status[b]) == o['status'], (b, force_cuboid, status[b], o['status'])
            cor_id, z0, z1 = res[b]
            assert abs(float(z1) - float(o['z1'])) <= 1e-5 * abs(float(o['z1']))
            if o['cor_id'] is None:
                assert cor_id is None
                continue
            assert cor_id.shape == o['cor_id'].shape
            np.testing.assert_allclose(cor_id, o['cor_id'], rtol=0, atol=1e-5)
    # the B = 1 path of the batched merge is hn_model_infer_tta itself: the raw export reproduces its boundary
    res = infer_layout(net, x[:1], flip=flip, rotate=rotate, force_raw=True)
    yb, _ = tta_forward(net, x[:1], flip=flip, rotate=rotate)
    assert np.array_equal(res[0][0][0::2, 1] * 512, yb[0].astype(np.float32))


def test_infer_layout_chunks_and_limits():
    net = HorizonNet('resnet18', True).eval()
    net.load_state_dict(synthetic_state_dict(2, 'random', backbone='resnet18'), strict=True)
    net = net.to(DEV)
    x = synthetic_panoramas(2, seed=5)
    with pytest.raises(ValueError):
        infer_layout(net, x, rotate=[0.01] * 64)
    rot = [i / 40 for i in range(1, 32)]                 # 32 views: chunks of 2 panoramas
    a, sa = infer_layout(net, x, rotate=rot, force_cuboid=True, return_status=True)
    b0, s0 = infer_layout(net, x[:1], rotate=rot, force_cuboid=True, return_status=True)
    assert sa[0] == s0[0]
    if a[0][0] is not None:
        np.testing.assert_allclose(a[0][0], b0[0][0], rtol=0, atol=1e-5)
