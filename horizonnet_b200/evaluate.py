"""Device-side evaluation of general room layouts: the reference's eval_general.py and the validation pass of train.py.

``eval_general(dt_cor_ids, gt_cor_ids)`` scores B (dt, gt) pairs in one call of the CUDA kernels of csrc/layout_eval.cu:
the 2D IoU and 3D IoU of the floor polygons and the RMSE and delta_1 of the two depth renders, as eval_general.py's
``test_general`` computes them.  ``validate(net, x, gt_cor_ids)`` is train.py:301-318 for a batch: inference with
``force_raw=True`` and the scoring, on the device, with one copy of the results to the host.  ``summarize`` buckets the
results by the gt's corner count (eval_general.py:106-122) and prints the reference's summary (:162-173).

``python -m horizonnet_b200.evaluate --dt_glob ... --gt_glob ...`` is eval_general.py's command line.
"""
import argparse
import glob
import json
import os

import numpy as np
import torch

from . import _lib
from ._spec import PANO_H, PANO_W

MAX_ROWS = 2 * PANO_W       # corner rows a pair may have (hn_layout_eval_general)
MAX_BATCH = 64              # panoramas per validate() forward

# hn_layout_eval_general status codes (include/horizonnet_b200.h)
OK, DT_INVALID, SKIP_GT_INVALID, ERR_GT_DEPTH, ERR_COLUMNS, ERR_RING = 0, 1, 2, 3, 4, 5
_ERRORS = {
    ERR_GT_DEPTH: (AssertionError, 'layout_2_depth fails on the ground truth'),
    ERR_COLUMNS: (AssertionError, 'odd row count, or ceiling and floor columns differ'),
    ERR_RING: (ValueError, 'fewer than 3 floor corners: not a polygon'),
}
_FALLBACK_STATUS = 2        # a dt of None is scored as train.py's fallback box (any hn_layout_postproc error status)
BUCKETS = ['4', '6', '8', '10+', 'odd', 'overall']


def _check_size(w, h):
    if (w, h) != (PANO_W, PANO_H):
        raise NotImplementedError('test_general hard-codes 1024 x 512 panoramas')


def _pad(cors, dev):
    """Corner lists -> [B][R][2] float32 device tensor and rows [B] int32 (None stays zero rows)."""
    cors = [c if c is None or isinstance(c, torch.Tensor) else np.asarray(c, np.float32) for c in cors]
    rows = [0 if c is None else int(c.shape[0]) for c in cors]
    R = max(rows + [1])
    if R > MAX_ROWS:
        raise ValueError('at most %d corner rows per layout' % MAX_ROWS)
    out = torch.zeros(len(cors), R, 2, device=dev, dtype=torch.float32)
    for b, c in enumerate(cors):
        if c is not None and rows[b]:
            t = torch.as_tensor(c).to(device=dev, dtype=torch.float32)
            if t.dim() != 2 or t.shape[1] != 2:
                raise ValueError('pair %d: a corner list is [n, 2]' % b)
            out[b, :rows[b]] = t
    return out, torch.tensor(rows, device=dev, dtype=torch.int32)


def _device_of(items):
    for c in items:
        if isinstance(c, torch.Tensor) and c.is_cuda:
            return c.device
    return torch.device('cuda', torch.cuda.current_device())


def _results(o, raise_errors, first=0):
    res = {k: v.cpu().numpy() for k, v in o.items()}
    for b, st in enumerate(res['status']):
        st = int(st)
        if st in _ERRORS and raise_errors:
            exc, msg = _ERRORS[st]
            raise exc('pair %d: %s (the reference raises here too)' % (first + b, msg))
        if st == SKIP_GT_INVALID:
            print('Skip ground truth invalid (pair %d)' % (first + b))
    return res


def _outputs(B, dev):
    f64 = dict(device=dev, dtype=torch.float64)
    return dict(iou2d=torch.empty(B, **f64), iou3d=torch.empty(B, **f64), rmse=torch.empty(B, **f64),
                delta_1=torch.empty(B, **f64), status=torch.empty(B, device=dev, dtype=torch.int32))


def _eval(dt_cor_ids, gt_cor_ids, depth=False):
    if len(dt_cor_ids) != len(gt_cor_ids) or not len(gt_cor_ids):
        raise ValueError('eval_general expects as many dt as gt corner lists, at least one')
    dev = _device_of(list(dt_cor_ids) + list(gt_cor_ids))
    B = len(gt_cor_ids)
    dt, dt_rows = _pad(list(dt_cor_ids), dev)
    gt, gt_rows = _pad(list(gt_cor_ids), dev)
    R = max(dt.shape[1], gt.shape[1])
    dt = torch.nn.functional.pad(dt, (0, 0, 0, R - dt.shape[1]))
    gt = torch.nn.functional.pad(gt, (0, 0, 0, R - gt.shape[1]))
    dt_status = torch.tensor([_FALLBACK_STATUS if c is None else 0 for c in dt_cor_ids], device=dev, dtype=torch.int32)
    o = _outputs(B, dev)
    maps = torch.empty(B, 2, PANO_H, PANO_W, device=dev, dtype=torch.float32) if depth else None
    stream = torch.cuda.current_stream(dev).cuda_stream
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().hn_layout_eval_general(
            dt.data_ptr(), dt_rows.data_ptr(), dt_status.data_ptr(), gt.data_ptr(), gt_rows.data_ptr(), B, R,
            o['iou2d'].data_ptr(), o['iou3d'].data_ptr(), o['rmse'].data_ptr(), o['delta_1'].data_ptr(),
            o['status'].data_ptr(), maps.data_ptr() if depth else None, stream), 'hn_layout_eval_general')
    return o, maps


def eval_general(dt_cor_ids, gt_cor_ids, return_status=False):
    """test_general (eval_general.py:57-122) for B pairs on the device.

    dt_cor_ids: B corner lists [2n, 2] normalised by (1024, 512), as infer_layout returns them (numpy, or torch on any
    device), or None for a panorama whose inference failed: that pair scores train.py's fallback box.  gt_cor_ids: B
    corner lists [2m, 2] in pixels, as the label_cor files hold them.  Returns a dict of float64 arrays iou2d, iou3d,
    rmse, delta_1 [B] and int32 status [B] (OK, DT_INVALID: IoUs 0; SKIP_GT_INVALID: all NaN).  Raises like the
    reference where it raises, naming the pair, unless return_status (then those pairs are NaN with their status)."""
    o, _ = _eval(dt_cor_ids, gt_cor_ids)
    return _results(o, raise_errors=not return_status)


def layout_2_depth(cor_id, h=PANO_H, w=PANO_W):
    """eval_general.py:14-54 on the device: the [512, 1024] float32 depth of a layout in pixels ([2n, 2], n >= 3).
    Raises AssertionError where the reference asserts."""
    _check_size(w, h)
    c = torch.as_tensor(cor_id, dtype=torch.float32)
    if c.dim() != 2 or c.shape[1] != 2 or c.shape[0] < 6 or c.shape[0] % 2:
        raise ValueError('layout_2_depth expects [2n, 2] corners with n >= 3')
    norm = c.cpu() / torch.tensor([float(PANO_W), float(PANO_H)])
    o, maps = _eval([norm], [c], depth=True)
    st = int(o['status'][0])
    if st == ERR_COLUMNS:
        raise AssertionError('ceiling and floor columns differ')
    d = maps[0, 0].cpu().numpy()
    if st == ERR_GT_DEPTH or not d.any():
        raise AssertionError('layout_2_depth: the boundary crosses the horizon or a depth is zero')
    return d


def validate(net, x, gt_cor_ids, return_status=False):
    """train.py:301-318 for a batch: x [B, 3, 512, 1024] (any device), gt_cor_ids B corner lists in pixels.

    inference(net, x, force_raw=True) without augmentation and test_general run on the device; a failed inference is
    scored as train.py's fallback box.  Returns the dict of eval_general (per panorama 2DIoU / 3DIoU / rmse / delta_1
    and status)."""
    from .inference import _device
    if x.dim() != 4 or x.shape[1] != 3:
        raise ValueError('validate expects 3-channel panoramas [B, 3, 512, 1024]')
    _check_size(x.shape[3], x.shape[2])
    if len(gt_cor_ids) != x.shape[0]:
        raise ValueError('validate expects one gt corner list per panorama')
    dev = _device(net)
    B = x.shape[0]
    h = net._handle(dev, min(MAX_BATCH, B))
    stream = torch.cuda.current_stream(dev).cuda_stream
    outs = []
    for s in range(0, B, MAX_BATCH):
        xd = x[s:s + MAX_BATCH].detach().to(device=dev, dtype=torch.float32).contiguous()
        n = xd.shape[0]
        gt, gt_rows = _pad(list(gt_cor_ids[s:s + n]), dev)
        o = _outputs(n, dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().hn_model_validate(
                h['ptr'], xd.data_ptr(), n, 3, gt.data_ptr(), gt_rows.data_ptr(), gt.shape[1], o['iou2d'].data_ptr(),
                o['iou3d'].data_ptr(), o['rmse'].data_ptr(), o['delta_1'].data_ptr(), o['status'].data_ptr(), stream),
                'hn_model_validate')
        outs.append(o)
    o = {k: torch.cat([q[k] for q in outs]) for k in outs[0]}
    return _results(o, raise_errors=not return_status)


def bucket(n_rows):
    """eval_general.py:106-113: the bucket of a gt with n_rows corner rows."""
    n = n_rows // 2
    if n % 2 == 1:
        return 'odd'
    return str(n) if n < 10 else '10+'


def summarize(results, gt_cor_ids):
    """eval_general.py:106-122: {bucket: {'2DIoU', '3DIoU', 'rmse', 'delta_1': lists}} over the scored pairs."""
    losses = {k: {'2DIoU': [], '3DIoU': [], 'rmse': [], 'delta_1': []} for k in BUCKETS}
    for b, gt in enumerate(gt_cor_ids):
        if int(results['status'][b]) not in (OK, DT_INVALID):
            continue
        for k in (bucket(len(gt)), 'overall'):
            losses[k]['2DIoU'].append(float(results['iou2d'][b]))
            losses[k]['3DIoU'].append(float(results['iou3d'][b]))
            losses[k]['rmse'].append(float(results['rmse'][b]))
            losses[k]['delta_1'].append(float(results['delta_1'][b]))
    return losses


def print_summary(losses):
    """eval_general.py:162-173."""
    for k, result in losses.items():
        iou2d, iou3d = np.array(result['2DIoU']), np.array(result['3DIoU'])
        rmse, delta_1 = np.array(result['rmse']), np.array(result['delta_1'])
        if len(iou2d) == 0:
            continue
        print('GT #Corners: %s  (%d instances)' % (k, len(iou2d)))
        print('    2DIoU  : %.2f' % (iou2d.mean() * 100))
        print('    3DIoU  : %.2f' % (iou3d.mean() * 100))
        print('    RMSE   : %.2f' % (rmse.mean()))
        print('    delta^1: %.2f' % (delta_1.mean()))


def gtdt_pairs(gt_glob, dt_glob):
    """(gt, dt) path pairs: every gt file, sorted, whose name up to its first dot names a dt .json file."""
    dts = {os.path.split(p)[-1].split('.')[0]: p for p in glob.glob(dt_glob) if p.endswith('json')}
    pairs = []
    for p in sorted(glob.glob(gt_glob)):
        k = os.path.split(p)[-1].split('.')[0]
        if k in dts:
            pairs.append((p, dts[k]))
    return pairs


def main(argv=None):
    p = argparse.ArgumentParser(description='Evaluate general layouts on the GPU (reference eval_general.py CLI)',
                                formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument('--dt_glob', help='quoted glob of the json files inference writes')
    p.add_argument('--gt_glob', help='quoted glob of the label_cor txt files')
    p.add_argument('--w', default=1024, type=int, help='GT images width')
    p.add_argument('--h', default=512, type=int, help='GT images height')
    p.add_argument('--batch', default=256, type=int, help='pairs per device call')
    args = p.parse_args(argv)
    _check_size(args.w, args.h)
    pairs = gtdt_pairs(args.gt_glob, args.dt_glob)
    gts, dts = [], []
    for gt_path, dt_path in pairs:
        with open(gt_path) as f:
            gts.append(np.array([line.split() for line in f], np.float32))
        with open(dt_path) as f:
            dts.append(np.array(json.load(f)['uv'], np.float32))
    losses = {k: {'2DIoU': [], '3DIoU': [], 'rmse': [], 'delta_1': []} for k in BUCKETS}
    for s in range(0, len(pairs), args.batch):
        res = eval_general(dts[s:s + args.batch], gts[s:s + args.batch])
        part = summarize(res, gts[s:s + args.batch])
        for k in BUCKETS:
            for m in losses[k]:
                losses[k][m] += part[k][m]
    print_summary(losses)


if __name__ == '__main__':
    main()
