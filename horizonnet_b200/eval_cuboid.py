"""Device-side evaluation of cuboid room layouts: the reference's eval_cuboid.py.

``eval_cuboid(dt_cor_ids, z0s, z1s, gt_cor_ids)`` scores B (dt, gt) pairs in one call of the CUDA kernels of
csrc/layout_cuboid.cu: the corner error, the pixel error of the ceiling / wall / floor labels and the 3D IoU, as
eval_cuboid.py's ``test`` computes them.  ``evaluate_cuboid(net, x, gt_cor_ids)`` is the README's protocol for a batch:
inference with ``force_cuboid=True`` (test-time augmentation optional) and the scoring, on the device, with one copy of
the results to the host.

``python -m horizonnet_b200.eval_cuboid --dt_glob ... --gt_glob ...`` is eval_cuboid.py's command line.
"""
import argparse
import ctypes
import json

import numpy as np
import torch

from . import _lib
from .evaluate import _check_size, _device_of, _pad, gtdt_pairs

MAX_VIEWS = 64              # views x panoramas per evaluate_cuboid() forward

# hn_layout_eval_cuboid status codes (include/horizonnet_b200.h)
OK, ERR_ROWS, ERR_INDEX, ERR_COLUMNS, ERR_HULL, DT_FAILED = 0, 1, 2, 3, 4, 5
_ERRORS = {
    ERR_ROWS: (ValueError, 'dt and gt must both be 8 corner rows (a cuboid)'),
    ERR_INDEX: (IndexError, 'a boundary row is past the image or NaN'),
    ERR_COLUMNS: (AssertionError, 'ceiling and floor columns differ'),
    ERR_HULL: (ValueError, 'the halfspace intersection is unbounded or flat (qhull refuses it)'),
    DT_FAILED: (RuntimeError, 'the layout inference failed: there is no cuboid to score'),
}


def _outputs(B, dev):
    f64 = dict(device=dev, dtype=torch.float64)
    return dict(ce=torch.empty(B, **f64), pe=torch.empty(B, **f64), iou3d=torch.empty(B, **f64),
                status=torch.empty(B, device=dev, dtype=torch.int32))


def _results(o, raise_errors, first=0):
    res = {k: v.cpu().numpy() for k, v in o.items()}
    if raise_errors:
        for b, st in enumerate(res['status']):
            if int(st) in _ERRORS:
                exc, msg = _ERRORS[int(st)]
                raise exc('pair %d: %s (the reference fails here too)' % (first + b, msg))
    return res


def eval_cuboid(dt_cor_ids, z0s, z1s, gt_cor_ids, return_status=False):
    """test (eval_cuboid.py:100-145) for B pairs on the device.

    dt_cor_ids: B corner lists [8, 2] normalised by (1024, 512), as infer_layout(force_cuboid=True) returns them and the
    inference json holds them (numpy, or torch on any device), or None for a panorama whose inference failed.  z0s,
    z1s: B floats (the json's z0 and z1).  gt_cor_ids: B corner lists [8, 2] in pixels, as the label_cor files hold
    them.  Returns a dict of float64 arrays ce, pe, iou3d [B] (percent) and int32 status [B].  Raises like the
    reference where it raises, naming the pair, unless return_status (then those pairs are NaN with their status)."""
    B = len(gt_cor_ids)
    if len(dt_cor_ids) != B or len(z0s) != B or len(z1s) != B or not B:
        raise ValueError('eval_cuboid expects as many dt, z0, z1 as gt corner lists, at least one')
    dev = _device_of(list(dt_cor_ids) + list(gt_cor_ids))
    dt, dt_rows = _pad(list(dt_cor_ids), dev)
    gt, gt_rows = _pad(list(gt_cor_ids), dev)
    R = max(dt.shape[1], gt.shape[1], 8)
    dt = torch.nn.functional.pad(dt, (0, 0, 0, R - dt.shape[1]))
    gt = torch.nn.functional.pad(gt, (0, 0, 0, R - gt.shape[1]))
    dt_status = torch.tensor([DT_FAILED if c is None else 0 for c in dt_cor_ids], device=dev, dtype=torch.int32)
    z0 = torch.tensor([float(z) for z in z0s], device=dev, dtype=torch.float64)
    z1 = torch.tensor([float(z) for z in z1s], device=dev, dtype=torch.float64)
    o = _outputs(B, dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().hn_layout_eval_cuboid(
            dt.data_ptr(), dt_rows.data_ptr(), dt_status.data_ptr(), z0.data_ptr(), z1.data_ptr(), gt.data_ptr(),
            gt_rows.data_ptr(), B, R, o['ce'].data_ptr(), o['pe'].data_ptr(), o['iou3d'].data_ptr(),
            o['status'].data_ptr(), stream), 'hn_layout_eval_cuboid')
    return _results(o, raise_errors=not return_status)


def evaluate_cuboid(net, x, gt_cor_ids, flip=False, rotate=(), r=0.05, return_status=False):
    """The README's cuboid protocol for a batch: inference.py --force_cuboid, then eval_cuboid.py, on the device.

    x [B, 3, 512, 1024] (any device), gt_cor_ids B corner lists [8, 2] in pixels; flip / rotate are inference.py's
    test-time augmentations.  Returns the dict of eval_cuboid for the results of
    infer_layout(net, x, flip, rotate, force_cuboid=True), bit for bit, without copying them to the host."""
    from .inference import _device, _postproc_args, _shifts
    if x.dim() != 4 or x.shape[1] != 3:
        raise ValueError('evaluate_cuboid expects 3-channel panoramas [B, 3, 512, 1024]')
    _check_size(x.shape[3], x.shape[2])
    if len(gt_cor_ids) != x.shape[0]:
        raise ValueError('evaluate_cuboid expects one gt corner list per panorama')
    dev = _device(net)
    shifts = _shifts(rotate)
    views = 1 + (1 if flip else 0) + len(shifts)
    if views > MAX_VIEWS:
        raise ValueError('at most %d views per panorama' % MAX_VIEWS)
    r_px, mv = _postproc_args(True, None, r)
    B = x.shape[0]
    chunk = max(1, MAX_VIEWS // views)
    h = net._handle(dev, min(chunk, B) * views)
    arr = (ctypes.c_int * max(len(shifts), 1))(*shifts) if shifts else None
    stream = torch.cuda.current_stream(dev).cuda_stream
    outs = []
    for s in range(0, B, chunk):
        xd = x[s:s + chunk].detach().to(device=dev, dtype=torch.float32).contiguous()
        n = xd.shape[0]
        gt, gt_rows = _pad(list(gt_cor_ids[s:s + n]), dev)
        if gt.shape[1] < 8:
            gt = torch.nn.functional.pad(gt, (0, 0, 0, 8 - gt.shape[1]))
        o = _outputs(n, dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().hn_model_eval_cuboid(
                h['ptr'], xd.data_ptr(), n, 3, 1 if flip else 0, arr, len(shifts), r_px, mv, gt.data_ptr(),
                gt_rows.data_ptr(), gt.shape[1], o['ce'].data_ptr(), o['pe'].data_ptr(), o['iou3d'].data_ptr(),
                o['status'].data_ptr(), stream), 'hn_model_eval_cuboid')
        outs.append(o)
    o = {k: torch.cat([q[k] for q in outs]) for k in outs[0]}
    return _results(o, raise_errors=not return_status)


def print_summary(losses):
    """eval_cuboid.py:198-202."""
    print(' Testing Result '.center(50, '='))
    print('Corner Error (%):', np.mean(losses['CE']))
    print('Pixel  Error (%):', np.mean(losses['PE']))
    print('3DIoU        (%):', np.mean(losses['3DIoU']))
    print('=' * 50)


def main(argv=None):
    p = argparse.ArgumentParser(description='Evaluate cuboid layouts on the GPU (reference eval_cuboid.py CLI)',
                                formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument('--dt_glob', required=True, help='quoted glob of the json files inference writes')
    p.add_argument('--gt_glob', default='data/test/label_cor/*txt', help='quoted glob of the label_cor txt files')
    p.add_argument('--w', default=1024, type=int, help='GT images width')
    p.add_argument('--h', default=512, type=int, help='GT images height')
    p.add_argument('--batch', default=256, type=int, help='pairs per device call')
    args = p.parse_args(argv)
    _check_size(args.w, args.h)
    pairs = gtdt_pairs(args.gt_glob, args.dt_glob)
    gts, dts, z0s, z1s = [], [], [], []
    for gt_path, dt_path in pairs:
        with open(gt_path) as f:
            gts.append(np.array([line.split() for line in f], np.float32))
        with open(dt_path) as f:
            dt = json.load(f)
        dts.append(np.array(dt['uv'], np.float32))
        z0s.append(dt['z0'])
        z1s.append(dt['z1'])
    losses = {'CE': [], 'PE': [], '3DIoU': []}
    for s in range(0, len(pairs), args.batch):
        e = s + args.batch
        res = eval_cuboid(dts[s:e], z0s[s:e], z1s[s:e], gts[s:e])
        losses['CE'] += [float(v) for v in res['ce']]
        losses['PE'] += [float(v) for v in res['pe']]
        losses['3DIoU'] += [float(v) for v in res['iou3d']]
    print_summary(losses)


if __name__ == '__main__':
    main()
