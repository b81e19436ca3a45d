"""Device-side inference of the reference's inference.py: test-time augmentation and room-layout post-processing.

``tta_forward(net, x, flip, rotate)`` replaces the first half of the reference's ``inference()`` (inference.py:32-62,
77-93): ``augment`` (numpy flip / roll on the host), ``net(x.to(device))``, two ``.cpu()`` round trips, ``sigmoid``,
``augment_undo(...).mean(0)`` and the boundary -> pixel-row conversion with clipping.  Here one panorama is uploaded
once; the views, the forward and the merge all run on the device.

``infer_layout(net, x, ...)`` is the whole ``inference()`` for a batch of panoramas: the views of all of them in one
forward, the merge per panorama, then the layout post-processing of inference.py:95-141 (ceiling height, wall-wall
peaks, Manhattan wall fitting, the polygon-validity fallback, corner packing) in one CUDA kernel with one CTA per
panorama (csrc/layout.cu).  ``post_process(y_bon_pix, y_cor, ...)`` runs that kernel on signals the caller already has.

``python -m horizonnet_b200.inference --pth ... --img_glob ... --output_dir ...`` writes the reference's JSON per image.
"""
import argparse
import ctypes
import glob
import json
import os
import sys

import numpy as np
import torch

from . import _lib
from ._spec import PANO_H, PANO_W

MAX_VIEWS = 64              # views of one panorama per forward (hn_model_infer_tta / hn_model_infer_layout)
MAX_ROWS = 2 * PANO_W       # cor_id rows every result fits in (force_raw: 1024 ceiling / floor pairs)

# hn_layout_postproc status codes (include/horizonnet_b200.h)
OK, FALLBACK, ERR_GROUPS, ERR_VOTE, ERR_RING, ERR_OVERFLOW = 0, 1, 2, 3, 4, 5
_ERRORS = {
    ERR_GROUPS: (AssertionError, 'gen_ww: the peaks do not give the wall groups the fit needs '
                                 '(a cuboid needs 4 peaks, a general layout at least 1)'),
    ERR_VOTE: (AssertionError, 'vote: the best run of a wall group is a single value'),
    ERR_RING: (ValueError, 'the general layout has fewer than 3 walls: not a polygon'),
    ERR_OVERFLOW: (RuntimeError, 'the corners do not fit in the output rows'),
}


def _device(net):
    dev = next(net.parameters()).device
    if dev.type != 'cuda':
        raise RuntimeError('horizonnet_b200 has no CPU path: move the model to a cuda device')
    return dev


def _shifts(rotate):
    return [int(round(p * PANO_W)) for p in rotate]                 # inference.py:40


def tta_forward(net, x, flip=False, rotate=()):
    """x: [1, 3, 512, 1024] float tensor (any device).  Returns (y_bon_ [2,1024] pixel rows, y_cor_ [1024]) as
    float32 numpy arrays -- the values the reference holds after inference.py:93 (before post-processing)."""
    if x.dim() != 4 or x.shape[0] != 1 or x.shape[1] != 3:
        raise ValueError('tta_forward expects one 3-channel panorama [1, 3, 512, 1024] (inference.py:196-200)')
    if x.shape[2] != PANO_H or x.shape[3] != PANO_W:
        raise NotImplementedError()
    dev = _device(net)
    shifts = _shifts(rotate)
    views = 1 + (1 if flip else 0) + len(shifts)
    h = net._handle(dev, max(views, 1))
    xd = x.detach().to(device=dev, dtype=torch.float32).contiguous()
    y_bon = torch.empty(2, PANO_W, device=dev, dtype=torch.float32)
    y_cor = torch.empty(PANO_W, device=dev, dtype=torch.float32)
    arr = (ctypes.c_int * max(len(shifts), 1))(*shifts) if shifts else None
    stream = torch.cuda.current_stream(dev).cuda_stream
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().hn_model_infer_tta(h['ptr'], xd.data_ptr(), 3, 1 if flip else 0, arr, len(shifts),
                                                 y_bon.data_ptr(), y_cor.data_ptr(), stream), 'hn_model_infer_tta')
    return y_bon.cpu().numpy(), y_cor.cpu().numpy()


def _postproc_args(force_cuboid, min_v, r):
    if min_v is None:
        min_v = 0 if force_cuboid else 0.05                          # inference.py:106-107
    return int(round(PANO_W * r / 2)), float(min_v)                  # inference.py:108


class _Outputs:
    def __init__(self, B, dev):
        self.cor_id = torch.empty(B, MAX_ROWS, 2, device=dev, dtype=torch.float32)
        self.n_rows = torch.empty(B, device=dev, dtype=torch.int32)
        self.z0 = torch.empty(B, device=dev, dtype=torch.float32)
        self.z1 = torch.empty(B, device=dev, dtype=torch.float32)
        self.status = torch.empty(B, device=dev, dtype=torch.int32)

    def ptrs(self):
        return [self.cor_id.data_ptr(), self.n_rows.data_ptr(), self.z0.data_ptr(), self.z1.data_ptr(),
                self.status.data_ptr()]

    def results(self, first=0, raise_errors=True):
        cor_id, n_rows = self.cor_id.cpu().numpy(), self.n_rows.cpu().numpy()
        z0, z1, status = self.z0.cpu().numpy(), self.z1.cpu().numpy(), self.status.cpu().numpy()
        out = []
        for b in range(len(status)):
            st = int(status[b])
            if st in _ERRORS:
                if raise_errors:
                    exc, msg = _ERRORS[st]
                    raise exc('panorama %d: %s (the reference raises here too)' % (first + b, msg))
                out.append((None, float(z0[b]), z1[b]))
                continue
            if st == FALLBACK:
                print('panorama %d: Fail to generate valid general layout!! Generate cuboid as fallback.' % (first + b),
                      file=sys.stderr)
            out.append((cor_id[b, :n_rows[b]].copy(), int(z0[b]), z1[b]))
        return out, status


def post_process(y_bon_pix, y_cor, force_cuboid=False, force_raw=False, min_v=None, r=0.05, return_status=False):
    """Layout post-processing of inference.py:95-141 on the device for signals the caller has (e.g. from tta_forward).

    y_bon_pix: [2, 1024] or [B, 2, 1024] pixel-row boundaries, y_cor: [1024] or [B, 1024], float32 (numpy or torch; a
    cuda tensor stays on its device).  Returns one (cor_id [2n, 2] float32, z0, z1 float32) per panorama, the values
    reference inference() returns, and raises like the reference where it raises, naming the panorama.  With
    return_status, also returns the per-panorama status codes (OK / FALLBACK / ERR_*) and does not raise."""
    yb = torch.as_tensor(y_bon_pix, dtype=torch.float32)
    yc = torch.as_tensor(y_cor, dtype=torch.float32)
    single = yb.dim() == 2
    if single:
        yb, yc = yb[None], yc[None]
    if yb.shape[1:] != (2, PANO_W) or yc.shape[1:] != (PANO_W,) or yb.shape[0] != yc.shape[0]:
        raise ValueError('post_process expects y_bon_pix [B, 2, 1024] and y_cor [B, 1024]')
    dev = yb.device if yb.is_cuda else torch.device('cuda', torch.cuda.current_device())
    yb = yb.to(dev).contiguous()
    yc = yc.to(dev).contiguous()
    B = yb.shape[0]
    r_px, mv = _postproc_args(force_cuboid, min_v, r)
    o = _Outputs(B, dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().hn_layout_postproc(yb.data_ptr(), yc.data_ptr(), B, r_px, mv, int(force_cuboid),
                                                 int(force_raw), MAX_ROWS, *o.ptrs(), None, None, stream),
                   'hn_layout_postproc')
    res, status = o.results(raise_errors=not return_status)
    if single and not return_status:
        return res[0]
    return (res, status) if return_status else res


def infer_layout(net, x, flip=False, rotate=(), force_cuboid=False, force_raw=False, min_v=None, r=0.05,
                 return_status=False):
    """Reference inference() (inference.py:65-141) for a batch: x [B, 3, 512, 1024] float in [0, 1] (any device).

    Returns one (cor_id [2n, 2] float32, z0, z1 float32) per panorama.  Panoramas run in chunks of 64 // views, each chunk
    as one forward of all its views.  Raises like the reference where it raises, naming the panorama; with return_status
    returns (results, status codes) instead and leaves None in place of the failed panoramas' cor_id."""
    if x.dim() != 4 or x.shape[1] != 3:
        raise ValueError('infer_layout expects 3-channel panoramas [B, 3, 512, 1024] (inference.py:196-200)')
    if x.shape[2] != PANO_H or x.shape[3] != PANO_W:
        raise NotImplementedError()
    dev = _device(net)
    shifts = _shifts(rotate)
    views = 1 + (1 if flip else 0) + len(shifts)
    if views > MAX_VIEWS:
        raise ValueError('at most %d views per panorama' % MAX_VIEWS)
    r_px, mv = _postproc_args(force_cuboid, min_v, r)
    B = x.shape[0]
    chunk = max(1, MAX_VIEWS // views)
    h = net._handle(dev, min(chunk, B) * views)
    arr = (ctypes.c_int * max(len(shifts), 1))(*shifts) if shifts else None
    stream = torch.cuda.current_stream(dev).cuda_stream
    results, statuses = [], []
    for s in range(0, B, chunk):
        xd = x[s:s + chunk].detach().to(device=dev, dtype=torch.float32).contiguous()
        n = xd.shape[0]
        y_bon = torch.empty(n, 2, PANO_W, device=dev, dtype=torch.float32)
        y_cor = torch.empty(n, PANO_W, device=dev, dtype=torch.float32)
        o = _Outputs(n, dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().hn_model_infer_layout(
                h['ptr'], xd.data_ptr(), n, 3, 1 if flip else 0, arr, len(shifts), r_px, mv, int(force_cuboid),
                int(force_raw), MAX_ROWS, y_bon.data_ptr(), y_cor.data_ptr(), *o.ptrs(), stream), 'hn_model_infer_layout')
        res, st = o.results(first=s, raise_errors=not return_status)
        results += res
        statuses.append(st)
    return (results, np.concatenate(statuses)) if return_status else results


def load_checkpoint(path, device):
    """A checkpoint of reference misc/utils.py save_model ({'kwargs': {backbone, use_rnn}, 'state_dict': ...}) as our
    HorizonNet on `device`, in eval mode (what utils.load_trained_model + .eval() give the reference CLI)."""
    from .model import HorizonNet
    ck = torch.load(path, map_location='cpu', weights_only=False)
    net = HorizonNet(**ck['kwargs'])
    net.load_state_dict(ck['state_dict'], strict=True)
    return net.to(device).eval()


def load_image(path):
    """inference.py:196-200: RGB(A) image -> [1, 3, 512, 1024] float in [0, 1], bicubic resize when needed."""
    from PIL import Image
    img = Image.open(path)
    if img.size != (PANO_W, PANO_H):
        img = img.resize((PANO_W, PANO_H), Image.BICUBIC)
    arr = np.array(img)[..., :3].transpose([2, 0, 1]).copy()
    return torch.FloatTensor(np.array([arr / 255]))


def main(argv=None):
    p = argparse.ArgumentParser(description='Room layouts of panoramas on the GPU (reference inference.py CLI; '
                                            '--visualize is not supported)',
                                formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument('--pth', required=True, help='checkpoint saved by the reference misc/utils.py save_model')
    p.add_argument('--img_glob', required=True, help='quoted glob of aligned panoramas')
    p.add_argument('--output_dir', required=True)
    p.add_argument('--flip', action='store_true', help='add the left-right flipped view')
    p.add_argument('--rotate', nargs='*', default=[], type=float, help='horizontal rotations, fractions of the width')
    p.add_argument('--r', default=0.05, type=float)
    p.add_argument('--min_v', default=None, type=float)
    p.add_argument('--force_cuboid', action='store_true')
    p.add_argument('--force_raw', action='store_true')
    p.add_argument('--batch', default=8, type=int, help='panoramas per call')
    args = p.parse_args(argv)

    paths = sorted(glob.glob(args.img_glob))
    if not paths:
        print('no images found')
    os.makedirs(args.output_dir, exist_ok=True)
    net = load_checkpoint(args.pth, torch.device('cuda'))
    with torch.no_grad():
        for s in range(0, len(paths), args.batch):
            group = paths[s:s + args.batch]
            x = torch.cat([load_image(q) for q in group], 0)
            res = infer_layout(net, x, flip=args.flip, rotate=args.rotate, force_cuboid=args.force_cuboid,
                               force_raw=args.force_raw, min_v=args.min_v, r=args.r)
            for q, (cor_id, z0, z1) in zip(group, res):
                k = os.path.split(q)[-1][:-4]
                with open(os.path.join(args.output_dir, k + '.json'), 'w') as f:
                    json.dump({'z0': float(z0), 'z1': float(z1), 'uv': [[float(u), float(v)] for u, v in cor_id]}, f)


if __name__ == '__main__':
    main()
