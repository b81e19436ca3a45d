"""The data path of a training loop (reference dataset.py, PanoCorBonDataset + a DataLoader), with the targets on the device.

``read_corners(path)`` reads a label_cor file as dataset.py:57-67 does.  ``train_targets`` is the label half of
``__getitem__`` (dataset.py:84-120: cor_2_1d, find_occlusion, the flip / roll bookkeeping and the wall-wall probability)
for N samples in one call of the CUDA kernels of csrc/targets.cu.  ``PanoCorBonBatches`` iterates over a dataset
directory (``img/`` + ``label_cor/``) in device batches ``(x, y_bon, y_cor[, cor])``, what
``DataLoader(PanoCorBonDataset(...))`` yields in train.py:164-179: on the host, PIL decodes the images in a thread pool into
a pinned uint8 buffer and one ``np.random.RandomState(seed)`` draws the augmentations (augment.draw_params, in the
reference's order); on the device, one ``augment_batch`` and one ``train_targets`` per batch.  The host side of batch
i + 1 is prepared while the caller runs step i.  No CPU fallback: without the library / a GPU the calls raise.
"""
import os
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import _lib
from ._spec import PANO_H, PANO_W
from .augment import augment_batch, augment_corners, draw_params

MAX_ROWS = 2 * PANO_W       # corner rows a sample may have (hn_train_targets)

# hn_train_targets status codes (include/horizonnet_b200.h)
OK, ERR_ROWS, ERR_CORNERS, ERR_BOUNDARY, ERR_OCCLUDED = 0, 1, 2, 3, 4
_ERRORS = {
    ERR_ROWS: (AssertionError, 'an odd corner row count, or more than %d rows' % MAX_ROWS),
    ERR_CORNERS: (ValueError, 'fewer than 3 ceiling corners: find_occlusion has no polyline to test'),
    ERR_BOUNDARY: (ValueError, 'no wall samples a column of a boundary: cor_2_1d has no point'),
    ERR_OCCLUDED: (ValueError, 'every corner is occluded: y_cor has no corner'),
}


def read_corners(path):
    """dataset.py:57-67: the float32 [2n, 2] corners of a label_cor file, rolled so that the ceiling corner with the
    smallest x comes first.  Raises the reference's two assertions (ceiling and floor columns more than 1 % of the width
    apart; a ceiling corner below its floor corner), naming the file."""
    with open(path) as f:
        cor = np.array([line.strip().split() for line in f if line.strip()], np.float32)
    cor = np.roll(cor[:, :2], -2 * np.argmin(cor[::2, 0]), 0)
    assert (np.abs(cor[0::2, 0] - cor[1::2, 0]) > PANO_W / 100).sum() == 0, path
    assert (cor[0::2, 1] > cor[1::2, 1]).sum() == 0, path
    return cor


def _pad(cors, n_rows, dev, pin=False):
    R = max(n_rows + [1])
    host = torch.zeros(len(cors), R, 2, dtype=torch.float32, pin_memory=pin)
    for b, c in enumerate(cors):
        host[b, :n_rows[b]] = torch.as_tensor(np.asarray(c, np.float32))
    return host.to(dev, non_blocking=pin)


def _launch_targets(cor0s, cors, flip, dx, p_base, dev, pin=False):
    """Enqueue hn_train_targets on the current stream of `dev`; returns the device outputs (status included)."""
    n = len(cor0s)
    if not n or len(cors) != n or len(flip) != n or len(dx) != n:
        raise ValueError('train_targets expects N >= 1 samples with N cor0s, cors, flip and dx entries')
    rows = [int(np.asarray(c).shape[0]) for c in cor0s]
    if any(int(np.asarray(c).shape[0]) != r for c, r in zip(cors, rows)):
        raise ValueError('train_targets: cor0s[i] and cors[i] must have the same row count')
    if max(rows) > MAX_ROWS:
        raise ValueError('train_targets: at most %d corner rows per sample' % MAX_ROWS)
    if any(d is not None and not -1 <= int(d) < PANO_W for d in dx):
        raise ValueError('train_targets: dx must be in 0..%d, or -1 / None for no roll' % (PANO_W - 1))
    if not 0 < p_base < 1:
        raise ValueError('train_targets: p_base must be in (0, 1)')
    c0 = _pad(cor0s, rows, dev, pin)
    c1 = _pad(cors, rows, dev, pin)
    ints = torch.tensor([rows, [1 if f else 0 for f in flip], [-1 if d is None else int(d) for d in dx]],
                        dtype=torch.int32, pin_memory=pin).to(dev, non_blocking=pin)
    R = c0.shape[1]
    out = dict(y_bon=torch.empty(n, 2, PANO_W, device=dev), y_cor=torch.empty(n, 1, PANO_W, device=dev),
               cor=torch.empty(n, R, 2, device=dev), occlusion=torch.empty(n, R, device=dev, dtype=torch.int32),
               status=torch.empty(n, device=dev, dtype=torch.int32), rows=rows)
    stream = torch.cuda.current_stream(dev).cuda_stream
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().hn_train_targets(
            c0.data_ptr(), c1.data_ptr(), ints[0].data_ptr(), ints[1].data_ptr(), ints[2].data_ptr(), n, R, float(p_base),
            out['y_bon'].data_ptr(), out['y_cor'].data_ptr(), out['cor'].data_ptr(), out['occlusion'].data_ptr(),
            out['status'].data_ptr(), stream), 'hn_train_targets')
    out['_keep'] = (c0, c1, ints)              # the inputs stay alive until the kernels have read them
    return out


def _raise_status(status, names):
    for b, st in enumerate(np.asarray(status).tolist()):
        if st != OK:
            exc, msg = _ERRORS.get(st, (RuntimeError, 'status %d' % st))
            raise exc('%s: %s (the reference raises here too)' % (names[b], msg))


def train_targets(cor0s, cors, flip, dx, p_base=0.96, device=None, return_all=False):
    """The targets of dataset.py:84-120 for N samples on the device.

    cor0s: N corner lists [2n, 2] in pixels as read_corners returns them; cors: the same corners after the stretch
    (augment.augment_corners(cor0, 512, 1024, kx, ky), or cor0 without one); flip: N bools; dx: N np.roll shifts (None or
    -1: no roll).  Returns y_bon [N, 2, 1024] and y_cor [N, 1, 1024] float32 CUDA tensors; with return_all, also the
    flipped and rolled corners [N, R, 2] and the occlusion flags [N, R] (R = the largest row count).  Raises, naming the
    sample, where the reference raises."""
    dev = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
    out = _launch_targets(list(cor0s), list(cors), list(flip), list(dx), p_base, dev)
    _raise_status(out['status'].cpu(), ['sample %d' % b for b in range(len(out['rows']))])
    if return_all:
        return out['y_bon'], out['y_cor'], out['cor'], out['occlusion'].bool()
    return out['y_bon'], out['y_cor']


class PanoCorBonBatches:
    """Device batches of a dataset directory, as DataLoader(PanoCorBonDataset(root_dir, flip, rotate, gamma, stretch,
    p_base, max_stretch, return_cor), batch_size, shuffle, drop_last) yields them (reference dataset.py:13-134).

    Each iteration yields ``(x, y_bon, y_cor)`` -- CUDA float32 [B, 3, 512, 1024], [B, 2, 1024], [B, 1, 1024] -- and,
    with return_cor, the list of the B flipped and rolled corner lists as CUDA float32 [2n, 2] tensors.  The random
    draws come from one ``np.random.RandomState(seed)`` in sample order (the shuffle permutation first), so the same seed
    gives the same stream.  Only 512 x 1024 images are accepted.  A sample the reference cannot label raises, naming its
    file, at most one batch after it is yielded (its status is read without stalling the device)."""

    def __init__(self, root_dir, batch_size, flip=False, rotate=False, gamma=False, stretch=False, p_base=0.96,
                 max_stretch=2.0, shuffle=False, drop_last=False, seed=0, device='cuda', num_threads=8, return_cor=False):
        self.img_dir = os.path.join(root_dir, 'img')
        self.cor_dir = os.path.join(root_dir, 'label_cor')
        self.img_fnames = sorted(f for f in os.listdir(self.img_dir) if f.endswith('.jpg') or f.endswith('.png'))
        self.txt_fnames = ['%s.txt' % f[:-4] for f in self.img_fnames]
        for f in self.txt_fnames:                                        # dataset.py:40-44
            assert os.path.isfile(os.path.join(self.cor_dir, f)), '%s not found' % os.path.join(self.cor_dir, f)
        if batch_size < 1:
            raise ValueError('batch_size must be >= 1')
        self.batch_size = batch_size
        self.aug = dict(flip=flip, rotate=rotate, gamma=gamma, stretch=stretch)
        self.p_base, self.max_stretch = p_base, max_stretch
        self.shuffle, self.drop_last, self.return_cor = shuffle, drop_last, return_cor
        self.rng = np.random.RandomState(seed)
        self.device = torch.device(device)
        if self.device.type == 'cuda' and self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())
        self.pool = ThreadPoolExecutor(max(1, num_threads))
        self.prep = ThreadPoolExecutor(1)                                # the host side of the next batch
        self._corners = {}
        self._lock = threading.Lock()
        self._bufs = [torch.empty(batch_size, PANO_H, PANO_W, 3, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
        self._uploaded = [None, None]                                    # event: the buffer's copy to the device is done

    def __len__(self):
        n = len(self.img_fnames)
        return n // self.batch_size if self.drop_last else -(-n // self.batch_size)

    def _cor0(self, i):
        with self._lock:
            c = self._corners.get(i)
        if c is None:
            c = read_corners(os.path.join(self.cor_dir, self.txt_fnames[i]))
            with self._lock:
                self._corners[i] = c
        return c

    def _decode(self, buf, slot, i):
        from PIL import Image
        path = os.path.join(self.img_dir, self.img_fnames[i])
        with Image.open(path) as img:
            a = np.asarray(img)
        if a.ndim != 3 or a.shape[2] < 3 or a.shape[:2] != (PANO_H, PANO_W):
            raise ValueError('%s: only %d x %d RGB(A) panoramas are supported (the model refuses other sizes), got %s'
                             % (path, PANO_W, PANO_H, 'x'.join(map(str, a.shape))))
        buf[slot].numpy()[...] = a[..., :3]

    def _host(self, k, idx):
        """Decode + draws of one batch into pinned buffer k."""
        if self._uploaded[k] is not None:
            self._uploaded[k].synchronize()
        buf = self._bufs[k]
        decodes = [self.pool.submit(self._decode, buf, s, i) for s, i in enumerate(idx)]
        draws = []
        for i in idx:                                                    # dataset.py:69-105, in sample order
            c0 = self._cor0(i)
            p = draw_params(c0, PANO_W, max_stretch=self.max_stretch, rng=self.rng, **self.aug)
            cs = augment_corners(c0, PANO_H, PANO_W, p['kx'], p['ky']) if p['kx'] is not None else c0
            draws.append((c0, cs, p))
        for d in decodes:
            d.result()
        return k, idx, draws

    def _device(self, host):
        k, idx, draws = host
        n = len(idx)
        dev = self.device
        imgs = self._bufs[k][:n].to(dev, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(dev))
        self._uploaded[k] = ev
        ps = [d[2] for d in draws]
        x = augment_batch(imgs, [p['kx'] for p in ps], [p['ky'] for p in ps], [p['flip'] for p in ps],
                          [p['dx'] for p in ps], [p['p'] for p in ps])
        t = _launch_targets([d[0] for d in draws], [d[1] for d in draws], [p['flip'] for p in ps],
                            [p['dx'] if self.aug['rotate'] else -1 for p in ps], self.p_base, dev, pin=True)
        status = torch.empty(n, dtype=torch.int32, pin_memory=True)
        status.copy_(t['status'], non_blocking=True)
        done = torch.cuda.Event()
        done.record(torch.cuda.current_stream(dev))
        names = [self.txt_fnames[i] for i in idx]
        batch = (x, t['y_bon'], t['y_cor'])
        if self.return_cor:
            batch += ([t['cor'][b, :t['rows'][b]] for b in range(n)],)
        return batch, (status, done, names, t)

    @staticmethod
    def _check(pending):
        status, done, names, _ = pending
        done.synchronize()
        _raise_status(status.numpy(), names)

    def __iter__(self):
        n = len(self.img_fnames)
        order = self.rng.permutation(n) if self.shuffle else np.arange(n)
        bs = self.batch_size
        groups = [order[s:s + bs].tolist() for s in range(0, n, bs)]
        if self.drop_last and groups and len(groups[-1]) < bs:
            groups.pop()
        pending = None
        fut = self.prep.submit(self._host, 0, groups[0]) if groups else None
        for g in range(len(groups)):
            host = fut.result()
            batch, nxt = self._device(host)
            if g + 1 < len(groups):
                fut = self.prep.submit(self._host, (g + 1) % 2, groups[g + 1])
            if pending is not None:
                self._check(pending)
            pending = nxt
            yield batch
        if pending is not None:
            self._check(pending)
