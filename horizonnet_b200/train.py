"""Train HorizonNet from a dataset directory on the GPU: the reference's train.py loop on this library.

``python -m horizonnet_b200.train --id NAME --train_root_dir DIR [--valid_root_dir DIR] ...`` takes train.py's flags with
their names and defaults.  Each iteration sets the warm-up + poly learning rate (misc/utils.py:35-46), runs the
library's train-mode forward and backward on ``l1_loss + binary_cross_entropy_with_logits`` and steps Adam or SGD
(train.py:216-225).  Batches come from ``dataset.PanoCorBonBatches``: the images are augmented and the targets computed
on the device.  The validation pass (train.py:283-325) scores the valid set with ``evaluate.validate`` and keeps the
model with the best 3D IoU.  Checkpoints are train.py's: ``checkpoint.pth.tar`` every epoch with a valid set (copied to
``best_model_{ep}.pth.tar`` when it is the best so far) and ``epoch_N.pth`` in save_model's format every --save_every
epochs.  tensorboardX is not a dependency: the scalars train.py logs go, with the same tags, to
``<logs>/<id>/scalars.jsonl`` as one JSON object per line.

The step is fp32 (no autocast or GradScaler: the library's training step has one precision).  Training losses stay on
the device between --disp_iter reads.  The draws are reproducible under --seed; train.py reseeds every worker from OS
entropy.  Not supported: --no_cuda, --multi_gpu, backbones the library does not build.
"""
import argparse
import json
import os
import shutil
import sys
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .dataset import PanoCorBonBatches
from .evaluate import DT_INVALID, OK, validate


def learning_rate(cur_iter, lr, warmup_lr, lr_pow, warmup_iters, max_iters):
    """misc/utils.py:35-46 adjust_learning_rate: the learning rate of iteration cur_iter (counted from 0)."""
    if cur_iter < warmup_iters:
        frac = cur_iter / warmup_iters
        return warmup_lr + (lr - warmup_lr) * frac
    frac = (float(cur_iter) - warmup_iters) / (max_iters - warmup_iters)
    return lr * max((1. - frac), 0.) ** lr_pow


def parse_args(argv=None):
    p = argparse.ArgumentParser(description='Train HorizonNet on the GPU (reference train.py CLI)',
                                formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument('--id', required=True, help='experiment id to name checkpoints and logs')
    p.add_argument('--ckpt', default='./ckpt', help='folder to output checkpoints')
    p.add_argument('--logs', default='./logs', help='folder to logging')
    p.add_argument('--pth', default=None, help='path to load saved checkpoint.(finetuning)')
    p.add_argument('--backbone', default='resnet50', help='backbone of the network (resnet50 or resnet18)')
    p.add_argument('--no_rnn', action='store_true', help='whether to remove rnn or not')
    p.add_argument('--train_root_dir', default='data/layoutnet_dataset/train',
                   help='root directory to training dataset. should contains img, label_cor subdirectories')
    p.add_argument('--train_aug_root_dir', default=None,
                   help='root directory to an extra training dataset (img, label_cor). As in train.py, the main '
                        'dataset keeps the full --batch_size_train and this one adds --batch_size_train // 2 per step')
    p.add_argument('--valid_root_dir', default='data/layoutnet_dataset/valid',
                   help='root directory to validation dataset. should contains img, label_cor subdirectories')
    p.add_argument('--no_flip', action='store_true', help='disable left-right flip augmentation')
    p.add_argument('--no_rotate', action='store_true', help='disable horizontal rotate augmentation')
    p.add_argument('--no_gamma', action='store_true', help='disable gamma augmentation')
    p.add_argument('--no_pano_stretch', action='store_true', help='disable pano stretch')
    p.add_argument('--num_workers', default=8, type=int, help='host threads decoding images')
    p.add_argument('--freeze_earlier_blocks', default=-1, type=int)
    p.add_argument('--batch_size_train', default=8, type=int, help='training mini-batch size')
    p.add_argument('--batch_size_valid', default=2, type=int, help='validation mini-batch size')
    p.add_argument('--epochs', default=300, type=int, help='epochs to train')
    p.add_argument('--optim', default='Adam', help='optimizer to use. only support SGD and Adam')
    p.add_argument('--lr', default=1e-4, type=float, help='learning rate')
    p.add_argument('--lr_pow', default=0.9, type=float, help='power in poly to drop LR')
    p.add_argument('--warmup_lr', default=1e-6, type=float, help='starting learning rate for warm up')
    p.add_argument('--warmup_epochs', default=0, type=int, help='numbers of warmup epochs')
    p.add_argument('--beta1', default=0.9, type=float, help='momentum for sgd, beta1 for adam')
    p.add_argument('--weight_decay', default=0, type=float, help='factor for L2 regularization')
    p.add_argument('--bn_momentum', type=float)
    p.add_argument('--no_cuda', action='store_true', help='not supported: the library has no CPU path')
    p.add_argument('--multi_gpu', action='store_true', help='not supported: train one GPU per process')
    p.add_argument('--device', default='0', help='the GPU to use')
    p.add_argument('--seed', default=594277, type=int, help='manual seed')
    p.add_argument('--disp_iter', type=int, default=1, help='iterations frequency to display')
    p.add_argument('--save_every', type=int, default=25, help='epochs frequency to save state_dict')
    args = p.parse_args(argv)
    if args.no_cuda:
        p.error('--no_cuda is not supported: horizonnet_b200 has no CPU path')
    if args.multi_gpu or ',' in args.device:
        p.error('--multi_gpu is not supported: run one process per GPU (parallel.average_gradients, INTEGRATION.md)')
    if not -1 <= args.freeze_earlier_blocks <= 4:
        p.error('--freeze_earlier_blocks must be in -1..4')
    if args.optim not in ('SGD', 'Adam'):
        p.error('--optim: only SGD and Adam are supported')
    return args


class ScalarLog:
    """The scalars train.py writes with tensorboardX, as JSON lines {"tag", "value", "step"}."""

    def __init__(self, path):
        os.makedirs(os.path.dirname(path), exist_ok=True)
        self.f = open(path, 'a')

    def add(self, tag, value, step):
        self.f.write(json.dumps({'tag': tag, 'value': float(value), 'step': int(step)}) + '\n')

    def flush(self):
        self.f.flush()


def build_net(args, dev):
    from .model import HorizonNet
    if args.pth is not None:
        print('Finetune model is given.')
        print('Ignore --backbone and --no_rnn')
        ck = torch.load(args.pth, map_location='cpu', weights_only=False)
        net = HorizonNet(**ck['kwargs'])
        net.load_state_dict(ck['state_dict'])
    else:
        net = HorizonNet(args.backbone, not args.no_rnn)
    net = net.to(dev)
    if args.freeze_earlier_blocks != -1:                                     # train.py:200-207
        blocks = net.feature_extractor.list_blocks()
        for i in range(args.freeze_earlier_blocks + 1):
            print('Freeze block%d' % i)
            for m in blocks[i]:
                for param in m.parameters():
                    param.requires_grad = False
    if args.bn_momentum:                                                     # train.py:209-213
        for m in net.modules():
            if isinstance(m, (nn.BatchNorm1d, nn.BatchNorm2d)):
                m.momentum = args.bn_momentum
    return net


def make_optimizer(args, net):
    params = [p for p in net.parameters() if p.requires_grad]
    if args.optim == 'SGD':
        return torch.optim.SGD(params, lr=args.lr, momentum=args.beta1, weight_decay=args.weight_decay)
    return torch.optim.Adam(params, lr=args.lr, betas=(args.beta1, 0.999), weight_decay=args.weight_decay)


def save_model(net, path, args):
    """misc/utils.py:49-58."""
    torch.save(OrderedDict({'args': dict(vars(args)), 'kwargs': {'backbone': net.backbone, 'use_rnn': net.use_rnn},
                            'state_dict': net.state_dict()}), path)


def train_step(net, optimizer, x, y_bon, y_cor):
    """One iteration of train.py:258-271 (fp32): forward, the two losses, backward, optimizer step.  Returns the device
    tensor [bon, cor, total] without reading it."""
    optimizer.zero_grad()
    bon_, cor_ = net(x)
    l_bon = F.l1_loss(bon_, y_bon)
    l_cor = F.binary_cross_entropy_with_logits(cor_, y_cor)
    total = l_bon + l_cor
    total.backward()
    optimizer.step()
    optimizer.zero_grad()
    return torch.stack([l_bon, l_cor, total]).detach()


def run_validation(net, loader, n_valid):
    """train.py:283-325 in batches: sums of the per-panorama losses (eval-mode forward) and validate's metrics, divided
    by the dataset size.  A panorama whose gt validate cannot score (where the reference would crash) is left out of
    the metric sums and named."""
    net.eval()
    sums = {k: 0.0 for k in ('bon', 'cor', 'total', '2DIoU', '3DIoU', 'rmse', 'delta_1')}
    first = 0
    with torch.no_grad():
        for x, y_bon, y_cor, cors in loader:
            bon_, cor_ = net(x)
            l_bon = F.l1_loss(bon_, y_bon, reduction='none').flatten(1).mean(1)
            l_cor = F.binary_cross_entropy_with_logits(cor_, y_cor, reduction='none').flatten(1).mean(1)
            sums['bon'] += float(l_bon.sum())
            sums['cor'] += float(l_cor.sum())
            sums['total'] += float((l_bon + l_cor).sum())
            res = validate(net, x, cors, return_status=True)
            for b, st in enumerate(res['status'].tolist()):
                if st not in (OK, DT_INVALID):
                    print('valid: %s left out: validate status %d (the reference cannot score it)'
                          % (loader.txt_fnames[first + b], st))
                    continue
                for k, r in (('2DIoU', 'iou2d'), ('3DIoU', 'iou3d'), ('rmse', 'rmse'), ('delta_1', 'delta_1')):
                    sums[k] += float(res[r][b])
            first += x.shape[0]
    return {k: v / n_valid for k, v in sums.items()}


def main(argv=None):
    args = parse_args(argv)
    dev = torch.device('cuda', int(args.device))
    torch.cuda.set_device(dev)
    np.random.seed(args.seed)
    torch.manual_seed(args.seed)
    os.makedirs(os.path.join(args.ckpt, args.id), exist_ok=True)
    try:
        net = build_net(args, dev)
    except NotImplementedError as e:
        sys.exit(str(e))
    aug = dict(flip=not args.no_flip, rotate=not args.no_rotate, gamma=not args.no_gamma, stretch=not args.no_pano_stretch)
    loader_train = PanoCorBonBatches(args.train_root_dir, args.batch_size_train, shuffle=True, drop_last=True,
                                     seed=args.seed, device=dev, num_threads=args.num_workers, **aug)
    print('training dataset contains %d images!!!' % len(loader_train.img_fnames))
    loader_aug = None
    if args.train_aug_root_dir:
        loader_aug = PanoCorBonBatches(args.train_aug_root_dir, args.batch_size_train // 2, shuffle=True, drop_last=True,
                                       seed=args.seed + 1, device=dev, num_threads=args.num_workers, **aug)
        print('train batch size: %d, train augmentation batch size: %d' % (args.batch_size_train,
                                                                           args.batch_size_train // 2))
    loader_valid = None
    if args.valid_root_dir:
        loader_valid = PanoCorBonBatches(args.valid_root_dir, args.batch_size_valid, device=dev,
                                         num_threads=args.num_workers, return_cor=True)
    if len(loader_train) == 0:
        sys.exit('the training set has fewer panoramas than --batch_size_train')
    optimizer = make_optimizer(args, net)
    log = ScalarLog(os.path.join(args.logs, args.id, 'scalars.jsonl'))

    warmup_iters = args.warmup_epochs * len(loader_train)
    max_iters = args.epochs * len(loader_train)
    cur_iter, best_valid_score = 0, 0
    aug_iter = iter(loader_aug) if loader_aug is not None else None
    for ep in range(1, args.epochs + 1):
        net.train()
        if args.freeze_earlier_blocks != -1:                                 # train.py:251-256
            blocks = net.feature_extractor.list_blocks()
            for i in range(args.freeze_earlier_blocks + 1):
                for m in blocks[i]:
                    m.eval()
        pending = []                                                         # (iteration, lr, device losses)

        def flush():
            if not pending:
                return
            vals = torch.stack([p[2] for p in pending]).cpu().numpy()
            for (it, lr, _), v in zip(pending, vals):
                for k, val in zip(('bon', 'cor', 'total'), v):
                    log.add('train/%s' % k, val, it)
                log.add('train/lr', lr, it)
            print('ep%d it%d: bon %.4f cor %.4f total %.4f lr %.3g' % (ep, pending[-1][0], *vals[-1], pending[-1][1]))
            pending.clear()
            log.flush()

        for x, y_bon, y_cor in loader_train:
            lr = learning_rate(cur_iter, args.lr, args.warmup_lr, args.lr_pow, warmup_iters, max_iters)
            for g in optimizer.param_groups:
                g['lr'] = lr
            cur_iter += 1
            if aug_iter is not None:
                try:
                    xa, ba, ca = next(aug_iter)
                except StopIteration:
                    aug_iter = iter(loader_aug)
                    xa, ba, ca = next(aug_iter)
                x, y_bon, y_cor = torch.cat((x, xa)), torch.cat((y_bon, ba)), torch.cat((y_cor, ca))
            pending.append((cur_iter, lr, train_step(net, optimizer, x, y_bon, y_cor)))
            if cur_iter % args.disp_iter == 0:
                flush()
        flush()

        if loader_valid is not None:
            v = run_validation(net, loader_valid, len(loader_valid.img_fnames))
            for k, val in v.items():
                log.add('valid/%s' % k, val, ep)
            log.flush()
            now = v['3DIoU']
            print('Ep%3d %.4f vs. Best %.4f' % (ep, now, best_valid_score))
            is_best = now > best_valid_score
            if is_best:
                best_valid_score = now
            path = os.path.join(args.ckpt, args.id, 'checkpoint.pth.tar')
            torch.save({'epoch': ep, 'state_dict': net.state_dict(), 'optimizer': optimizer.state_dict(),
                        'best_valid_score': best_valid_score, 'backbone': net.backbone}, path)
            if is_best:
                shutil.copyfile(path, os.path.join(args.ckpt, args.id, 'best_model_%d.pth.tar' % ep))
        if ep % args.save_every == 0:
            save_model(net, os.path.join(args.ckpt, args.id, 'epoch_%d.pth' % ep), args)


if __name__ == '__main__':
    main()
