#!/usr/bin/env python
"""CoCLR co-training driver -- command line of the reference's main_coclr.py (:38-95) for the accelerated hot
path, with --synthetic / --gpu-augment / --jpeg / --precision / --steps-per-epoch as in main_nce.py.

Loop semantics kept from the reference (main_coclr.py:348-435): the sampler stays in eval mode (:363); the
self-positive column is masked out with probability 0.9 for rows that have other positives (:382-388, Python
`random`); no optimizer step is taken until the queue is full (:403-406) while EMA / enqueue still run.
Dropped: torch.cuda.empty_cache() every step (:409) and the per-step .item() syncs (:396-400).
"""
import os
import random
import sys
import time

import numpy as np
import torch
import torch.distributed as dist
import torch.nn.functional as F

import main_nce as base
from model.pretrain import CoCLR
from coclr_b200 import moco


def parse_args(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    extra = {"topk": 5, "reverse": False, "pretrain": ['random', 'random']}
    rest = []
    i = 0
    while i < len(argv):
        a = argv[i]
        if a == '--topk':
            extra["topk"] = int(argv[i + 1]); i += 2
        elif a == '--reverse':
            extra["reverse"] = True; i += 1
        elif a == '--cos':      # accepted and unused, exactly as in the reference (main_coclr.py:92-93, never read)
            i += 1
        elif a == '--pretrain':
            extra["pretrain"] = [argv[i + 1], argv[i + 2]]; i += 3
        else:
            rest.append(a); i += 1
    args = base.parse_args(rest)
    if '--model' not in rest:
        args.model = 'coclr'
    if '--dataset' not in rest:
        args.dataset = 'ucf101-2stream-2clip'
    args.topk, args.reverse, args.pretrain2 = extra["topk"], extra["reverse"], extra["pretrain"]
    return args


def multi_nce_loss(logits, mask):
    """-log sum(softmax(logits) * mask) (reference main_coclr.py:343-346)."""
    return (-torch.log((F.softmax(logits, dim=1) * mask).sum(1))).mean()


class SyntheticTwoStream:
    """Stand-in for the 2-stream 2-clip datasets (lmdb_dataset.py:372-528): two blocks [B,2(view),3,T,H,W] and
    an int64 video id per sample."""

    def __init__(self, args, device):
        self.args, self.device = args, device
        self.gen = torch.Generator(device=device).manual_seed(args.seed * 1000 + args.rank)

    def __iter__(self):
        a = self.args
        shape = (a.batch_size, 2, 3, a.seq_len, a.img_dim, a.img_dim)
        for _ in range(a.steps_per_epoch):
            b1 = torch.randn(shape, device=self.device, generator=self.gen)
            b2 = torch.randn(shape, device=self.device, generator=self.gen)
            vname = torch.randint(0, 10000, (a.batch_size,), device=self.device, generator=self.gen)
            yield (b1, b2), vname

    def __len__(self):
        return self.args.steps_per_epoch


def _strip_module(k):
    return k[len('module.'):] if k.startswith('module.') else k


def two_checkpoint_state(paths):
    """State dict of the reference's two-checkpoint initialisation (main_coclr.py:250-302):
      * second path = the ORACLE: only its encoder_q.* weights, renamed sampler.* (never trained here);
      * first path  = the network to train: only its encoder_q.* weights, copied into BOTH encoder_q.* and encoder_k.*
        (its own encoder_k.* EMA weights, its sampler.* -- present from co-training cycle 2 on -- and every queue
        buffer are dropped);
      * merged as {**first, **second}; the queues are always re-filled."""
    second = {}
    if os.path.isfile(paths[1]):
        ckpt = torch.load(paths[1], map_location='cpu')
        for k, v in ckpt['state_dict'].items():
            k = _strip_module(k)
            if 'encoder_q.' in k and 'queue' not in k:
                second[k.replace('encoder_q.', 'sampler.')] = v
        print("=> Use Oracle checkpoint '%s' (epoch %s)" % (paths[1], ckpt.get('epoch')))
    else:
        print("=> NO Oracle checkpoint found at '%s', use random init" % paths[1])
    first = {}
    if os.path.isfile(paths[0]):
        ckpt = torch.load(paths[0], map_location='cpu')
        for k, v in ckpt['state_dict'].items():
            k = _strip_module(k)
            if 'encoder_q.' in k and 'queue' not in k:
                first[k] = v
                first[k.replace('encoder_q.', 'encoder_k.')] = v
        print("=> Use Training checkpoint '%s' (epoch %s)" % (paths[0], ckpt.get('epoch')))
    else:
        print("=> NO Training checkpoint found at '%s', use random init" % paths[0])
    state = {**first, **second}
    state.pop('queue_label', None)
    return state


def load_two_checkpoints(model, paths):
    """One non-strict load of two_checkpoint_state() (the reference uses neq_load_customized, main_coclr.py:302)."""
    res = model.load_state_dict(two_checkpoint_state(paths), strict=False)
    print('missing keys: %d, unexpected keys: %d' % (len(res.missing_keys), len(res.unexpected_keys)))
    return res


def train_one_epoch(loader, model, optimizer, epoch, args):
    model.train()
    model.sampler.eval()                                           # the sampler is always fixed (:363)
    stat = torch.zeros(3, device=torch.device('cuda', args.gpu))   # loss, self-top1, steps
    tic = time.time()
    for idx, ((block1, block2), vname) in enumerate(loader):
        output, mask = model(block1, block2, vname)
        mask_sum = mask.sum(1)
        if random.random() < 0.9:
            mask_clone = mask.clone()
            mask_clone[mask_sum != 1, 0] = 0                       # mask out self-similarity (:382-388)
            loss = multi_nce_loss(output, mask_clone)
        else:
            loss = multi_nce_loss(output, mask)
        if model.queue_is_full:                                    # (:403-406)
            optimizer.zero_grad()
            loss.backward()
            optimizer.step()
        with torch.no_grad():
            stat[0] += loss.detach()
            stat[1] += (output.argmax(1) == 0).float().mean()
            stat[2] += 1
        args.iteration += 1
        if idx % args.print_freq == 0:
            s = stat.tolist()
            n = max(s[2], 1.0)
            dt = (time.time() - tic) / n
            print('Epoch: [%d][%d/%d] loss %.4f self-top1 %.3f queue_full %s  %.1f ms/step'
                  % (epoch, idx, len(loader), s[0] / n, s[1] / n, model.queue_is_full, dt * 1e3))
    s = stat.tolist()
    return s[0] / max(s[2], 1.0), s[1] / max(s[2], 1.0)


def main_worker(args):
    base.setup_distributed(args)
    device = torch.device('cuda', args.gpu)
    torch.manual_seed(args.seed)
    np.random.seed(args.seed)
    random.seed(args.seed)
    model = CoCLR(args.net, args.moco_dim, args.moco_k, args.moco_m, args.moco_t, topk=args.topk,
                  reverse=args.reverse, precision=args.precision)
    model = model.to(device)
    optimizer = moco.FlatAdam(model.encoder_q, lr=args.lr, weight_decay=args.wd)
    args.iteration = 1
    best_acc = 0.0
    if args.resume:                                               # restart training (reference main_coclr.py:230-248)
        if os.path.isfile(args.resume):
            ckpt = torch.load(args.resume, map_location='cpu')
            args.start_epoch = ckpt['epoch'] + 1
            args.iteration = ckpt.get('iteration', 1)
            best_acc = ckpt.get('best_acc', 0.0)
            try:
                model.load_state_dict(ckpt['state_dict'])
            except RuntimeError:
                print('[WARNING] Non-Equal load for resuming training!')
                print(model.load_state_dict(ckpt['state_dict'], strict=False))
            print("=> load resumed checkpoint '%s' (epoch %d)" % (args.resume, ckpt['epoch']))
            if not base.load_optimizer_state(optimizer, ckpt.get('optimizer'), model.encoder_q, device):
                print('[WARNING] Not loading optimizer states')
        else:
            print("[Warning] no checkpoint found at '%s', use random init" % args.resume)
    elif args.pretrain2 != ['random', 'random']:
        load_two_checkpoints(model, args.pretrain2)
    if args.test:
        return model
    if not args.synthetic:
        raise NotImplementedError("the 2-stream LMDB datasets are outside the accelerated hot path; use --synthetic")
    base.check_jpeg_flag(args)
    if args.gpu_augment:
        model.set_input_transform(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])
        loader = base.SyntheticSourceFrames(args, device, two_stream=True)
    else:
        loader = SyntheticTwoStream(args, device)
    model_path = base.set_path(args)
    for epoch in range(args.start_epoch, args.epochs):
        np.random.seed(epoch)                                      # reference main_coclr.py:314-315: the 90 % self-mask
        random.seed(epoch)                                         # draws restart per epoch (reproducible across resume)
        base.adjust_learning_rate(optimizer, epoch, args)
        loss, acc = train_one_epoch(loader, model, optimizer, epoch, args)
        if args.rank == 0 and ((epoch % args.save_freq == 0) or (epoch == args.epochs - 1)):
            is_best = acc > best_acc
            best_acc = max(acc, best_acc)
            base.save_checkpoint({'epoch': epoch, 'state_dict': model.state_dict(), 'best_acc': best_acc,
                                  'optimizer': optimizer.state_dict(), 'iteration': args.iteration},
                                 is_best, gap=args.save_freq,
                                 filename=os.path.join(model_path, 'epoch%d.pth.tar' % epoch),
                                 keep_all='k400' in args.dataset)
    print('Training from ep %d to ep %d finished' % (args.start_epoch, args.epochs))
    if args.distributed:
        dist.destroy_process_group()
    return model


if __name__ == '__main__':
    main_worker(parse_args())
