#!/usr/bin/env python
"""InfoNCE / UberNCE pre-training driver -- same command line as the reference's main_nce.py (:38-93) for the
hot path this repository accelerates, plus:

  --synthetic            random clips of the dataset's shape instead of the LMDB loaders (without --synthetic or
                         --data-root a dataset name raises)
  --precision MODE       parity | mixed | fast (see DESIGN.md)
  --steps-per-epoch N    length of a synthetic epoch
  --gpu-augment          with --synthetic: the loader yields seeded uint8 source frames (--source-size H W, 240 320 by
                         default) and the reference's get_transform('train') runs on the GPU (coclr_b200.augment); the
                         clips go to the model in loader layout with the input normalisation fused
  --jpeg                 with --synthetic --gpu-augment: the loader holds a seeded pool of videos as lists of JPEG
                         bytes (the reference LMDB's value format, encoded once by Pillow at --source-size); each
                         batch's frames are decoded on the GPU (coclr_b200.jpeg) in front of the augmentation
  --data-root DIR        the reference's LMDB databases in its relative layout (UCF101/ucf101_frame.lmdb, ...,
  --split-root DIR       kinetics400-256/frame_full/lmdb/k400_frame_train.lmdb) and its split files (ucf101/, k400/
                         as in process_data/data/): the dataset is read with coclr_b200.datasets, each batch's
                         distinct frames are decoded once on the GPU and augmented there (coclr_b200.loaders)

Launch like the reference: `python -m torch.distributed.run --nproc_per_node=N main_nce.py ...` (one process per
GPU; --local_rank, --local-rank and the LOCAL_RANK env variable are all accepted).

What differs from the reference loop (main_nce.py:286-353), by design:
  * no DistributedDataParallel wrapper: the encoder's backward writes one flat gradient buffer that
    FlatAdam all-reduces (mean) in one NCCL call; weights and queue are replica-identical by construction, so DDP's
    per-step buffer broadcast (SURVEY.md C6) has nothing to do for them.  BatchNorm RUNNING statistics are per-rank
    (no SyncBN, as in the reference) and are not read in train mode; rank 0's copy is the one that is saved, which is
    what the reference's rank-0 broadcast + rank-0 save amounts to;
  * top-k accuracy and loss are accumulated on the device and read back every --print_freq steps
    (the reference forces three .item() syncs per step, main_nce.py:325-327).
"""
import argparse
import os
import random
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

from model.pretrain import InfoNCE, UberNCE
from coclr_b200 import moco


def parse_args(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument('--net', default='s3d', type=str)
    p.add_argument('--model', default='infonce', type=str)
    p.add_argument('--dataset', default='ucf101-2clip', type=str)
    p.add_argument('--seq_len', default=32, type=int, help='number of frames in each video block')
    p.add_argument('--num_seq', default=2, type=int, help='number of video blocks')
    p.add_argument('--ds', default=1, type=int, help='frame down sampling rate')
    p.add_argument('--batch_size', default=32, type=int)
    p.add_argument('--lr', default=1e-3, type=float, help='learning rate')
    p.add_argument('--schedule', default=[120, 160], nargs='*', type=int, help='epochs at which lr drops 10x')
    p.add_argument('--wd', default=1e-5, type=float, help='weight decay')
    p.add_argument('--resume', default='', type=str, help='path of model to resume')
    p.add_argument('--pretrain', default='', type=str, help='path of pretrained model')
    p.add_argument('--test', default='', type=str, help='path of model to load and pause')
    p.add_argument('--epochs', default=10, type=int)
    p.add_argument('--start_epoch', default=0, type=int)
    p.add_argument('--gpu', default=None, type=int)
    p.add_argument('--print_freq', default=5, type=int)
    p.add_argument('--save_freq', default=1, type=int)
    p.add_argument('--reset_lr', action='store_true')
    p.add_argument('--img_dim', default=128, type=int)
    p.add_argument('--prefix', default='pretrain', type=str)
    p.add_argument('--name_prefix', default='', type=str)
    p.add_argument('-j', '--workers', default=16, type=int)
    p.add_argument('--seed', default=0, type=int)
    p.add_argument('--world-size', default=-1, type=int)
    p.add_argument('--rank', default=-1, type=int)
    p.add_argument('--dist-url', default='env://', type=str)
    p.add_argument('--dist-backend', default='nccl', type=str)
    p.add_argument('--multiprocessing-distributed', action='store_true')
    p.add_argument('--local_rank', '--local-rank', dest='local_rank', default=-1, type=int)
    p.add_argument('--moco-dim', default=128, type=int)
    p.add_argument('--moco-k', default=2048, type=int)
    p.add_argument('--moco-m', default=0.999, type=float)
    p.add_argument('--moco-t', default=0.07, type=float)
    # additions
    p.add_argument('--synthetic', action='store_true')
    p.add_argument('--raw-input', action='store_true',
                   help='feed the loader layout [B,3,num_seq*seq_len,H,W] in [0,1]; T.Normalize + view + transpose of the '
                        'reference\'s GPU-side `tr` (main_nce.py:207-209,299-302) run fused in the clip-packing kernel')
    p.add_argument('--gpu-augment', action='store_true',
                   help='with --synthetic: augment seeded uint8 source frames on the GPU (get_transform("train"))')
    p.add_argument('--source-size', default=[240, 320], nargs=2, type=int, metavar=('H', 'W'),
                   help='height and width of the synthetic source frames of --gpu-augment')
    p.add_argument('--jpeg', action='store_true',
                   help='with --synthetic --gpu-augment: decode a pool of JPEG-encoded videos on the GPU in front of '
                        'the augmentation')
    p.add_argument('--data-root', default=None, help='directory of the reference\'s LMDB databases')
    p.add_argument('--split-root', default=None, help='directory of the reference\'s split files (ucf101/, k400/)')
    p.add_argument('--precision', default='parity', choices=['parity', 'mixed', 'fast'])
    p.add_argument('--steps-per-epoch', default=20, type=int)
    p.add_argument('--num-classes', default=101, type=int, help='label range of the synthetic UberNCE labels')
    return p.parse_args(argv)


def setup_distributed(args):
    env_world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.local_rank == -1 and "LOCAL_RANK" in os.environ:
        args.local_rank = int(os.environ["LOCAL_RANK"])
    args.world_size = env_world if args.world_size == -1 else args.world_size
    args.distributed = args.world_size > 1
    args.rank = int(os.environ.get("RANK", "0")) if args.rank == -1 else args.rank
    args.gpu = args.local_rank if args.local_rank != -1 else (args.gpu or 0)
    torch.cuda.set_device(args.gpu)
    if args.distributed:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group(backend=args.dist_backend, init_method=args.dist_url, world_size=args.world_size,
                                rank=args.rank)
    if args.rank != 0:                      # silence non-master prints (reference main_nce.py:147-151)
        import builtins
        builtins.print = lambda *a, **k: None


class SyntheticClips:
    """Stand-in for the *_2CLIP datasets after the GPU-side `tr` transform (main_nce.py:207-209,299-302):
    [B, 2, 3, T, H, W] fp32, N(0,1) like normalised frames, plus int64 labels."""

    def __init__(self, args, device):
        self.args, self.device = args, device
        self.gen = torch.Generator(device=device).manual_seed(args.seed * 1000 + args.rank)

    def __iter__(self):
        a = self.args
        for _ in range(a.steps_per_epoch):
            if getattr(a, "raw_input", False):   # what the reference's DataLoader yields before `tr`
                x = torch.rand(a.batch_size, 3, 2 * a.seq_len, a.img_dim, a.img_dim, device=self.device, generator=self.gen)
            else:
                x = torch.randn(a.batch_size, 2, 3, a.seq_len, a.img_dim, a.img_dim, device=self.device, generator=self.gen)
            y = torch.randint(0, a.num_classes, (a.batch_size,), device=self.device, generator=self.gen)
            yield x, y

    def __len__(self):
        return self.args.steps_per_epoch


class SyntheticSourceFrames:
    """--gpu-augment: seeded uint8 source frames [B, F, H, W, 3] (what stacked decoded JPEGs give) augmented on the
    GPU by the reference's get_transform('train').  The augmentation draws from its own random / np.random / torch
    generators, as the reference's do in its DataLoader workers, so the training loop's draws are unchanged."""

    def __init__(self, args, device, two_stream=False):
        from coclr_b200.augment import PretrainAugment
        self.args, self.device = args, device
        self.aug = PretrainAugment(args.seq_len, args.img_dim, two_stream=two_stream)
        seed = args.seed * 1000 + args.rank
        self.gen = torch.Generator(device=device).manual_seed(seed)
        self.py, self.np = random.Random(seed), np.random.RandomState(seed)
        self.tg = torch.Generator().manual_seed(seed)
        self.pool = None
        if getattr(args, 'jpeg', False):
            from coclr_b200.jpeg import JpegDecoder, JpegVideoPool
            h, w = args.source_size
            self.pool = JpegVideoPool(8, self.aug.frames, h, w, seed=seed)
            self.dec, self.pick = JpegDecoder(), random.Random(seed + 1)

    def __iter__(self):
        a = self.args
        h, w = a.source_size
        for _ in range(a.steps_per_epoch):
            if self.pool is not None:        # the dataset's pil_from_raw_rgb, on the GPU
                batch = self.dec.parse(self.pool.frames([self.pick.randrange(len(self.pool))
                                                         for _ in range(a.batch_size)]))
                frames = self.dec(batch)
                frames = frames.view(a.batch_size, self.aug.frames, *frames.shape[1:])
                plan = self.aug.plan(batch.sample_sizes(a.batch_size), self.py, self.np, self.tg)
                y = torch.randint(0, a.num_classes, (a.batch_size,), device=self.device, generator=self.gen)
                yield self.aug(frames, plan), y
                continue
            frames = torch.randint(0, 256, (a.batch_size, self.aug.frames, h, w, 3), dtype=torch.uint8,
                                   device=self.device, generator=self.gen)
            plan = self.aug.plan([(h, w)] * a.batch_size, self.py, self.np, self.tg)
            y = torch.randint(0, a.num_classes, (a.batch_size,), device=self.device, generator=self.gen)
            yield self.aug(frames, plan), y

    def __len__(self):
        return self.args.steps_per_epoch


def check_jpeg_flag(args):
    if getattr(args, 'jpeg', False) and not (args.synthetic and args.gpu_augment):
        raise NotImplementedError("--jpeg decodes the synthetic JPEG pool of --synthetic --gpu-augment")


def lmdb_dataset(args, mode='train'):
    """get_data of the reference's main_nce.py / main_coclr.py over --data-root / --split-root."""
    from coclr_b200 import datasets as D
    if not args.split_root:
        raise ValueError("--data-root needs --split-root (the reference's process_data/data directory)")
    data, split = args.data_root, args.split_root
    kw = dict(mode=mode, num_frames=args.seq_len, ds=args.ds, return_label=True)
    k400 = os.path.join(data, 'kinetics400-256')
    if args.dataset == 'ucf101-2clip':
        return D.UCF101LMDB_2CLIP(root=os.path.join(split, 'ucf101'),
                                  db_path=os.path.join(data, 'UCF101', 'ucf101_frame.lmdb'), **kw)
    if args.dataset == 'ucf101-f-2clip':
        return D.UCF101Flow_LMDB_2CLIP(root=os.path.join(split, 'ucf101'),
                                       db_path=os.path.join(data, 'UCF101', 'ucf101_tvl1_frame.lmdb'), **kw)
    if args.dataset == 'k400-2clip':
        return D.K400_LMDB_2CLIP(root=os.path.join(split, 'k400'),
                                 db_path=os.path.join(k400, 'frame_full', 'lmdb'), **kw)
    if args.dataset == 'k400-f-2clip':
        return D.K400_Flow_LMDB_2CLIP(root=os.path.join(split, 'k400'),
                                      db_path=os.path.join(k400, 'tvl1_flow', 'lmdb'), **kw)
    if args.dataset == 'ucf101-2stream-2clip':
        return D.UCF101_2STREAM_LMDB_2CLIP(root=os.path.join(split, 'ucf101'),
                                           db_path_flow=os.path.join(data, 'UCF101', 'ucf101_tvl1_frame.lmdb'),
                                           db_path_rgb=os.path.join(data, 'UCF101', 'ucf101_frame.lmdb'),
                                           return_source=True, **kw)
    if args.dataset == 'k400-2stream-2clip':
        return D.K400_2STREAM_LMDB_2CLIP(root=os.path.join(split, 'k400'),
                                         db_path_flow=os.path.join(k400, 'tvl1_flow', 'lmdb'),
                                         db_path_rgb=os.path.join(k400, 'frame_full', 'lmdb'),
                                         return_source=True, **kw)
    raise NotImplementedError("dataset %r" % args.dataset)


def lmdb_loader(args, device, two_stream=False):
    """Pre-training batches of --data-root: what SyntheticSourceFrames yields, from the dataset's frames."""
    from coclr_b200.loaders import PretrainBatches
    if two_stream != args.dataset.endswith('2stream-2clip'):
        raise NotImplementedError("dataset %r" % args.dataset)
    return PretrainBatches(lmdb_dataset(args), args.batch_size, args.seq_len, args.img_dim, device,
                           seed=args.seed * 1000 + args.rank, rank=args.rank, world_size=args.world_size,
                           two_stream=two_stream)


def get_data(args, device):
    if getattr(args, 'data_root', None) and not args.synthetic:
        check_jpeg_flag(args)
        return lmdb_loader(args, device)
    if not args.synthetic:
        raise NotImplementedError(
            "dataset %r: the LMDB/JPEG loaders of the reference (dataset/) are outside the accelerated hot path; run "
            "with --synthetic, or feed [B,2,3,T,H,W] float tensors (or uint8 frames through coclr_b200.augment) from "
            "your own loader" % args.dataset)
    check_jpeg_flag(args)
    return SyntheticSourceFrames(args, device) if args.gpu_augment else SyntheticClips(args, device)


def adjust_learning_rate(optimizer, epoch, args):
    """lr = base * 0.1 ** (#milestones passed) (reference main_nce.py:356-363)."""
    lr = args.lr
    for milestone in args.schedule:
        lr *= 0.1 if epoch >= milestone else 1.
    for g in optimizer.param_groups:
        g['lr'] = lr


def set_path(args):
    if args.resume:
        exp_path = os.path.dirname(os.path.dirname(args.resume))
    elif args.test:
        exp_path = os.path.dirname(os.path.dirname(args.test))
    else:
        exp_path = 'log-{a.prefix}/{a.name_prefix}{a.model}_k{a.moco_k}_{a.dataset}-{a.img_dim}_{a.net}_' \
                   'bs{a.batch_size}_lr{a.lr}_seq{a.num_seq}_len{a.seq_len}_ds{a.ds}'.format(a=args)
    model_path = os.path.join(exp_path, 'model')
    if args.rank == 0:
        os.makedirs(model_path, exist_ok=True)
    return model_path


def save_checkpoint(state, is_best, gap, filename, keep_all=False):
    """torch.save + prune the checkpoint `gap` epochs back (reference utils/utils.py:12-26)."""
    torch.save(state, filename)
    last = os.path.join(os.path.dirname(filename), 'epoch%d.pth.tar' % (state['epoch'] - gap))
    if not keep_all and os.path.exists(last):
        os.remove(last)
    if is_best:
        torch.save(state, os.path.join(os.path.dirname(filename), 'model_best_epoch%d.pth.tar' % state['epoch']))


def multi_label_nce_loss(logits, mask):
    """UberNCE loss: -(log_softmax * mask).sum(1) / mask.sum(1), mean (reference main_nce.py:321-322)."""
    return -(torch.log_softmax(logits, dim=1) * mask).sum(1).div(mask.sum(1)).mean()


def train_one_epoch(loader, model, optimizer, epoch, args):
    model.train()
    stat = torch.zeros(4, device=torch.device('cuda', args.gpu))  # loss sum, top1 sum, top5 sum, steps
    tic = time.time()
    for idx, (input_seq, label) in enumerate(loader):
        if args.model == 'infonce':
            output, target = model(input_seq)
            loss = moco.nce_cross_entropy(output, target)
            with torch.no_grad():
                top5 = output.topk(5, dim=1).indices
                stat[1] += (top5[:, 0] == 0).float().mean()
                stat[2] += (top5 == 0).any(1).float().mean()
        else:
            output, mask = model(input_seq, label)
            loss = multi_label_nce_loss(output, mask)
            with torch.no_grad():
                top5 = output.topk(5, dim=1).indices
                hit = mask.gather(1, top5)
                stat[1] += hit[:, 0].float().mean()
                stat[2] += hit.any(1).float().mean()
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
        with torch.no_grad():
            stat[0] += loss.detach()
            stat[3] += 1
        args.iteration += 1
        if idx % args.print_freq == 0:
            s = stat.tolist()                                   # the only host sync, every print_freq steps
            n = max(s[3], 1.0)
            dt = (time.time() - tic) / n
            print('Epoch: [%d][%d/%d] loss %.4f top1 %.3f top5 %.3f  %.1f ms/step  %.0f clips/s'
                  % (epoch, idx, len(loader), s[0] / n, s[1] / n, s[2] / n, dt * 1e3,
                     2 * args.batch_size * max(args.world_size, 1) / dt))
    s = stat.tolist()
    n = max(s[3], 1.0)
    return s[0] / n, s[1] / n


def load_optimizer_state(optimizer, sd, encoder, device):
    """Restore FlatAdam from a checkpoint's 'optimizer' entry: either FlatAdam's own flat state or a torch.optim.Adam
    state_dict as the reference writes it (main_nce.py:190-200,276: one param group per named_parameter of the WHOLE
    model in named_parameters() order; only the encoder_q tensors carry state).  Returns False when nothing usable was
    found (the moments then restart from zero, which the caller reports)."""
    if not isinstance(sd, dict):
        return False
    if 'exp_avg' in sd:
        optimizer.load_state_dict({k: (v.to(device) if torch.is_tensor(v) else v) for k, v in sd.items()})
        return True
    state, groups = sd.get('state'), sd.get('param_groups')
    if not isinstance(state, dict) or not groups:
        return False
    named = list(encoder.named_parameters())      # encoder_q's tensors are the first entries of the reference's list
    ids = [i for g in groups for i in g['params']]
    if len(ids) < len(named):
        return False
    st = optimizer._state()
    steps = []
    for (name, p), i in zip(named, ids):
        ent = state.get(i)
        if ent is None:
            continue
        if tuple(ent['exp_avg'].shape) != tuple(p.shape):
            print('[WARNING] optimizer state of parameter %d does not have the shape of %s' % (i, name))
            return False
        off, n, _ = st.offsets[name]
        optimizer.exp_avg[off:off + n].copy_(ent['exp_avg'].reshape(-1).to(device))
        optimizer.exp_avg_sq[off:off + n].copy_(ent['exp_avg_sq'].reshape(-1).to(device))
        steps.append(int(ent['step']))
    if not steps:
        return False
    optimizer.step_count = max(steps)
    g0 = groups[0]
    optimizer.param_groups[0].update({k: g0[k] for k in ('lr', 'betas', 'eps', 'weight_decay') if k in g0})
    return True


def main_worker(args):
    setup_distributed(args)
    device = torch.device('cuda', args.gpu)
    torch.manual_seed(args.seed)
    np.random.seed(args.seed)
    random.seed(args.seed)
    cls = {'infonce': InfoNCE, 'ubernce': UberNCE}[args.model]
    model = cls(args.net, args.moco_dim, args.moco_k, args.moco_m, args.moco_t, precision=args.precision).to(device)
    if args.raw_input or args.gpu_augment or (args.data_root and not args.synthetic):
        model.set_input_transform(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])   # reference main_nce.py:207-209
    optimizer = moco.FlatAdam(model.encoder_q, lr=args.lr, weight_decay=args.wd)
    args.iteration = 1
    best_acc = 0.0
    if args.resume or args.pretrain or args.test:
        path = args.resume or args.test or args.pretrain
        ckpt = torch.load(path, map_location='cpu')
        missing = model.load_state_dict(ckpt['state_dict'], strict=not args.pretrain)
        print('loaded %s (epoch %s) %s' % (path, ckpt.get('epoch'), missing if args.pretrain else ''))
        if args.resume:
            args.start_epoch = ckpt['epoch'] + 1              # reference main_nce.py:218
            args.iteration = ckpt.get('iteration', 1)
            best_acc = ckpt.get('best_acc', 0.0)
            if not args.reset_lr and not load_optimizer_state(optimizer, ckpt.get('optimizer'), model.encoder_q, device):
                print('[WARNING] Not loading optimizer states')      # reference main_nce.py:231-232
    if args.test:
        return model
    loader = get_data(args, device)
    model_path = set_path(args)
    try:
        for epoch in range(args.start_epoch, args.epochs):
            np.random.seed(epoch)
            random.seed(epoch)
            adjust_learning_rate(optimizer, epoch, args)
            loss, acc = train_one_epoch(loader, model, optimizer, epoch, args)
            if args.rank == 0 and ((epoch % args.save_freq == 0) or (epoch == args.epochs - 1)):
                is_best = acc > best_acc
                best_acc = max(acc, best_acc)
                save_checkpoint({'epoch': epoch, 'state_dict': model.state_dict(), 'best_acc': best_acc,
                                 'optimizer': optimizer.state_dict(), 'iteration': args.iteration},
                                is_best, gap=args.save_freq,
                                filename=os.path.join(model_path, 'epoch%d.pth.tar' % epoch),
                                keep_all='k400' in args.dataset)
    finally:
        if hasattr(loader, 'close'):
            loader.close()
    print('Training from ep %d to ep %d finished' % (args.start_epoch, args.epochs))
    if args.distributed:
        dist.destroy_process_group()
    return model


if __name__ == '__main__':
    main_worker(parse_args())
