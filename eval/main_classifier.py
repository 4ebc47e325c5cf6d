#!/usr/bin/env python
"""Fine-tuning / linear-probe driver -- same command line as the reference's eval/main_classifier.py (:37-77) for the
train / validate loop, on the engine's LinearClassifier (model/classifier.py), plus:

  --synthetic            random clips [B, 3, seq_len, img_dim, img_dim] with labels in [0, num_class) instead of the
                         LMDB loaders (without it a dataset name raises, as in main_nce.py)
  --precision MODE       parity | mixed | fast (see DESIGN.md)
  --steps-per-epoch N    length of a synthetic epoch (the validation pass takes the same number of steps)

--train_what last (linear probe: l2norm + final BN, no dropout, frozen eval-mode backbone), ft (backbone at lr / 10)
and all (everything at lr) select the parameters and learning rates as the reference does (:102-147); the optimizer is
Adam with coupled L2 (--wd) as one launch per group over flat buffers (coclr_b200.moco.SpanAdam).  Accuracy and loss are
accumulated on the device and read back every --print_freq steps.

--test CKPT with --retrieval (nearest-neighbour retrieval, R@1/5/10/20/50) or --center_crop / --five_crop / --ten_crop
(per-video test accuracy over the crops) runs the reference's test paths (:170-208, :425-718) on the engine
(coclr_b200.evaluate) and writes the reference's output files.  The per-video LMDB datasets are not part of this
repository, so these paths run with --synthetic only (the PIL crop / scale / jitter transforms run on the GPU with
--gpu-augment):

  --synthetic-videos N   videos per split: seeded, 1-4 clips each, a per-class pattern so that the accuracies are well
                         above chance; every (crop, flip) view of a video has its own deterministic content

  --gpu-augment          with --synthetic: seeded uint8 source frames (--source-size H W, 240 320 by default) go through
                         the reference's PIL transforms on the GPU (coclr_b200.clf_augment): get_transform('train' /
                         'val') with the train batch's flip for training and validation, and the flip / FiveCrop /
                         CenterCrop / Scale / ColorJitter views of --test; the test videos carry the per-class pattern
                         at source resolution.  Training feeds [0, 1] clips with the input normalisation fused
                         (LinearClassifier.set_input_transform)
  --jpeg                 with --synthetic --gpu-augment: the training and validation loaders hold a seeded pool of
                         videos as lists of JPEG bytes (the reference LMDB's value format, encoded once by Pillow at
                         --source-size), decoded on the GPU (coclr_b200.jpeg) in front of the augmentation

--optim sgd and more than one GPU (the reference's nn.DataParallel) are not available: they raise.
"""
import argparse
import json
import os
import pickle
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

from model.classifier import LinearClassifier  # noqa: E402
from coclr_b200 import moco  # noqa: E402
from coclr_b200 import evaluate as EV  # noqa: E402

NUM_CLASS = {'ucf101': 101, 'hmdb51': 51, 'k400': 400, 'ucf101-f': 101, 'hmdb51-f': 51, 'k400-f': 400}   # :98-100


def parse_args(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument('--net', default='s3d', type=str)
    p.add_argument('--model', default='lincls', type=str)
    p.add_argument('--dataset', default='ucf101', type=str)
    p.add_argument('--which_split', default=1, type=int)
    p.add_argument('--seq_len', default=32, type=int, help='number of frames in each video block')
    p.add_argument('--num_seq', default=1, type=int, help='number of video blocks')
    p.add_argument('--num_fc', default=1, type=int, help='number of fc')
    p.add_argument('--ds', default=1, type=int, help='frame down sampling rate')
    p.add_argument('--batch_size', default=32, type=int, help='batch size per GPU')
    p.add_argument('--optim', default='adam', type=str)
    p.add_argument('--lr', default=1e-3, type=float, help='learning rate')
    p.add_argument('--schedule', default=[60, 80], nargs='*', type=int, help='epochs at which lr drops 10x')
    p.add_argument('--wd', default=1e-3, type=float, help='weight decay')
    p.add_argument('--dropout', default=0.9, type=float, help='dropout')
    p.add_argument('--epochs', default=10, type=int, help='number of total epochs to run')
    p.add_argument('--start_epoch', default=0, type=int, help='manual epoch number (useful on restarts)')
    p.add_argument('--gpu', default=None, type=str)
    p.add_argument('--train_what', default='last', type=str)
    p.add_argument('--img_dim', default=128, type=int)
    p.add_argument('--print_freq', default=5, type=int, help='frequency of printing output during training')
    p.add_argument('--eval_freq', default=1, type=int)
    p.add_argument('--reset_lr', action='store_true', help='Reset learning rate when resume training?')
    p.add_argument('--prefix', default='linclr', type=str)
    p.add_argument('-j', '--workers', default=8, type=int)
    p.add_argument('--cos', action='store_true', help='use cosine lr schedule')
    p.add_argument('--resume', default='', type=str, help='path of model to resume')
    p.add_argument('--pretrain', default='', type=str, help='path of pretrained model')
    p.add_argument('--test', default='', type=str, help='path of model to load and pause')
    p.add_argument('--retrieval', action='store_true', help='path of model to ucf retrieval')
    p.add_argument('--dirname', default=None, type=str, help='dirname for feature')
    p.add_argument('--center_crop', action='store_true')
    p.add_argument('--five_crop', action='store_true')
    p.add_argument('--ten_crop', action='store_true')
    # additions
    p.add_argument('--synthetic', action='store_true')
    p.add_argument('--precision', default='parity', choices=['parity', 'mixed', 'fast'])
    p.add_argument('--steps-per-epoch', default=20, type=int)
    p.add_argument('--synthetic-videos', default=24, type=int, help='videos per split of the synthetic test sets')
    p.add_argument('--gpu-augment', action='store_true',
                   help='with --synthetic: augment seeded uint8 source frames on the GPU (the reference\'s transforms)')
    p.add_argument('--source-size', default=[240, 320], nargs=2, type=int, metavar=('H', 'W'),
                   help='height and width of the synthetic source frames of --gpu-augment')
    p.add_argument('--jpeg', action='store_true',
                   help='with --synthetic --gpu-augment: decode a pool of JPEG-encoded videos on the GPU in front of '
                        'the train / val augmentation')
    return p.parse_args(argv)


def check_supported(args):
    """Raise for what this driver does not run (see the module docstring)."""
    for flag in ('test', 'retrieval', 'center_crop', 'five_crop', 'ten_crop'):
        if getattr(args, flag) and not args.synthetic:
            raise NotImplementedError("--%s needs the per-video LMDB test datasets of the reference (dataset/), which are "
                                      "not part of this repository; run it with --synthetic" % flag)
    if args.jpeg and not (args.synthetic and args.gpu_augment):
        raise NotImplementedError("--jpeg decodes the synthetic JPEG pool of --synthetic --gpu-augment")
    if args.optim != 'adam':
        raise NotImplementedError("--optim %s: only Adam is available (--optim adam)" % args.optim)
    if args.model != 'lincls':
        raise NotImplementedError("--model %s" % args.model)
    if args.train_what not in ('last', 'ft', 'all'):
        raise ValueError("--train_what must be last, ft or all")
    if args.gpu is not None and len(str(args.gpu).split(',')) > 1:
        raise NotImplementedError("--gpu %s: multi-GPU fine-tuning (the reference's nn.DataParallel) is not available; "
                                  "use one GPU" % args.gpu)
    if args.dataset not in NUM_CLASS:
        raise NotImplementedError("dataset %r" % args.dataset)


def build_model(args):
    """LinearClassifier in the configuration of --train_what (:102-118) and the parameters it trains (:125-147)."""
    last = args.train_what == 'last'
    args.final_bn, args.final_norm, args.use_dropout = last, last, not last
    model = LinearClassifier(network=args.net, num_class=args.num_class, dropout=args.dropout,
                             use_dropout=args.use_dropout, use_final_bn=args.final_bn, use_l2_norm=args.final_norm,
                             precision=args.precision)
    if last:
        for p in model.backbone.parameters():
            p.requires_grad = False
    return model


def build_optimizer(model, args):
    """Adam groups (:125-161): the head at lr, plus the backbone at lr / 10 (ft) or lr (all); none for it with last."""
    spans = model.flat_spans()
    groups = [dict(name='head', params=spans['head'][0], grad=spans['head'][1], lr=args.lr)]
    if args.train_what != 'last':
        groups.insert(0, dict(name='backbone', params=spans['backbone'][0], grad=spans['backbone'][1],
                              lr=args.lr / 10 if args.train_what == 'ft' else args.lr))
    return moco.SpanAdam(groups, weight_decay=args.wd)


def map_pretrained(state_dict):
    """Pre-training checkpoint keys -> classifier keys: encoder_q.0. -> backbone. (:251-255); the DistributedDataParallel
    prefix of the reference's pre-training checkpoints is dropped first."""
    out = {}
    for k, v in state_dict.items():
        if k.startswith('module.'):
            k = k[len('module.'):]
        out[k.replace('encoder_q.0.', 'backbone.')] = v
    return out


def load_pretrained(model, state_dict):
    """Non-strict load of the backbone part; returns the classifier keys that the checkpoint did not provide."""
    sd = {k: v for k, v in map_pretrained(state_dict).items() if k in model.state_dict()}
    return model.load_state_dict(sd, strict=False).missing_keys


def adjust_learning_rate(optimizer, epoch, args):
    """Every group's lr x 0.1 at an epoch listed in --schedule (:721-726); unlike main_nce.py, the drop is applied to
    the current lr at that epoch, not recomputed from the base lr."""
    ratio = 0.1 if epoch in args.schedule else 1.
    for g in optimizer.param_groups:
        g['lr'] = g['lr'] * ratio


class SyntheticClips:
    """Stand-in for the classification datasets after the GPU-side transform: [B, 3, seq_len, H, W] fp32 N(0, 1) and
    labels in [0, num_class)."""

    def __init__(self, args, device, seed):
        self.args, self.device = args, device
        self.gen = torch.Generator(device=device).manual_seed(seed)

    def __iter__(self):
        a = self.args
        for _ in range(a.steps_per_epoch):
            x = torch.randn(a.batch_size, 3, a.seq_len, a.img_dim, a.img_dim, device=self.device, generator=self.gen)
            y = torch.randint(0, a.num_class, (a.batch_size,), device=self.device, generator=self.gen)
            yield x, y

    def __len__(self):
        return self.args.steps_per_epoch


def get_data(args, device, mode):
    if not args.synthetic:
        raise NotImplementedError(
            "dataset %r: the LMDB loaders and PIL augmentations of the reference (dataset/, utils/augmentation.py) are "
            "outside the accelerated hot path; run with --synthetic, or feed [B,3,T,H,W] float tensors from your own "
            "loader" % args.dataset)
    seed = args.seed_base + (0 if mode == 'train' else 1)
    if args.gpu_augment:
        return SyntheticSourceClips(args, device, seed, mode)
    return SyntheticClips(args, device, seed=seed)


class SyntheticSourceClips:
    """--gpu-augment: seeded uint8 source frames [B, num_seq * seq_len, H, W, 3] (what stacked decoded JPEGs give) and
    labels, augmented on the GPU by get_transform(mode) (coclr_b200.clf_augment).  The augmentation draws from its own
    random.Random, as the reference's DataLoader workers do; the train batch's flip (T.RandomHorizontalFlip of
    transform_train_cuda) is drawn from `random` itself, where the reference's main process draws it."""

    def __init__(self, args, device, seed, mode):
        from coclr_b200.clf_augment import ClassifierAugment
        self.args, self.device, self.mode = args, device, mode
        self.aug = ClassifierAugment(mode, args.seq_len, args.img_dim, num_seq=args.num_seq)
        self.gen = torch.Generator(device=device).manual_seed(seed)
        self.py = random.Random(seed)
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
                sizes = batch.sample_sizes(a.batch_size)
            else:
                frames = torch.randint(0, 256, (a.batch_size, self.aug.frames, h, w, 3), dtype=torch.uint8,
                                       device=self.device, generator=self.gen)
                sizes = [(h, w)] * a.batch_size
            y = torch.randint(0, a.num_class, (a.batch_size,), device=self.device, generator=self.gen)
            plan = self.aug.plan(sizes, self.py)
            if self.mode == 'train':
                flip = random.random() < 0.5                       # transform_train_cuda's T.RandomHorizontalFlip
                for sp in plan.samples:
                    sp.flip = flip
            yield self.aug(frames, plan), y

    def __len__(self):
        return self.args.steps_per_epoch


class SyntheticVideos:
    """Stand-in for the per-video test datasets: (video [3, T_total, img_dim, img_dim] in [0, 1], label, vname) for
    --synthetic-videos videos of one split.  Video i has 1-4 clips plus 0 to seq_len - 1 leftover frames; its label is
    i modulo a class count that gives every class about three videos per split.  The content is a per-class pattern
    (the same in every split) under seeded per-video noise; `view` = (aug_idx, flip_idx) shifts the crop window and
    flips it, standing in for the reference's FiveCrop / horizontal flip of each test view."""

    def __init__(self, args, split, device, view=(5, 0)):
        self.args, self.split, self.device, self.view = args, split, device, view
        self.n_cls = max(1, min(args.num_class, args.synthetic_videos // 3))

    def __len__(self):
        return self.args.synthetic_videos

    def _pattern(self, label):
        a = self.args
        g = torch.Generator(device=self.device).manual_seed(7919 + label)
        return torch.rand(3, 1, a.img_dim, a.img_dim, device=self.device, generator=g) * 2 - 1

    def __iter__(self):
        a = self.args
        base = 1000003 * (1 if self.split == 'test' else 2)
        aug, flip = self.view
        for i in range(a.synthetic_videos):
            label = i % self.n_cls
            g = torch.Generator(device=self.device).manual_seed(base + 31 * i)
            n_clips = 1 + (i * 5 + (3 if self.split == 'test' else 0)) % 4
            T = n_clips * a.seq_len + (i * 3) % a.seq_len
            noise = torch.rand(3, T, a.img_dim, a.img_dim, device=self.device, generator=g) * 2 - 1
            video = 0.5 + 0.3 * self._pattern(label) + 0.15 * noise
            if aug != 5:
                video = video.roll(shifts=(aug, 2 * aug), dims=(2, 3))
            if flip:
                video = video.flip(3)
            vname = 'synthetic/c%03d/v_c%03d_%s%04d' % (label, label, self.split, i)
            yield video.clamp_(0, 1), label, vname


class SyntheticSourceVideos(SyntheticVideos):
    """--gpu-augment: the same split of seeded videos as uint8 source frames at --source-size, each a per-class pattern
    under per-video noise, augmented on the GPU by one test view (mode 'test', view = (aug_idx, flip_idx)) or the
    retrieval transform, `chunk` videos per launch.  The view's draws come from its own random.Random."""

    def __init__(self, args, split, device, view=(5, 0), mode='test', chunk=8):
        from coclr_b200.clf_augment import ClassifierAugment
        super().__init__(args, split, device, view)
        self.aug = ClassifierAugment(mode, args.seq_len, args.img_dim, num_seq=args.num_seq, view=view)
        self.py = random.Random((1 if split == 'test' else 2) * 1000 + (500 if mode == 'retrieval' else 0)
                                + 10 * view[0] + view[1])
        self.chunk = chunk

    def _pattern(self, label):
        h, w = self.args.source_size
        g = torch.Generator(device=self.device).manual_seed(7919 + label)
        return torch.rand(1, h, w, 3, device=self.device, generator=g) * 2 - 1

    def _source(self, i):
        a = self.args
        h, w = a.source_size
        base = 1000003 * (1 if self.split == 'test' else 2)
        label = i % self.n_cls
        g = torch.Generator(device=self.device).manual_seed(base + 31 * i)
        n_clips = 1 + (i * 5 + (3 if self.split == 'test' else 0)) % 4
        T = n_clips * a.seq_len + (i * 3) % a.seq_len
        noise = torch.rand(T, h, w, 3, device=self.device, generator=g) * 2 - 1
        video = (0.5 + 0.3 * self._pattern(label) + 0.15 * noise).clamp_(0, 1).mul_(255).round_().to(torch.uint8)
        return video, label, 'synthetic/c%03d/v_c%03d_%s%04d' % (label, label, self.split, i)

    def __iter__(self):
        a = self.args
        h, w = a.source_size
        for i0 in range(0, a.synthetic_videos, self.chunk):
            src = [self._source(i) for i in range(i0, min(i0 + self.chunk, a.synthetic_videos))]
            plan = self.aug.plan([(h, w)] * len(src), self.py, lengths=[v.shape[0] for v, _, _ in src])
            videos = self.aug(torch.cat([v for v, _, _ in src]), plan)
            for video, (_, label, vname) in zip(videos, src):
                yield video, label, vname


def test_videos(args, split, device, view=(5, 0), mode='test'):
    if args.gpu_augment:
        return SyntheticSourceVideos(args, split, device, view, mode)
    return SyntheticVideos(args, split, device, view)


def load_test_checkpoint(model, args):
    """:170-185: with --retrieval, a pre-training checkpoint's encoder_q.0. -> backbone. (map_pretrained) loaded
    non-strict; otherwise strict, falling back to the checkpoint entries whose name and shape match."""
    if not os.path.isfile(args.test):
        raise FileNotFoundError("no checkpoint found at '%s'" % args.test)
    print("=> loading testing checkpoint '%s'" % args.test)
    ckpt = torch.load(args.test, map_location='cpu', weights_only=False)
    state_dict = ckpt['state_dict']
    if args.retrieval:
        missing = load_pretrained(model, state_dict)
        print("=> keys not in the checkpoint: %s" % missing)
        return ckpt.get('epoch', 0)
    try:
        model.load_state_dict(state_dict)
    except RuntimeError:
        own = model.state_dict()
        sd = {k: v for k, v in state_dict.items() if k in own and own[k].shape == v.shape}
        missing = model.load_state_dict(sd, strict=False).missing_keys
        print("=> non-strict load; keys not in the checkpoint: %s" % missing)
    return ckpt.get('epoch', 0)


def retrieval_paths(args):
    """Output files of test_retrieval (:607-700) under dirname(--test)/<--dirname or 'feature'>/."""
    d = os.path.join(os.path.dirname(args.test), args.dirname if args.dirname is not None else 'feature')
    out = {'dir': d, 'sim': os.path.join(d, '%s_sim.pth.tar' % args.dataset)}
    for split in ('test', 'train'):
        for what, ext in (('feature', 'pth.tar'), ('label', 'pth.tar'), ('vname', 'pkl')):
            out[split, what] = os.path.join(d, '%s_%s_%s.%s' % (args.dataset, split, what, ext))
    return out


def vname_records(vnames):
    """What the reference pickles: the vname of every batch of one video under default collation, i.e. a list of
    one-element lists."""
    return [[v] for v in vnames]


def test_retrieval(model, args, device):
    paths = retrieval_paths(args)
    feats = {}
    for split in ('test', 'train'):                      # test first, then train, as the reference
        if os.path.exists(paths[split, 'feature']):
            feats[split] = (torch.load(paths[split, 'feature']).to(device), torch.load(paths[split, 'label']).to(device))
            continue
        os.makedirs(paths['dir'], exist_ok=True)
        print('Computing %s set feature ... ' % split)
        res = EV.evaluate(model, test_videos(args, split, device, mode='retrieval'), args.seq_len, args.batch_size,
                          args.num_seq)
        print(res.feature.size())
        torch.save(res.feature.cpu(), paths[split, 'feature'])
        torch.save(res.label.cpu(), paths[split, 'label'])
        with open(paths[split, 'vname'], 'wb') as fp:
            pickle.dump(vname_records(res.vname), fp)
        feats[split] = (res.feature, res.label)
    sim, _, accs = EV.retrieval(feats['test'][0], feats['test'][1], feats['train'][0], feats['train'][1])
    torch.save(sim.cpu(), paths['sim'])
    for k, acc in zip(EV.RETRIEVAL_KS, accs):
        print('%dNN acc = %.4f' % (k, acc))
    return accs


def crop_schedule(args):
    """test_10crop's views (:431-442, :453-512): [(flip_idx, aug_idx, [titles of the summaries written after it])] and
    the mode's title.  The final summary is always written as 'ten' (:515), whatever the mode."""
    if args.ten_crop:
        augs, flips, title = [5, 1, 2, 3, 4], [0, 1], 'ten'
    elif args.five_crop:
        augs, flips, title = [5, 1, 2, 3, 4], [0], 'five'
    else:
        augs, flips, title = [5], [0], 'center'
    views = []
    for flip_idx in flips:
        for aug_idx in augs:
            after = []
            if title == 'ten' and flip_idx == 0 and aug_idx == 5:
                after.append('center')
            if title == 'ten' and flip_idx == 0 and aug_idx == augs[-1]:
                after.append('five')
            views.append((flip_idx, aug_idx, after))
    views[-1][2].append('ten')
    return views, title


def prob_json_path(test, title):
    return os.path.join(os.path.dirname(test), '%s-prob-%s.json' % (os.path.basename(test), title))


def summarize_probability(res, test, title):
    """summarize_probability (:524-545) from the engine's per-video means: {vname: {'mean_prob': [[...C...]]}}."""
    print('Mean: Acc@1: %.4f Acc@5: %.4f' % (res.top1, res.top5))
    prob = res.prob.cpu().tolist()
    stat = {v: {'mean_prob': [p]} for v, p in zip(res.vname, prob)}
    with open(prob_json_path(test, title), 'w') as fp:
        json.dump(stat, fp)
    return res.top1, res.top5


def test_10crop(model, args, device):
    views, title = crop_schedule(args)
    print('Test using %s crop' % {'center': 'center', 'five': '5', 'ten': '10'}[title])
    res, summaries = None, []
    for flip_idx, aug_idx, after in views:
        print('Aug type: %d; flip: %d' % (aug_idx, flip_idx))
        res = EV.evaluate(model, test_videos(args, 'test', device, view=(aug_idx, flip_idx)), args.seq_len,
                          args.batch_size, args.num_seq, previous=res)
        for t in after:
            print('%s-crop result:' % (title if t == 'ten' else t))
            summaries.append((t, summarize_probability(res, args.test, t)))
    return summaries


def run_test(model, args, device):
    load_test_checkpoint(model, args)
    if args.retrieval:
        return test_retrieval(model, args, device)
    if args.center_crop or args.five_crop or args.ten_crop:
        return test_10crop(model, args, device)
    raise NotImplementedError("--test needs --retrieval or one of --center_crop / --five_crop / --ten_crop")


def set_path(args):
    if args.resume:
        exp_path = os.path.dirname(os.path.dirname(args.resume))
    else:
        exp_path = 'log-eval-{a.prefix}/{a.dataset}-{a.img_dim}_sp{a.which_split}_{a.model}_{a.net}_Adam_bs{a.batch_size}_' \
                   'lr{a.lr}_dp{a.dropout}_wd{a.wd}_seq{a.num_seq}_len{a.seq_len}_ds{a.ds}_train-{a.train_what}{pt}'.format(
                       a=args, pt='_pt=%s' % args.pretrain.replace('/', '-') if args.pretrain else '')
    model_path = os.path.join(exp_path, 'model')
    os.makedirs(model_path, exist_ok=True)
    return model_path


def _accumulate(stat, logit, target, loss):
    with torch.no_grad():
        top5 = logit.topk(min(5, logit.shape[1]), dim=1).indices
        hit = top5 == target.unsqueeze(1)
        stat[0] += loss.detach()
        stat[1] += hit[:, 0].float().mean()
        stat[2] += hit.any(1).float().mean()
        stat[3] += 1


def train_one_epoch(loader, model, criterion, optimizer, epoch, args):
    if args.train_what == 'last':
        model.eval()                     # frozen backbone BN (:319-320)
    else:
        model.train()
    if args.final_bn:
        model.final_bn.train()           # :324-325
    stat = torch.zeros(4, device=torch.device('cuda'))   # loss sum, top1 sum, top5 sum, steps
    tic = time.time()
    for idx, (input_seq, target) in enumerate(loader):
        logit, _ = model(input_seq)
        loss = criterion(logit, target)
        _accumulate(stat, logit, target, loss)
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
        if idx % args.print_freq == 0:
            s = stat.tolist()
            n = max(s[3], 1.0)
            dt = (time.time() - tic) / n
            print('Epoch: [%d][%d/%d] loss %.4f acc@1 %.4f acc@5 %.4f  %.1f ms/step  %.0f clips/s'
                  % (epoch, idx, len(loader), s[0] / n, s[1] / n, s[2] / n, dt * 1e3, args.batch_size / dt))
        args.iteration += 1
    s = stat.tolist()
    n = max(s[3], 1.0)
    return s[0] / n, s[1] / n


def validate(loader, model, criterion, epoch, args):
    model.eval()
    stat = torch.zeros(4, device=torch.device('cuda'))
    with torch.no_grad():
        for input_seq, target in loader:
            logit, _ = model(input_seq)
            _accumulate(stat, logit, target, criterion(logit, target))
    s = stat.tolist()
    n = max(s[3], 1.0)
    print('Epoch: [%d]\tLoss: %.4f Acc@1: %.4f Acc@5: %.4f' % (epoch, s[0] / n, s[1] / n, s[2] / n))
    return s[0] / n, s[1] / n


def main(args):
    check_supported(args)
    if args.gpu is not None:
        torch.cuda.set_device(int(args.gpu))
    device = torch.device('cuda')
    torch.manual_seed(0)
    np.random.seed(0)
    random.seed(0)
    args.seed_base = 0
    args.num_class = NUM_CLASS[args.dataset]
    model = build_model(args).to(device)
    if args.gpu_augment:
        if not args.synthetic:
            raise NotImplementedError("--gpu-augment reads the synthetic source frames of --synthetic")
        model.set_input_transform(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])   # :216-220
    if args.test:
        return run_test(model, args, device)
    optimizer = build_optimizer(model, args)
    criterion = nn.CrossEntropyLoss()
    args.iteration = 1
    best_acc = 0.0
    if args.resume:
        ckpt = torch.load(args.resume, map_location='cpu')
        args.start_epoch = ckpt['epoch'] + 1
        args.iteration = ckpt['iteration']
        best_acc = ckpt['best_acc']
        model.load_state_dict(ckpt['state_dict'])
        if not args.reset_lr:
            optimizer.load_state_dict(ckpt['optimizer'])
        print("=> load resumed checkpoint '%s' (epoch %d)" % (args.resume, ckpt['epoch']))
    elif args.pretrain:
        ckpt = torch.load(args.pretrain, map_location='cpu')
        missing = load_pretrained(model, ckpt['state_dict'])
        print("=> loaded pretrained checkpoint '%s' (epoch %s); keys not in it: %s"
              % (args.pretrain, ckpt.get('epoch'), missing))
    else:
        print("=> train from scratch")
    model_path = set_path(args)
    args.seed_base = args.start_epoch * 2
    train_loader = get_data(args, device, 'train')
    val_loader = get_data(args, device, 'val')
    for epoch in range(args.start_epoch, args.epochs):
        np.random.seed(epoch)
        random.seed(epoch)
        adjust_learning_rate(optimizer, epoch, args)
        train_one_epoch(train_loader, model, criterion, optimizer, epoch, args)
        if epoch % args.eval_freq == 0:
            _, val_acc = validate(val_loader, model, criterion, epoch, args)
            is_best = val_acc > best_acc
            best_acc = max(val_acc, best_acc)
            state = {'epoch': epoch, 'state_dict': model.state_dict(), 'best_acc': best_acc,
                     'optimizer': optimizer.state_dict(), 'iteration': args.iteration}
            torch.save(state, os.path.join(model_path, 'epoch%d.pth.tar' % epoch))
            prev = os.path.join(model_path, 'epoch%d.pth.tar' % (epoch - 1))
            if os.path.exists(prev):
                os.remove(prev)
            if is_best:
                torch.save(state, os.path.join(model_path, 'model_best.pth.tar'))
    print('Training from ep %d to ep %d finished' % (args.start_epoch, args.epochs))
    return model


if __name__ == '__main__':
    main(parse_args())
