#!/usr/bin/env python
"""Two-stream merge -- the reference's eval/merge_2stream_prob.py (same flags and printed lines) on the engine
(coclr_b200.evaluate, csrc/evaluate.cu).

  --mode c   fuses the per-video class probabilities of two streams: --prob1 and --prob2 are the -prob-*.json files
             of `eval/main_classifier.py --test CKPT --center_crop | --five_crop | --ten_crop` ({vname: {'mean_prob':
             [[...]]}}) or of `eval/feature_linear_probe.py` ({vname: [[...]]}).  A video's label is the index of its
             action, vname.split('/')[-3] ([-2] for k400), in the class list --class-index.  Prints the top-1
             accuracy of stream 1, of stream 2 and of (p1 + p2) / 2.
  --mode s   sums the retrieval similarities of two streams: --prob1 is the feature directory of stream 1
             ({dataset}_{train,test}_{feature,label}.pth.tar, {dataset}_{train,test}_vname.pkl, as `--test CKPT
             --retrieval` writes them) and --prob2 that of stream 2 ({dataset}-f_...).  The videos are aligned by name
             as the reference does (coclr_b200.evaluate.align_two_stream) and ranked by test1 . train1^T + test2 .
             train2^T of the centred, normalised features.  Prints R@1/5/10/20/50.

The one addition to the command line: --class-index PATH (required with --mode c).  The reference reads the class list
from a fixed path next to its checkout (process_data/data/<dataset>_beegfs/ClassInd.txt), which this repository does
not ship; the file is read the same way (stripped lines, each cut to its last ','-separated field when the first line
has a ',').  A vname missing from --prob2, or an action not in the class list, raises ValueError naming it.
"""
import argparse
import json
import os
import pickle
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from coclr_b200 import evaluate as EV  # noqa: E402


def parse_args(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument('--prob1', default='', type=str)
    parser.add_argument('--prob2', default='', type=str)
    parser.add_argument('--dataset', default='ucf101', type=str)
    parser.add_argument('--mode', default='c', type=str, choices=['c', 's'])
    parser.add_argument('--class-index', default=None, type=str,
                        help='class list of --mode c (the reference\'s ClassInd.txt): one class per line, line order '
                             'is the class index')
    args = parser.parse_args(argv)
    if args.mode == 'c' and not args.class_index:
        parser.error('--mode c needs --class-index')
    return args


def read_class_index(path):
    """The reference's get_action_idx on `path`: read_file's stripped lines, each cut to its last ','-separated field
    when the first line contains a ','."""
    with open(path, 'r') as f:
        action_list = [i.strip() for i in f.readlines()]
    if action_list and ',' in action_list[0]:
        action_list = [i.split(',')[-1] for i in action_list]
    return action_list


def action_of(vname, dataset):
    """The action name in a vname: its third-last '/'-separated field (a UCF101 / HMDB51 vname ends in '/'), its
    second-last for k400."""
    parts = vname.split('/')
    i = -2 if dataset == 'k400' else -3
    if len(parts) < -i:
        raise ValueError("vname %r has no action field at split('/')[%d]" % (vname, i))
    return parts[i]


def prob_row(value, vname, path):
    """One JSON value as a [C] float64 row: {'mean_prob': [[...]]} (main_classifier.py --test) or a plain list
    ([[...]] from feature_linear_probe.py, or [...])."""
    p = np.array(value['mean_prob'] if isinstance(value, dict) else value, dtype=np.float64)
    if p.ndim == 2 and p.shape[0] == 1:
        p = p[0]
    if p.ndim != 1 or p.size == 0:
        raise ValueError("%s: the probabilities of %r are not one row of classes (shape %s)" % (path, vname, p.shape))
    return p


def load_probabilities(args):
    """(prob1 [Nv, C], prob2 [Nv, C], target [Nv]) in the order of --prob1's videos."""
    with open(args.prob1, 'r') as fp:
        prob_dict1 = json.load(fp)
    with open(args.prob2, 'r') as fp:
        prob_dict2 = json.load(fp)
    if not prob_dict1:
        raise ValueError("%s holds no videos" % args.prob1)
    action_list = read_class_index(args.class_index)
    action_to_idx = dict(zip(action_list, range(len(action_list))))   # a repeated name keeps its last index
    rows1, rows2, target = [], [], []
    for k in prob_dict1:
        if k not in prob_dict2:
            raise ValueError("video %r of %s is not in %s" % (k, args.prob1, args.prob2))
        action = action_of(k, args.dataset)
        if action not in action_to_idx:
            raise ValueError("action %r of video %r is not in the class list %s" % (action, k, args.class_index))
        rows1.append(prob_row(prob_dict1[k], k, args.prob1))
        rows2.append(prob_row(prob_dict2[k], k, args.prob2))
        target.append(action_to_idx[action])
    widths = {len(r) for r in rows1 + rows2}
    if len(widths) != 1:
        raise ValueError("the probability rows have different numbers of classes: %s" % sorted(widths))
    return np.stack(rows1), np.stack(rows2), np.array(target, dtype=np.int64)


def merge_prob(args, device):
    p1, p2, target = load_probabilities(args)
    _, (a1, a2, af) = EV.merge_probabilities(torch.from_numpy(p1).to(device), torch.from_numpy(p2).to(device),
                                             torch.from_numpy(target).to(device))
    print('merged accuracy: %.6f + %.6f => %.6f' % (a1, a2, af))
    return a1, a2, af


def load_stream(directory, name, device, labels):
    """{split: (feature, label or None, vname list)} of one stream's retrieval files."""
    out = {}
    for split in ('train', 'test'):
        def path(what, ext):
            return os.path.join(directory, '%s_%s_%s.%s' % (name, split, what, ext))
        feat = torch.load(path('feature', 'pth.tar'), map_location=device)
        label = torch.load(path('label', 'pth.tar'), map_location=device) if labels else None
        with open(path('vname', 'pkl'), 'rb') as fp:
            vname = pickle.load(fp)
        out[split] = (feat, label, vname)
    return out


def merge_sim(args, device):
    s1 = load_stream(args.prob1, args.dataset, device, labels=True)     # the labels are stream 1's, as in the reference
    s2 = load_stream(args.prob2, '%s-f' % args.dataset, device, labels=False)
    idx = EV.align_two_stream(s1['train'][2], s1['test'][2], s2['train'][2], s2['test'][2])
    tr1, te1, tr2, te2 = (i.to(device) for i in idx)
    _, _, accs = EV.two_stream_retrieval(s1['test'][0][te1], s1['train'][0][tr1], s2['test'][0][te2],
                                         s2['train'][0][tr2], s1['test'][1][te1], s1['train'][1][tr1])
    for k, acc in zip(EV.RETRIEVAL_KS, accs):
        # the reference prints a float32 mean (.float().mean().item()): hits / Nq rounded to float32
        print('%dNN acc = %.4f' % (k, np.float32(acc)))
    return accs


def main(argv=None):
    args = parse_args(argv)
    if not torch.cuda.is_available():
        raise RuntimeError("merge_2stream_prob.py runs on a CUDA device (sm_90a); there is no CPU path")
    device = torch.device('cuda')
    if args.mode == 'c':
        print('Merge classification probability')
        return merge_prob(args, device)
    print('Merge similarity')
    return merge_sim(args, device)


if __name__ == '__main__':
    main()
