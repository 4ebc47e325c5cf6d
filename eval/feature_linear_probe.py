#!/usr/bin/env python
"""Linear probe on extracted features -- the reference's eval/feature_linear_probe.py (same flags, defaults, input
files, printed lines and probability JSON) trained on the engine (coclr_b200.probe, csrc/probe.cu).

Reads {dataset}_{train,test}_{feature,label}.pth.tar and {dataset}_test_vname.pkl from dirname(--test)/--dirname, as
written by `eval/main_classifier.py --test CKPT --retrieval` (host tensors) or by the reference (CUDA tensors; loaded
with map_location).  Missing features print `feature path does not exist` and exit with status 0, as the reference does.

The one change to the command line: --lr and --wd take one or more values.
  * one of each: the reference's run.  It prints the reference's lines and writes
    {basename(test)}-lp-{dataset}-prob.json = {vname: [[p_0 .. p_C-1]]}, the final model's softmax (the reference's
    best_model aliases the live parameters, so the probabilities it saves are the final model's, printed under the
    best epoch's number).
  * a grid: every (lr, wd) of lrs x wds trains in one device run over the same batches (each config gives the same
    bits as a run of it alone).  It writes {basename}-lp-{dataset}-lr{lr}-wd{wd}-prob.json per config and
    {basename}-lp-{dataset}-sweep.json (best acc, best epoch, final acc and the eval curve of each config), and prints
    a table.
--verbose only drove the reference's tqdm bars; it is accepted and ignored.
"""
import argparse
import json
import os
import pickle
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from coclr_b200 import probe as P  # noqa: E402


def parse_args(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument('--test', default='', type=str)
    parser.add_argument('--dataset', default='ucf101', type=str)
    parser.add_argument('--dirname', default='feature', type=str)

    parser.add_argument('--batch_size', default=1024, type=int)
    parser.add_argument('--lr', default=[1.0], type=float, nargs='+', help='one value, or several for a sweep')
    parser.add_argument('--wd', default=[1e-3], type=float, nargs='+', help='one value, or several for a sweep')
    parser.add_argument('--epochs', default=100, type=int)
    parser.add_argument('--eval_freq', default=5, type=int)
    parser.add_argument('--verbose', default=0, type=int)
    parser.add_argument('--schedule', default=[60, 80], nargs='*', type=int,
                        help='learning rate schedule (when to drop lr by 10x)')
    parser.add_argument('--normalize', action='store_true', help='normalize feature')
    parser.add_argument('--final_bn', action='store_true', help='final bn')
    return parser.parse_args(argv)


def feature_dir(args):
    return os.path.join(os.path.dirname(args.test), args.dirname)


def input_paths(args):
    d = feature_dir(args)
    out = {'%s_%s' % (split, what): os.path.join(d, '%s_%s_%s.pth.tar' % (args.dataset, split, what))
           for split in ('train', 'test') for what in ('feature', 'label')}
    out['test_vname'] = os.path.join(d, '%s_test_vname.pkl' % args.dataset)
    return out


def is_sweep(args):
    return len(args.lr) * len(args.wd) > 1


def prob_path(args, lr=None, wd=None):
    """The reference's -lp-{dataset}-prob.json; in a sweep, one per config with its lr and wd in the name."""
    base = '%s-lp-%s' % (os.path.basename(args.test), args.dataset)
    if is_sweep(args):
        base += '-lr%g-wd%g' % (lr, wd)
    return os.path.join(feature_dir(args), base + '-prob.json')


def sweep_path(args):
    return os.path.join(feature_dir(args), '%s-lp-%s-sweep.json' % (os.path.basename(args.test), args.dataset))


def unwrap_vnames(records):
    """The pickled test vnames as the reference's DataLoader hands them out: a record [v] (what --retrieval writes,
    one per video) collates to v."""
    return [r[0] if isinstance(r, (list, tuple)) and len(r) == 1 else r for r in records]


def load_features(args):
    """(train_feature, train_label, test_feature, test_label, test_vnames) on the host, or None when the train
    features are missing."""
    p = input_paths(args)
    if not os.path.exists(p['train_feature']):
        return None
    load = lambda k: torch.load(p[k], map_location='cpu')   # noqa: E731
    with open(p['test_vname'], 'rb') as fp:
        vnames = unwrap_vnames(pickle.load(fp))
    return load('train_feature'), load('train_label'), load('test_feature'), load('test_label'), vnames


def report_lines(res, args, path):
    """The lines the reference prints for one run, after its preamble."""
    lines = []
    evals = dict(zip(res.eval_epochs, zip(res.val_loss, res.val_acc)))
    best = 0.0
    for epoch in range(len(res.train_loss)):
        lines.append('train: Epoch[{}] loss {:.4f} acc {:.4f}'.format(epoch, res.train_loss[epoch], res.train_acc[epoch]))
        if epoch in evals:
            loss, acc = evals[epoch]
            lines.append('eval[{}] loss {:.4f} acc {:.4f}'.format(epoch, loss, acc))
            if acc >= best:
                best = acc
                lines.append('Best acc: %.4f' % acc)
    lines.append('Final best acc: %.4f' % res.best_acc)
    lines.append('Save probability ... ')
    lines.append('eval[{}] loss {:.4f} acc {:.4f}'.format(res.best_epoch, res.final_loss, res.final_acc))
    lines.append('prob saved to %s' % path)
    return lines


def preamble(args):
    return (['Using normalized feature'] if args.normalize else []) + \
        (['Use final BN layer in network'] if args.final_bn else [])


def prob_json(res, vnames):
    """{vname: [[p_0 .. p_C-1]]} -- the reference's stats[v] = p.tolist() of a [1, C] row."""
    return {v: [p] for v, p in zip(vnames, res.prob.tolist())}


def write_json(path, obj):
    with open(path, 'w') as fp:
        json.dump(obj, fp)


def main(argv=None):
    args = parse_args(argv)
    loaded = load_features(args)
    if loaded is None:
        print('feature path does not exist')
        sys.exit(0)
    train_feature, train_label, test_feature, test_label, vnames = loaded
    for line in preamble(args):
        print(line)
    results = P.fit(train_feature, train_label, test_feature, test_label, args.lr, args.wd, epochs=args.epochs,
                    batch_size=args.batch_size, schedule=args.schedule, eval_freq=args.eval_freq,
                    final_bn=args.final_bn, normalize=args.normalize)
    if not is_sweep(args):
        res = results[0]
        path = prob_path(args)
        write_json(path, prob_json(res, vnames))
        for line in report_lines(res, args, path):
            print(line)
        return results
    summary = []
    print('%-8s %-8s %-9s %-10s %-9s' % ('lr', 'wd', 'best_acc', 'best_epoch', 'final_acc'))
    for res in results:
        path = prob_path(args, res.lr, res.wd)
        write_json(path, prob_json(res, vnames))
        summary.append(dict(lr=res.lr, wd=res.wd, best_acc=res.best_acc, best_epoch=res.best_epoch,
                            final_acc=res.final_acc, eval_epochs=res.eval_epochs, eval_acc=res.val_acc,
                            eval_loss=res.val_loss, prob=os.path.basename(path)))
        print('%-8g %-8g %-9.4f %-10d %-9.4f' % (res.lr, res.wd, res.best_acc, res.best_epoch, res.final_acc))
    write_json(sweep_path(args), summary)
    print('sweep saved to %s' % sweep_path(args))
    return results


if __name__ == '__main__':
    main()
