"""Linear probe on extracted features, on the engine: what the reference's eval/feature_linear_probe.py trains, for a
whole grid of (lr, wd) in one run.

    results = fit(train_feature, train_label, test_feature, test_label, lrs=[0.1, 1.0], wds=[1e-4, 1e-3],
                  final_bn=True)
    results[i]            config i of the grid, lr-major: (lrs[0], wds[0]), (lrs[0], wds[1]), ...
    results[i].best_acc   best validation accuracy (the reference's `>=` rule: the last epoch reaching it)
    results[i].prob       [Nq, C] softmax probabilities of the final model (what the reference saves)
    results[i].state_dict()   the reference LP's keys: bn.* (with final_bn), fc.weight, fc.bias

The model is the reference's `LP`: an optional BatchNorm1d(D) (weight 1, bias 0, momentum 0.1, eps 1e-5) and a
Linear(D, C) with weights normal(0, 0.01) and a zero bias, trained by SGD (momentum 0.9, weight decay coupled and
applied to every parameter) on the batch-mean cross-entropy, with lr = base * 0.1 ** (milestones <= epoch).

Every config of a grid consumes torch's RNG as a separate reference run would: `plan` seeds the default generator,
builds the Linear (kaiming-uniform weight and uniform bias draws, then normal_) and iterates DataLoaders in the
reference's order -- the shuffled train loader every epoch, the test loader at every evaluation and once more for the
final pass, each iteration drawing a base seed.  So all configs share the initial weights and the batch order (and,
with final_bn, the BatchNorm statistics), and one device run (csrc/probe.cu) trains them together: config s of a
sweep gives the same bits as a run of that (lr, wd) alone.

Accuracies and losses are formed from per-batch sums exactly as the reference's AverageMeter forms them (a float32
per-batch mean times the batch size, summed and divided in double), so the best-epoch rule sees the same values.
"""
import ctypes as C
import math
from collections import OrderedDict
from dataclasses import dataclass, field

import numpy as np
import torch
import torch.nn as nn
from torch.utils import data

from coclr_b200 import lib as L

BN_MOMENTUM = 0.1
BN_EPS = 1e-5


@dataclass
class Plan:
    """What a reference run draws from torch's RNG, and its learning-rate table."""
    weight: torch.Tensor     # [C, D] float32: fc.weight after normal_(0, 0.01)
    bias: torch.Tensor       # [C] float32 zeros
    order: torch.Tensor      # [epochs, N] int64: each epoch's train rows in batch order
    lr: torch.Tensor         # [epochs, S] float64: lr of each config at each epoch
    batch_size: int
    eval_epochs: list        # epochs after which the test set is evaluated

    def batches(self, epoch):
        """The index batches of one epoch (the last may be partial)."""
        return list(self.order[epoch].split(self.batch_size))


def lr_at(base, epoch, schedule):
    """The reference's adjust_learning_rate: lr = base * 0.1 for every milestone <= epoch, recomputed each epoch."""
    lr = base
    for milestone in schedule:
        lr *= 0.1 if epoch >= milestone else 1.
    return lr


def plan(N, Nq, D, C, lrs=(1.0,), epochs=100, batch_size=1024, schedule=(60, 80), eval_freq=5, seed=0):
    """The initial LP parameters, per-epoch batch order and lr table of a reference run (no GPU needed).  torch's
    RNG state is restored afterwards."""
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        fc = nn.Linear(D, C, bias=True)
        fc.weight.data.normal_(mean=0.0, std=0.01)
        fc.bias.data.zero_()
        train_loader = data.DataLoader(range(N), batch_size=batch_size, shuffle=True, drop_last=False)
        test_loader = data.DataLoader(range(Nq), batch_size=batch_size, shuffle=False, drop_last=False)
        order, eval_epochs = [], []
        for epoch in range(epochs):
            order.append(torch.cat([b for b in train_loader]))
            if epoch % eval_freq == 0:
                eval_epochs.append(epoch)
                for _ in test_loader:
                    pass
        for _ in test_loader:   # the final pass with save_prob
            pass
    lr = torch.tensor([[lr_at(b, e, schedule) for b in lrs] for e in range(epochs)], dtype=torch.float64)
    return Plan(weight=fc.weight.data.clone(), bias=fc.bias.data.clone(), order=torch.stack(order), lr=lr,
                batch_size=batch_size, eval_epochs=eval_epochs)


@dataclass
class ProbeResult:
    """One (lr, wd) config of a run."""
    lr: float
    wd: float
    train_loss: list         # per epoch (the printed `train: Epoch[e] loss`)
    train_acc: list
    train_hits: list         # per epoch: correctly classified train rows
    eval_epochs: list
    val_loss: list           # per evaluation
    val_acc: list
    val_hits: list
    best_acc: float
    best_epoch: int
    final_loss: float        # the final pass: the final model (see eval/feature_linear_probe.py)
    final_acc: float
    final_hits: int
    prob: torch.Tensor       # [Nq, C] softmax of the final model
    state: OrderedDict = field(repr=False, default=None)

    def state_dict(self):
        return OrderedDict((k, v.clone()) for k, v in self.state.items())


def _meter(values, sizes):
    """AverageMeter.avg over batches: sum(val * n) / sum(n) in double, val being the batch's float32 value."""
    total, count = 0.0, 0
    for v, n in zip(values, sizes):
        total += float(v) * n
        count += n
    return total / count


def _batch_loss(loss_sum, n):
    return np.float32(loss_sum / n)


def _batch_top1(hits, n):
    """calc_topk_accuracy: correct.float().sum() * (1 / batch_size) in float32."""
    return np.float32(np.float32(hits) * np.float32(1 / n))


def chunk_sizes(n, batch_size):
    return [min(batch_size, n - i) for i in range(0, n, batch_size)]


def summarize(lr, wd, train_loss, train_hits, val_loss, val_hits, eval_epochs, N, Nq, batch_size, prob, state):
    """A ProbeResult from per-batch sums: train_* [epochs, steps] (loss sum and hits of each training step), val_*
    [evaluations + 1, chunks] (of each test batch; the final pass last)."""
    ts, vs = chunk_sizes(N, batch_size), chunk_sizes(Nq, batch_size)

    def curve(loss, hits, sizes):
        lo = _meter([_batch_loss(l, n) for l, n in zip(loss, sizes)], sizes)
        ac = _meter([_batch_top1(h, n) for h, n in zip(hits, sizes)], sizes)
        return lo, ac, int(sum(int(h) for h in hits))

    tr = [curve(train_loss[e], train_hits[e], ts) for e in range(len(train_loss))]
    va = [curve(val_loss[v], val_hits[v], vs) for v in range(len(val_loss))]
    best_acc, best_epoch = 0.0, 0
    for epoch, (_, acc, _) in zip(eval_epochs, va):
        if acc >= best_acc:
            best_acc, best_epoch = acc, epoch
    fin = va[len(eval_epochs)]
    return ProbeResult(lr=lr, wd=wd, train_loss=[t[0] for t in tr], train_acc=[t[1] for t in tr],
                       train_hits=[t[2] for t in tr], eval_epochs=list(eval_epochs),
                       val_loss=[v[0] for v in va[:len(eval_epochs)]], val_acc=[v[1] for v in va[:len(eval_epochs)]],
                       val_hits=[v[2] for v in va[:len(eval_epochs)]], best_acc=best_acc, best_epoch=best_epoch,
                       final_loss=fin[0], final_acc=fin[1], final_hits=fin[2], prob=prob, state=state)


def grid(lrs, wds):
    """The configs of a sweep, lr-major."""
    return [(float(lr), float(wd)) for lr in lrs for wd in wds]


def check_inputs(train_feature, train_label, test_feature, test_label, epochs, batch_size, eval_freq, final_bn):
    """Validates a run on the host (before anything is launched); returns (N, Nq, D, C)."""
    if train_feature.dim() != 2 or test_feature.dim() != 2 or train_feature.shape[1] != test_feature.shape[1]:
        raise ValueError("features are [N, D] and [Nq, D], got %s and %s"
                         % (list(train_feature.shape), list(test_feature.shape)))
    N, D = train_feature.shape
    Nq = test_feature.shape[0]
    if N < 1 or Nq < 1 or D < 1:
        raise ValueError("empty features: train %s, test %s" % (list(train_feature.shape), list(test_feature.shape)))
    if train_label.shape != (N,) or test_label.shape != (Nq,):
        raise ValueError("labels must be [N] and [Nq], got %s and %s" % (list(train_label.shape),
                                                                         list(test_label.shape)))
    if train_label.is_floating_point() or test_label.is_floating_point():
        raise ValueError("labels must be integers")
    if epochs < 1 or batch_size < 1 or eval_freq < 1:
        raise ValueError("epochs, batch_size and eval_freq must be >= 1")
    tmin, C = int(train_label.min()), int(train_label.max()) + 1
    if tmin < 0:
        raise ValueError("train label %d is negative" % tmin)
    qmin, qmax = int(test_label.min()), int(test_label.max())
    if qmin < 0 or qmax >= C:
        raise ValueError("test label %d is outside the %d classes of the train labels (num_class = train max + 1)"
                         % (qmin if qmin < 0 else qmax, C))
    if final_bn and N % batch_size == 1:
        raise ValueError("the last training batch has one row (N = %d, batch_size = %d): BatchNorm1d cannot train on "
                         "it (the reference raises there too); change batch_size" % (N, batch_size))
    return N, Nq, D, C


def _padded(x, D4, device):
    x = x.to(device, torch.float32).contiguous()
    if x.shape[1] == D4 and x.data_ptr() % 16 == 0:
        return x
    out = torch.zeros(x.shape[0], D4, dtype=torch.float32, device=device)
    out[:, :x.shape[1]].copy_(x)
    return out


def _l2normalize(x):
    """F.normalize(x, dim=1): x / max(||x||, 1e-12) (coclr_l2norm_fwd)."""
    y = torch.empty_like(x)
    L.check(L.load().coclr_l2norm_fwd(L.dptr(x), None, L.dptr(y), None, x.shape[0], x.shape[1], L.stream_ptr()),
            "coclr_l2norm_fwd")
    return y


def fit(train_feature, train_label, test_feature, test_label, lrs, wds, epochs=100, batch_size=1024,
        schedule=(60, 80), eval_freq=5, final_bn=False, normalize=False, seed=0):
    """Trains the reference's LP for every (lr, wd) of the grid lrs x wds (lr-major) in one device run on the
    current CUDA device.  Features may be on the host or the device.  Returns one ProbeResult per config."""
    configs = grid(lrs, wds)
    if not configs:
        raise ValueError("lrs and wds must each hold at least one value")
    N, Nq, D, Cn = check_inputs(train_feature, train_label, test_feature, test_label, epochs, batch_size, eval_freq,
                                final_bn)
    S = len(configs)
    p = plan(N, Nq, D, Cn, [c[0] for c in configs], epochs, batch_size, schedule, eval_freq, seed)
    lib = L.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    f32 = dict(dtype=torch.float32, device=dev)
    D4 = (D + 3) // 4 * 4
    xtr = train_feature.to(dev, torch.float32).contiguous()
    xte = test_feature.to(dev, torch.float32).contiguous()
    if normalize:
        xtr, xte = _l2normalize(xtr), _l2normalize(xte)
    xtr, xte = _padded(xtr, D4, dev), _padded(xte, D4, dev)
    ytr = train_label.to(dev, torch.long).contiguous()
    yte = test_label.to(dev, torch.long).contiguous()
    order = p.order.to(dev, torch.int32).contiguous()
    lr = p.lr.to(torch.float32).to(dev).contiguous()
    wd = torch.tensor([c[1] for c in configs], dtype=torch.float32).to(dev)
    W = torch.zeros(S, Cn, D4, **f32)
    W[:, :, :D].copy_(p.weight.to(dev).expand(S, Cn, D))
    bias = p.bias.to(dev).repeat(S, 1).contiguous()
    gamma = torch.ones(S, D4, **f32) if final_bn else None
    beta = torch.zeros(S, D4, **f32) if final_bn else None
    rmean = torch.zeros(D4, **f32) if final_bn else None
    rvar = torch.ones(D4, **f32) if final_bn else None
    bufs = [torch.zeros_like(t) if t is not None else None for t in (W, bias, gamma, beta)]
    steps, chunks, V = math.ceil(N / batch_size), math.ceil(Nq / batch_size), len(p.eval_epochs) + 1
    train_loss = torch.zeros(epochs * steps, S, dtype=torch.float64, device=dev)
    train_hits = torch.zeros(epochs * steps, S, dtype=torch.int32, device=dev)
    val_loss = torch.zeros(V * chunks, S, dtype=torch.float64, device=dev)
    val_hits = torch.zeros(V * chunks, S, dtype=torch.int32, device=dev)
    prob = torch.empty(S, Nq, Cn, **f32)
    a = L.Probe(N=N, Nq=Nq, D=D4, C=Cn, S=S, epochs=epochs, batch=batch_size, eval_freq=eval_freq,
                final_bn=int(final_bn), momentum=BN_MOMENTUM, eps=BN_EPS,
                train=L.dptr(xtr), train_label=L.dptr(ytr), test=L.dptr(xte), test_label=L.dptr(yte),
                order=L.dptr(order), lr=L.dptr(lr), wd=L.dptr(wd), W=L.dptr(W), bias=L.dptr(bias),
                gamma=L.dptr(gamma), beta=L.dptr(beta), W_buf=L.dptr(bufs[0]), bias_buf=L.dptr(bufs[1]),
                gamma_buf=L.dptr(bufs[2]), beta_buf=L.dptr(bufs[3]), running_mean=L.dptr(rmean),
                running_var=L.dptr(rvar), train_loss=L.dptr(train_loss), train_hits=L.dptr(train_hits),
                val_loss=L.dptr(val_loss), val_hits=L.dptr(val_hits), prob=L.dptr(prob))
    nwork = lib.coclr_probe_work_floats(C.byref(a))
    if nwork < 0:
        raise L.CoclrError("coclr_probe_work_floats rejected the shape")
    work = torch.empty(max(nwork, 4), **f32)
    a.work = L.dptr(work)
    L.check(lib.coclr_probe_run(C.byref(a), L.stream_ptr()), "coclr_probe_run")
    tl = train_loss.view(epochs, steps, S).cpu().numpy()
    th = train_hits.view(epochs, steps, S).cpu().numpy()
    vl = val_loss.view(V, chunks, S).cpu().numpy()
    vh = val_hits.view(V, chunks, S).cpu().numpy()
    prob, W, bias = prob.cpu(), W[:, :, :D].cpu(), bias.cpu()
    if final_bn:
        gamma, beta, rmean, rvar = gamma[:, :D].cpu(), beta[:, :D].cpu(), rmean[:D].cpu(), rvar[:D].cpu()
    out = []
    for s, (l, w) in enumerate(configs):
        state = OrderedDict()
        if final_bn:
            state["bn.weight"], state["bn.bias"] = gamma[s].clone(), beta[s].clone()
            state["bn.running_mean"], state["bn.running_var"] = rmean.clone(), rvar.clone()
            state["bn.num_batches_tracked"] = torch.tensor(epochs * steps, dtype=torch.long)
        state["fc.weight"], state["fc.bias"] = W[s].clone(), bias[s].clone()
        out.append(summarize(l, w, tl[:, :, s], th[:, :, s], vl[:, :, s], vh[:, :, s], p.eval_epochs, N, Nq,
                             batch_size, prob[s].clone(), state))
    return out
