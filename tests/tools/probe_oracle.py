"""The reference's feature linear probe (eval/feature_linear_probe.py) restated in stock torch, in any dtype and on any
device, over the batches of coclr_b200.probe.plan.  Returns the same ProbeResult fields as coclr_b200.probe.fit.

    res = run(train_feature, train_label, test_feature, test_label, lr, wd, p, final_bn=True, dtype=torch.float64)

The model, loss and optimizer are the reference's modules (BatchNorm1d, Linear, CrossEntropyLoss, optim.SGD); the
batches are the plan's, so a float32 run on the CPU reproduces the reference's trajectory.

reference_shaped=True keeps the features on the host and feeds them the reference's way, for timing: a per-row
Dataset, a DataLoader (the plan's batches as its batch_sampler) with pin_memory, a non-blocking copy per batch and
two .item() synchronisations per step.
"""
import os
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F
import torch.optim as optim
from torch.utils import data

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from coclr_b200.probe import lr_at, summarize, plan, grid, check_inputs  # noqa: E402


class LP(nn.Module):
    def __init__(self, dim, num_class, use_bn):
        super().__init__()
        self.use_bn = use_bn
        if use_bn:
            self.bn = nn.BatchNorm1d(dim)
        self.fc = nn.Linear(dim, num_class, bias=True)

    def forward(self, x):
        return self.fc(self.bn(x) if self.use_bn else x)


class Rows:
    """The reference's per-row feature dataset (class D)."""

    def __init__(self, feature, label):
        self.feature, self.label = feature, label

    def __getitem__(self, i):
        return self.feature[i, :], self.label[i]

    def __len__(self):
        return self.label.size(0)


def _margin(logit):
    top = logit.topk(2, dim=1).values if logit.shape[1] > 1 else torch.cat([logit, logit - float("inf")], 1)
    return (top[:, 0] - top[:, 1]).double()


def run(train_feature, train_label, test_feature, test_label, lr, wd, p, schedule=(60, 80), final_bn=False,
        normalize=False, dtype=torch.float64, device="cpu", reference_shaped=False, record=None):
    """One (lr, wd) config over plan p.  Returns a ProbeResult (host tensors).  record: a dict that receives, per
    epoch and per evaluation, every row's top-1 margin (largest logit minus the runner-up: `train_margin`,
    `val_margin`), so a comparison can tell which hits a small logit error may flip."""
    device = torch.device(device)
    epochs, B = p.order.shape[0], p.batch_size
    xtr, xte = train_feature.to(dtype), test_feature.to(dtype)
    if normalize:
        xtr, xte = F.normalize(xtr), F.normalize(xte)
    ytr, yte = train_label.long(), test_label.long()
    N, Nq, D = xtr.shape[0], xte.shape[0], xtr.shape[1]
    Cn = p.weight.shape[0]
    if not reference_shaped:
        xtr, xte, ytr, yte = xtr.to(device), xte.to(device), ytr.to(device), yte.to(device)
    model = LP(D, Cn, final_bn).to(device, dtype)
    with torch.no_grad():
        model.fc.weight.copy_(p.weight.to(dtype))
        model.fc.bias.copy_(p.bias.to(dtype))
    criterion = nn.CrossEntropyLoss()
    opt = optim.SGD(model.parameters(), lr=lr, weight_decay=wd, momentum=0.9)
    test_chunks = list(torch.arange(Nq).split(B))
    if reference_shaped:
        test_loader = data.DataLoader(Rows(xte, yte), batch_size=B, shuffle=False, pin_memory=True)

    def evaluate(with_prob):
        model.eval()
        losses, hits, probs, margins = [], [], [], []
        with torch.no_grad():
            if reference_shaped:
                batches = ((f.to(device, non_blocking=True), y.to(device, non_blocking=True)) for f, y in test_loader)
            else:
                batches = ((xte[c], yte[c]) for c in test_chunks)
            for f, y in batches:
                logit = model(f)
                loss = criterion(logit, y)
                hit = (logit.argmax(1) == y).sum()
                if record is not None:
                    margins.append(_margin(logit))
                if reference_shaped:
                    loss, hit = loss.item(), hit.item()
                losses.append(loss * y.shape[0])
                hits.append(hit)
                if with_prob:
                    probs.append(F.softmax(logit, dim=-1))
        if record is not None:
            record.setdefault("val_margin", []).append(torch.cat(margins).cpu())
        return losses, hits, (torch.cat(probs) if with_prob else None)

    tl, th, vl, vh = [], [], [], []
    for epoch in range(epochs):
        for g in opt.param_groups:
            g["lr"] = lr_at(lr, epoch, schedule)
        model.train()
        if reference_shaped:
            loader = data.DataLoader(Rows(xtr, ytr), batch_sampler=[b.tolist() for b in p.batches(epoch)],
                                     pin_memory=True)
            batches = ((f.to(device, non_blocking=True), y.to(device, non_blocking=True)) for f, y in loader)
        else:
            batches = ((xtr[b.to(device)], ytr[b.to(device)]) for b in p.batches(epoch))
        el, eh, em = [], [], []
        for f, y in batches:
            logit = model(f)
            loss = criterion(logit, y)
            hit = (logit.detach().argmax(1) == y).sum()
            if record is not None:
                em.append(_margin(logit.detach()))
            if reference_shaped:
                el.append(loss.item() * y.shape[0])
                eh.append(hit.item())
            else:
                el.append(loss.detach() * y.shape[0])
                eh.append(hit)
            opt.zero_grad()
            loss.backward()
            opt.step()
        tl.append(el)
        th.append(eh)
        if record is not None:
            record.setdefault("train_margin", []).append(torch.cat(em).cpu())
        if epoch in p.eval_epochs:
            l, h, _ = evaluate(False)
            vl.append(l)
            vh.append(h)
    l, h, prob = evaluate(True)
    vl.append(l)
    vh.append(h)
    num = lambda rows: [[float(v) for v in r] for r in rows]   # noqa: E731  (one host read at the end)
    state = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    return summarize(lr, wd, num(tl), num(th), num(vl), num(vh), p.eval_epochs, N, Nq, B, prob.cpu(), state)


def fit(train_feature, train_label, test_feature, test_label, lrs, wds, epochs=100, batch_size=1024,
        schedule=(60, 80), eval_freq=5, final_bn=False, normalize=False, seed=0, dtype=torch.float64, device="cpu",
        reference_shaped=False):
    """coclr_b200.probe.fit's signature: every config of the grid, one after the other."""
    N, Nq, D, Cn = check_inputs(train_feature, train_label, test_feature, test_label, epochs, batch_size, eval_freq,
                                final_bn)
    p = plan(N, Nq, D, Cn, [1.0], epochs, batch_size, schedule, eval_freq, seed)
    return [run(train_feature, train_label, test_feature, test_label, lr, wd, p, schedule, final_bn, normalize,
                dtype, device, reference_shaped) for lr, wd in grid(lrs, wds)]
