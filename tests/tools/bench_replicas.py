"""DataParallel replicas and SGD on one GPU: clips/s, ms/step and peak device memory of LinearClassifier training steps
(forward, backward, optimizer) at the README's shapes -- `ft` + Adam and `last` + SGD, each at R = 2 x batch and, for
context, R = 1 at batch and at 2 x batch -- and coclr_sgd_step over the backbone and head spans against torch.optim.SGD
over the reference's per-tensor param groups (kernel time and GB/s at 20 B per parameter: p, g, buf read; p, buf
written).  Prints one JSON line with the card's name, power limit and SM clock, read in the same run.

  python tests/tools/bench_replicas.py [--net s3d] [--batch 32] [--seq 32] [--img 128] [--steps 20] [--warmup 5]
"""
import argparse
import gc
import json
import os
import sys
import types

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "eval"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_classifier import gpu_info, time_steps  # noqa: E402


def train_run(args, train_what, optim, replicas, batch):
    """ms/step, clips/s and peak memory of one configuration; 'oom' when it does not fit."""
    import main_classifier as MC
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    cfg = types.SimpleNamespace(train_what=train_what, lr=0.1 if optim == "sgd" else 1e-3, wd=1e-3, net=args.net,
                                num_class=args.ncls, dropout=0.9, precision="parity", optim=optim, replicas=replicas)
    res = dict(train_what=train_what, optim=optim, replicas=replicas, batch=batch)
    try:
        model = MC.build_model(cfg).cuda()
        opt = MC.build_optimizer(model, cfg)
        if train_what == "last":
            model.eval()
            model.final_bn.train()
        else:
            model.train()
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randn(batch, 3, args.seq, args.img, args.img, device="cuda", generator=g)
        y = torch.randint(0, args.ncls, (batch,), device="cuda", generator=g)

        def step():
            logit, _ = model(x)
            loss = F.cross_entropy(logit, y)
            opt.zero_grad()
            loss.backward()
            opt.step()
        dt = time_steps(step, args.steps, args.warmup)
        res.update(ms_per_step=dt * 1e3, clips_per_s=batch / dt,
                   peak_mem_GiB=torch.cuda.max_memory_allocated() / 2 ** 30)
    except torch.OutOfMemoryError as e:
        res.update(oom=str(e).split("\n")[0][:200], peak_mem_GiB=torch.cuda.max_memory_allocated() / 2 ** 30)
    finally:
        model = opt = x = y = None
        gc.collect()
        torch.cuda.empty_cache()
    return res


def event_time(fn, iters, warmup=5):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e-3


def sgd_kernel(args):
    """SpanSGD (one coclr_sgd_step per span) against torch.optim.SGD (default foreach path) over per-tensor groups:
    the ft layout, backbone at lr / 10 and head at lr."""
    from model.classifier import LinearClassifier
    from coclr_b200 import moco
    model = LinearClassifier(num_class=args.ncls, network=args.net, dropout=0.9).cuda()
    spans = model.flat_spans()
    for _, gr in spans.values():
        gr.normal_(0, 1e-3)
    opt = moco.SpanSGD([dict(name="backbone", params=spans["backbone"][0], grad=spans["backbone"][1], lr=0.01),
                        dict(name="head", params=spans["head"][0], grad=spans["head"][1], lr=0.1)], weight_decay=1e-3)
    out = {}
    for name, (p, _) in spans.items():
        one = moco.SpanSGD([dict(name=name, params=p, grad=spans[name][1], lr=0.01)], weight_decay=1e-3)
        t = event_time(one.step, 200)
        out[name] = dict(params=p.numel(), us=t * 1e6, GBps=20 * p.numel() / t / 1e9)
    t_span = event_time(opt.step, 200)
    named = dict(model.named_parameters())
    ref = {k: p.detach().clone().requires_grad_(True) for k, p in named.items()}
    for k, p in ref.items():
        p.grad = torch.randn_like(p) * 1e-3
    groups = [{"params": [p], "lr": 0.01 if k.startswith("backbone.") else 0.1} for k, p in ref.items()]
    ref_opt = torch.optim.SGD(groups, lr=0.1, momentum=0.9, weight_decay=1e-3)
    t_ref = event_time(ref_opt.step, 200)
    n = sum(p.numel() for p, _ in spans.values())
    n_ref = sum(p.numel() for p in ref.values())
    out["both_spans"] = dict(params=n, us=t_span * 1e6, GBps=20 * n / t_span / 1e9)
    out["torch_sgd_per_tensor_groups"] = dict(params=n_ref, tensors=len(ref), us=t_ref * 1e6,
                                              GBps=20 * n_ref / t_ref / 1e9)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--net", default="s3d")
    ap.add_argument("--ncls", type=int, default=101)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seq", type=int, default=32)
    ap.add_argument("--img", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    torch.backends.cudnn.benchmark = False
    info = gpu_info()
    b = args.batch
    runs = []
    for train_what, optim in (("ft", "adam"), ("last", "sgd")):
        for replicas, batch in ((2, 2 * b), (1, b), (1, 2 * b)):
            runs.append(train_run(args, train_what, optim, replicas, batch))
            print(json.dumps(runs[-1]), file=sys.stderr)
    res = dict(gpu=info, shape=dict(net=args.net, seq=args.seq, img=args.img, ncls=args.ncls),
               train=runs, sgd_step=sgd_kernel(args), gpu_after=gpu_info())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
