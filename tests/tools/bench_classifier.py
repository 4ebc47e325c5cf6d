"""Clips/s of one LinearClassifier training step (forward, backward, Adam) on one GPU: the engine's LinearClassifier
against stock PyTorch (tests/tools/classifier_oracle.py on cuDNN, fp32 and TF32, torch.optim.Adam), for
`--train_what ft` (backbone at lr / 10, dropout head) and `last` (frozen eval-mode backbone, l2norm + final BN head).
Prints one JSON line with the card name, power limit and SM clock next to the numbers.

  python tests/tools/bench_classifier.py [--net s3d] [--batch 32] [--seq 32] [--img 128] [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "eval"))


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                         stdout=subprocess.PIPE, text=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def time_steps(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps


def engine_step(args, train_what, x, y):
    import types
    import main_classifier as MC
    cfg = types.SimpleNamespace(train_what=train_what, lr=1e-3, wd=1e-3, net=args.net, num_class=args.ncls, dropout=0.9,
                                precision="parity")
    model = MC.build_model(cfg).cuda()
    opt = MC.build_optimizer(model, cfg)
    if train_what == "last":
        model.eval()
        model.final_bn.train()
    else:
        model.train()

    def step():
        logit, _ = model(x)
        loss = F.cross_entropy(logit, y)
        opt.zero_grad()
        loss.backward()
        opt.step()
    return step


def torch_step(args, train_what, x, y, tf32):
    import classifier_oracle as O
    torch.backends.cudnn.benchmark = True            # as the reference's classifier script sets (:267)
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cuda.matmul.allow_tf32 = tf32
    last = train_what == "last"
    sd = {k: v.cuda() for k, v in O.classifier_state(args.net, args.ncls, not last, last).items()}
    train = [k for k in sd if (k.endswith(".weight") or k.endswith(".bias")) and not (last and k.startswith("backbone."))]
    for k in train:
        sd[k].requires_grad_(True)
    groups = [{"params": [sd[k]], "lr": 1e-4 if k.startswith("backbone.") else 1e-3} for k in train]
    opt = torch.optim.Adam(groups, lr=1e-3, weight_decay=1e-3)
    fs = 2048 if args.net == "r50" else 1024

    def step():
        mask = None if last else (torch.rand(x.shape[0], fs, device="cuda") >= 0.9)
        if last:
            with torch.no_grad():
                f = O.s3d(sd, "backbone.", x, False) if args.net != "r50" else O.r2d3d50(sd, "backbone.", x, False)
            logit, _ = _head_only(O, sd, f)
        else:
            logit, _ = O.classifier_forward(sd, x, True, False, False, mask, 0.9)
        loss = F.cross_entropy(logit, y)
        opt.zero_grad()
        loss.backward()
        opt.step()
    return step


def _head_only(O, sd, fmap):
    B = fmap.shape[0]
    f = F.normalize(F.adaptive_avg_pool3d(fmap, (1, 1, 1)).view(B, -1), p=2, dim=1)
    h = O._bn(sd, "final_bn", f, True)
    return F.linear(h, sd["final_fc.0.weight"], sd["final_fc.0.bias"]), f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--net", default="s3d")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seq", type=int, default=32)
    ap.add_argument("--img", type=int, default=128)
    ap.add_argument("--ncls", type=int, default=101)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_classifier.py measures on a CUDA device; none is available")
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(args.batch, 3, args.seq, args.img, args.img, device="cuda", generator=g)
    y = torch.randint(0, args.ncls, (args.batch,), device="cuda", generator=g)
    res = {"gpu": gpu_info(), "net": args.net, "batch": args.batch, "seq_len": args.seq, "img_dim": args.img,
           "num_class": args.ncls, "steps": args.steps, "warmup": args.warmup}
    for tw in ("ft", "last"):
        for impl in ("engine", "torch_fp32", "torch_tf32"):
            if impl == "engine":
                step = engine_step(args, tw, x, y)
            else:
                step = torch_step(args, tw, x, y, impl == "torch_tf32")
            dt = time_steps(step, args.steps, args.warmup)
            res["%s/%s/ms_per_step" % (tw, impl)] = round(dt * 1e3, 3)
            res["%s/%s/clips_per_s" % (tw, impl)] = round(args.batch / dt, 1)
            del step
            torch.cuda.empty_cache()
    res["gpu_after"] = gpu_info()
    line = json.dumps(res, sort_keys=True)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
