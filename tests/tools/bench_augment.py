"""Pre-training augmentation on one GPU (coclr_b200.augment): ms per batch, frames/s and achieved HBM bandwidth of the
kernel for the full reference recipe of main_nce.py (one stream) and main_coclr.py (two streams) on a device-resident
batch, and one InfoNCE training step with and without the augmentation in front of it.  The plan (host draws and
tables) is made once per recipe outside the timed window; what is timed is the kernel.  CUDA events around warmed-up
repetitions; prints one JSON line with the card name, power limit and SM clock.

Bytes moved are what the kernel must read and write at least: the source pixels inside each clip's crop box (read once
per clip; a one-clip sample reads its half twice) plus the fp32 output.

  python tests/tools/bench_augment.py [--batch 32] [--seq 32] [--img 128] [--src 240 320] [--reps 20] [--out FILE]
"""
import argparse
import json
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_classifier import gpu_info  # noqa: E402
from bench_eval import event_time  # noqa: E402


def bytes_moved(aug, plan):
    read = 0
    for sp in plan.samples:
        h, w = sp.size
        for c in sp.clips:
            cw, ch = (c.crop[2], c.crop[3]) if c.crop is not None else (w, h)
            read += aug.S * cw * ch * 3
    return read + len(plan) * 2 * aug.S * 3 * aug.img_dim ** 2 * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seq", type=int, default=32)
    ap.add_argument("--img", type=int, default=128)
    ap.add_argument("--src", type=int, nargs=2, default=[240, 320])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    from coclr_b200.augment import PretrainAugment
    from coclr_b200 import moco
    from model.pretrain import InfoNCE
    assert torch.cuda.is_available(), "bench_augment needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, T, D, (H, W) = a.batch, a.seq, a.img, a.src
    res = {"gpu": gpu_info(), "batch": B, "seq_len": T, "img_dim": D, "source": [H, W]}
    g = torch.Generator(device=dev).manual_seed(0)
    x_aug = None
    for name, two in (("nce", False), ("coclr", True)):
        aug = PretrainAugment(T, D, two_stream=two)
        frames = torch.randint(0, 256, (B, aug.frames, H, W, 3), dtype=torch.uint8, device=dev, generator=g)
        plan = aug.plan([(H, W)] * B, random.Random(1), np.random.RandomState(1), torch.Generator().manual_seed(1))
        ms = event_time(lambda: aug(frames, plan), a.reps, 3)
        nbytes = bytes_moved(aug, plan)
        res[name] = {"ms_per_batch": ms, "frames_per_s": B * 2 * aug.S / ms * 1e3, "bytes_moved": nbytes,
                     "achieved_GBps": nbytes / ms / 1e6, "source_bytes": frames.numel()}
        if not two:
            x_aug = (aug, frames, plan)
    # one InfoNCE step (S3D, K=2048) on already-augmented input, then with the augmentation in front
    aug, frames, plan = x_aug
    model = InfoNCE("s3d", 128, 2048).to(dev).train()
    model.set_input_transform()
    opt = moco.FlatAdam(model.encoder_q)
    x = aug(frames, plan)

    def step(inp):
        logits, labels = model(inp)
        loss = moco.nce_cross_entropy(logits, labels)
        opt.zero_grad()
        loss.backward()
        opt.step()

    reps = max(3, a.reps // 4)
    res["infonce_step_ms"] = event_time(lambda: step(x), reps, 3)
    res["infonce_step_with_augment_ms"] = event_time(lambda: step(aug(frames, plan)), reps, 3)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
