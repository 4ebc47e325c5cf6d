"""Classifier augmentation on one GPU (coclr_b200.clf_augment): ms per batch and achieved HBM bandwidth of the kernel
for the train recipe of eval/main_classifier.py (crop -> 224 -> img_dim, the reference's jitter mix, the batch flip)
and for one ten-crop test view over a batch of videos, on device-resident uint8 frames; plus the train recipe's cost
against the fine-tuning step times of DESIGN.md §6 (`ft` 33.0 ms, `last` 10.4 ms per 32-clip step, same card).  The plan
(host draws and tables) is made once outside the timed window; what is timed is the kernel.  CUDA events around
warmed-up repetitions; prints one JSON line with the card name, power limit and SM clock.

Bytes moved are what the kernel must read and write at least: the source pixels inside each sample's first-resize
window (read once per frame) plus the fp32 output.

  python tests/tools/bench_clf_augment.py [--batch 32] [--seq 32] [--img 128] [--src 240 320] [--reps 20] [--out FILE]

--pil instead times the reference's PIL train recipe per frame on the CPU (needs $COCLR_REFERENCE; run it under
`taskset -c 0` for one core):

  COCLR_REFERENCE=<checkout> taskset -c 0 python tests/tools/bench_clf_augment.py --pil
"""
import argparse
import json
import os
import random
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

STEP_MS = {"ft": 33.0, "last": 10.4}     # DESIGN.md §6, fine-tuning at B = 32, T = 32, 128², one H100 at 700 W


def bytes_moved(aug, plan):
    read = 0
    for sp in plan.samples:
        (xs, xn, _), (ys, yn, _) = aug.first_taps(sp)
        cols = int((xs + xn).max() - xs.min())
        rows = int((ys + yn).max() - ys.min())
        read += sp.frames * cols * rows * 3
    return read + sum(plan.lengths) * 3 * aug.img_dim ** 2 * 4


def pil_reference(a):
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_golden_clf_augment import load, recipe
    import make_golden_clf_augment as MG
    from PIL import Image
    torch.set_num_threads(1)
    A = load("utils/augmentation.py", "reference_augmentation")
    MG.D = a.img
    tf = recipe(A, a.seq, "train")
    rng = np.random.default_rng(0)
    H, W = a.src
    frames = [Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)) for _ in range(a.seq)]
    random.seed(0)
    tf(frames)
    n = max(3, a.reps // 4)
    t0 = time.perf_counter()
    for _ in range(n):
        torch.stack(tf(frames), 1)
    ms = (time.perf_counter() - t0) / n * 1e3
    return {"pil_ms_per_sample": ms, "pil_ms_per_frame": ms / a.seq, "frames_per_sample": a.seq, "source": [H, W],
            "img_dim": a.img, "cpu": open("/proc/cpuinfo").read().split("model name")[1].split("\n")[0].strip("\t: ")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seq", type=int, default=32)
    ap.add_argument("--img", type=int, default=128)
    ap.add_argument("--src", type=int, nargs=2, default=[240, 320])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--pil", action="store_true")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if a.pil:
        res = pil_reference(a)
    else:
        from bench_classifier import gpu_info
        from bench_eval import event_time
        from coclr_b200.clf_augment import ClassifierAugment
        assert torch.cuda.is_available(), "bench_clf_augment needs a CUDA device"
        dev = torch.device("cuda", 0)
        torch.cuda.set_device(dev)
        B, T, D, (H, W) = a.batch, a.seq, a.img, a.src
        res = {"gpu": gpu_info(), "batch": B, "seq_len": T, "img_dim": D, "source": [H, W]}
        g = torch.Generator(device=dev).manual_seed(0)
        aug = ClassifierAugment("train", T, D)
        frames = torch.randint(0, 256, (B, T, H, W, 3), dtype=torch.uint8, device=dev, generator=g)
        plan = aug.plan([(H, W)] * B, random.Random(1), batch_flip=True)
        ms = event_time(lambda: aug(frames, plan), a.reps, 3)
        nb = bytes_moved(aug, plan)
        res["train"] = {"ms_per_batch": ms, "frames_per_s": B * T / ms * 1e3, "bytes_moved": nb,
                        "achieved_GBps": nb / ms / 1e6, "jittered_samples": sum(s.jitter is not None for s in plan),
                        "vs_step": {k: ms / v for k, v in STEP_MS.items()}}
        view = ClassifierAugment("test", T, D, view=(1, 1))
        lengths = [T * (1 + i % 3) for i in range(B)]            # videos of 1-3 clips
        vframes = torch.randint(0, 256, (sum(lengths), H, W, 3), dtype=torch.uint8, device=dev, generator=g)
        vplan = view.plan([(H, W)] * B, random.Random(2), lengths=lengths)
        ms = event_time(lambda: view(vframes, vplan), a.reps, 3)
        nb = bytes_moved(view, vplan)
        res["ten_crop_view"] = {"videos": B, "frames": sum(lengths), "ms_per_batch": ms,
                                "frames_per_s": sum(lengths) / ms * 1e3, "bytes_moved": nb,
                                "achieved_GBps": nb / ms / 1e6}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
