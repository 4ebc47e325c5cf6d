"""JPEG decoding on one GPU (coclr_b200.jpeg): B = 32 batches of 240 x 320 4:2:0 frames at quality 75 and 90, 2048
frames (InfoNCE: 32 x 2 clips x 32) and 4096 (CoCLR: two streams).  Reports, in one JSON line with the card name, power
limit and SM clock:

  * ms per batch and frames/s of the whole call (CUDA events around warmed-up repetitions; the upload of the bytes is
    inside the call), and the three kernels' times from a separate torch.profiler run;
  * bytes in (JPEG), workspace traffic, uint8 out, and the achieved GB/s of the call;
  * host parse and pack time per batch (dec.parse on the list of bytes);
  * Pillow's `Image.open(BytesIO(raw)).convert('RGB')` on one core for the same frames (per frame, and per batch);
  * torchvision.io.decode_jpeg(device='cuda') (nvJPEG) on the same batch, with its max abs difference to Pillow;
  * one InfoNCE step (S3D, K = 2048) with augmentation alone, and with decode + augmentation in front.

Workspace traffic: the entropy stage writes 128 bytes per 8 x 8 block, the IDCT reads them and writes 64, the colour
stage reads the 64 (at least once).  The frame content is a smooth field plus noise, 256 distinct frames tiled.

  python tests/tools/bench_jpeg.py [--reps 20] [--out FILE]
"""
import argparse
import io
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

from bench_classifier import gpu_info  # noqa: E402
from bench_eval import event_time  # noqa: E402
import jpeg_cases as JC  # noqa: E402

H, W, B, T = 240, 320, 32, 32


def pool(quality, n=256):
    return [JC.encode(JC.field(H, W, 5000 + i, noise=6.0), quality=quality, subsampling=2) for i in range(n)]


def pillow_per_frame(raws):
    """ms per frame of pil_from_raw_rgb on one core."""
    from PIL import Image
    aff = os.sched_getaffinity(0)
    os.sched_setaffinity(0, {min(aff)})
    try:
        t0 = time.perf_counter()
        for r in raws:
            Image.open(io.BytesIO(r)).convert("RGB").load()
        return (time.perf_counter() - t0) / len(raws) * 1e3
    finally:
        os.sched_setaffinity(0, aff)


def kernel_ms(dec, batch, out, reps):
    """Mean ms per call of each of the decoder's kernels, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(2):
        dec(batch, out=out, check=False)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            dec(batch, out=out, check=False)
        torch.cuda.synchronize()
    res = {}
    for e in prof.key_averages():
        for k in ("entropy", "idct", "colour"):
            if "jpeg_%s_kernel" % k in e.key:
                res[k] = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3 / reps
    return res


def nvjpeg(raws, ref):
    try:
        from torchvision.io import decode_jpeg
        datas = [torch.frombuffer(bytearray(r), dtype=torch.uint8) for r in raws]
        imgs = decode_jpeg(datas, device="cuda")
        diff = max(int((i.permute(1, 2, 0).cpu().int() - torch.from_numpy(np.array(f)).int()).abs().max())
                   for i, f in zip(imgs[:64], ref))
        ms = event_time(lambda: decode_jpeg(datas, device="cuda"), 5, 2)
        return {"ms_per_batch": ms, "max_abs_diff_to_pillow_first64": diff}
    except Exception as e:  # noqa: BLE001 - reported, not raised: the comparison is optional
        return "not available: %s" % (str(e).splitlines()[0][:200] if str(e) else type(e).__name__)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    from coclr_b200.jpeg import JpegDecoder
    assert torch.cuda.is_available(), "bench_jpeg needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = {"gpu": gpu_info(), "frame": [H, W], "sampling": "4:2:0", "batch": B}
    dec = JpegDecoder()
    keep = None
    for q in (75, 90):
        frames = pool(q)
        ref = [JC.pillow_decode(r) for r in frames[:64]]
        res["q%d_pillow_ms_per_frame_one_core" % q] = pillow_per_frame(frames[:128])
        for name, n in (("nce", 2 * B * T), ("coclr", 4 * B * T)):
            raws = [frames[i % len(frames)] for i in range(n)]
            t0 = time.perf_counter()
            for _ in range(3):
                batch = dec.parse(raws)
            parse_ms = (time.perf_counter() - t0) / 3 * 1e3
            out = torch.empty(n, H, W, 3, dtype=torch.uint8, device=dev)
            dec(batch, out=out)
            got = out[:64].cpu().numpy()
            assert all(np.array_equal(g, r) for g, r in zip(got, ref)), "decode differs from Pillow"
            ms = event_time(lambda: dec(batch, out=out, check=False), a.reps, 3)
            nb = int(batch.frames["blocks"].sum())
            bytes_in, work, bytes_out = len(batch.data), nb * (128 + 128 + 64 + 64), n * H * W * 3
            r = {"frames": n, "ms_per_batch": ms, "frames_per_s": n / ms * 1e3, "kernels_ms": kernel_ms(dec, batch, out, 5),
                 "bytes_in": bytes_in, "workspace_bytes": batch.work_bytes, "workspace_traffic": work,
                 "bytes_out": bytes_out, "achieved_GBps": (bytes_in + work + bytes_out) / ms / 1e6,
                 "host_parse_ms": parse_ms, "pillow_one_core_ms_per_batch": res["q%d_pillow_ms_per_frame_one_core" % q] * n,
                 "jpeg_to_raw_ratio": bytes_out / bytes_in}
            if name == "nce":
                r["nvjpeg"] = nvjpeg(raws, ref)
            res["q%d_%s" % (q, name)] = r
            if q == 75 and name == "nce":
                keep = (raws, batch)
    # one InfoNCE step: augment alone (frames already decoded on the device), then decode + augment
    from coclr_b200.augment import PretrainAugment
    from coclr_b200 import moco
    from model.pretrain import InfoNCE
    raws, batch = keep
    aug = PretrainAugment(T, 128)
    frames = dec(batch).view(B, 2 * T, H, W, 3)
    plan = aug.plan(batch.sample_sizes(B), random.Random(1), np.random.RandomState(1), torch.Generator().manual_seed(1))
    model = InfoNCE("s3d", 128, 2048).to(dev).train()
    model.set_input_transform()
    opt = moco.FlatAdam(model.encoder_q)
    buf = torch.empty(2 * B * T, H, W, 3, dtype=torch.uint8, device=dev)

    def step(inp):
        logits, labels = model(inp)
        loss = moco.nce_cross_entropy(logits, labels)
        opt.zero_grad()
        loss.backward()
        opt.step()

    reps = max(3, a.reps // 4)
    res["infonce_step_with_augment_ms"] = event_time(lambda: step(aug(frames, plan)), reps, 3)
    res["infonce_step_with_decode_augment_ms"] = event_time(
        lambda: step(aug(dec(batch, out=buf, check=False).view(B, 2 * T, H, W, 3), plan)), reps, 3)
    res["augment_ms"] = event_time(lambda: aug(frames, plan), a.reps, 3)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
