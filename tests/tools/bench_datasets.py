"""Host and device cost of the LMDB batch loaders (coclr_b200.loaders) on a seeded UCF101-like database.

The database is written at run time to a temporary directory (tests/tools/lmdb_writer.py): 240 x 320 4:2:0 frames at
Pillow quality 75 and 90 (a pool of distinct frames per quality, repeated through the videos), video lengths drawn
from 29-900 frames.  Three configurations:
  nce     InfoNCE batch: UCF101LMDB_2CLIP, B = 32, seq_len 32, img_dim 128 (main_nce.py's flagship shape)
  coclr   CoCLR 2-stream batch: UCF101_2STREAM_LMDB_2CLIP, B = 32, seq_len 32
  test    ten-crop test pass: UCF101LMDB mode 'test', seq_len 32, 8 videos per launch, 10 views
Per configuration it prints sampled and decoded frame counts, host ms per batch (read, sample, parse, dedupe, plan:
the look-ahead thread's work), device ms per batch (decode + augment, CUDA events) and whether the host work fits in
one training step (--step-ms, 41 ms by default: DESIGN.md section 6).  The card's name and power limit are read in the
same run.  Usage: python tests/tools/bench_datasets.py [--videos 48] [--batches 6] [--step-ms 41]
"""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

import lmdb_writer as W  # noqa: E402
from coclr_b200 import datasets as D  # noqa: E402
from coclr_b200 import loaders as LD  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def make_db(root, n_videos, seed=0):
    from PIL import Image
    r = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:240, 0:320].astype(np.float32)
    pools = {}
    for q in (75, 90):
        pools[q] = []
        for _ in range(32):
            fx, fy, ph = r.uniform(6, 30, 3), r.uniform(6, 30, 3), r.uniform(0, 6.3, 3)
            img = np.stack([128 + 90 * np.sin(xx / fx[c] + ph[c]) * np.cos(yy / fy[c]) for c in range(3)], -1)
            img = np.clip(img + r.normal(0, 8, img.shape), 0, 255).astype(np.uint8)
            b = io.BytesIO()
            Image.fromarray(img).save(b, "JPEG", quality=q)
            pools[q].append(b.getvalue())
    classes = ["Class%02d" % c for c in range(4)]
    videos, rows, source = {}, {"train": [], "test": []}, {}
    for v in range(n_videos):
        c = classes[v % len(classes)]
        vid = "v_%s_g%02d_c01" % (c, v)
        n = int(r.randint(29, 901))
        pool = pools[75 if v % 2 else 90]
        start = int(r.randint(32))
        videos["%s/%s" % (c, vid)] = [pool[(start + t) % 32] for t in range(n)]
        rows["test" if (v // 4) % 4 == 3 else "train"].append("/data/UCF101/frame/%s/%s/,%d" % (c, vid, n))
        source[vid[:-4]] = v
    split = os.path.join(root, "split", "ucf101")
    os.makedirs(split)
    with open(os.path.join(split, "ClassInd.txt"), "w") as f:
        f.write("".join("%d, %s\n" % (i + 1, c) for i, c in enumerate(classes)))
    for s in ("train", "test"):
        with open(os.path.join(split, "%s_split01.csv" % s), "w") as f:
            f.write("\n".join(rows[s]) + "\n")
    with open(os.path.join(split, "video_source.json"), "w") as f:
        json.dump(source, f)
    order = sorted(videos)
    np.random.RandomState(seed + 1).shuffle(order)
    db = os.path.join(root, "ucf101_frame.lmdb")
    W.write_videos(db, videos, order)
    return split, db


def measure(loader, produce, finish, n):
    """Host ms of each produced batch, device ms of each finished one, sampled / decoded frame counts."""
    host, dev, sampled, decoded = [], [], 0, 0
    gen = produce()
    for i in range(n):
        t = time.perf_counter()
        try:
            item = next(gen)
        except StopIteration:
            break
        host.append((time.perf_counter() - t) * 1e3)
        batch, slots = item[0], item[1]
        sampled += sum(len(s) for s in slots)
        decoded += len(batch)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        finish(item)
        e1.record()
        torch.cuda.synchronize()
        dev.append(e0.elapsed_time(e1))
    return host, dev, sampled, decoded


def report(name, host, dev, sampled, decoded, step_ms, warm=1):
    h, d = host[warm:] or host, dev[warm:] or dev
    res = {"config": name, "batches": len(h), "sampled_frames": sampled, "decoded_frames": decoded,
           "host_ms_per_batch": round(float(np.median(h)), 2), "device_ms_per_batch": round(float(np.median(d)), 2),
           "lookahead_keeps_up": bool(np.median(h) <= step_ms)}
    print(json.dumps(res))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=48)
    ap.add_argument("--batches", type=int, default=6)
    ap.add_argument("--step-ms", type=float, default=41.0)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_datasets.py measures on a CUDA device"
    torch.cuda.set_device(0)
    print("card:", card())
    dev = torch.device("cuda")
    with tempfile.TemporaryDirectory() as tmp:
        t = time.perf_counter()
        split, db = make_db(tmp, a.videos)
        print("database: %d videos, %.0f MB, written in %.1f s" % (
            a.videos, os.path.getsize(os.path.join(db, "data.mdb")) / 2 ** 20, time.perf_counter() - t))
        nce = D.UCF101LMDB_2CLIP(root=split, db_path=db, mode="train", num_frames=32, return_label=True)
        ld = LD.PretrainBatches(nce, 32, 32, 128, dev, seed=0)
        ld.order = (ld.order * (1 + 32 * a.batches // max(len(ld.order), 1)))[:32 * a.batches]
        report("nce B=32 seq_len=32", *measure(ld, ld._produce, ld._finish, a.batches), a.step_ms)
        two = D.UCF101_2STREAM_LMDB_2CLIP(root=split, db_path_flow=db, db_path_rgb=db, mode="train", num_frames=32,
                                          return_label=True, return_source=True)
        ld = LD.PretrainBatches(two, 32, 32, 128, dev, seed=0, two_stream=True)
        ld.order = (ld.order * (1 + 32 * a.batches // max(len(ld.order), 1)))[:32 * a.batches]
        report("coclr 2-stream B=32 seq_len=32", *measure(ld, ld._produce, ld._finish, a.batches), a.step_ms)
        test = D.UCF101LMDB(root=split, db_path=db, mode="test", num_frames=32, return_label=True)
        host, devt, sampled, decoded = [], [], 0, 0
        for flip in (0, 1):
            for aug in (5, 1, 2, 3, 4):
                tv = LD.TestVideos(test, 32, 128, dev, seed=10 * aug + flip, view=(aug, flip))
                h, d, s, n = measure(tv, tv._produce, tv._finish, 10 ** 6)
                host += h
                devt += d
                sampled += s
                decoded += n
        report("ten-crop test, %d videos x 10 views, 8 per launch" % len(test), host, devt, sampled, decoded,
               a.step_ms, warm=0)


if __name__ == "__main__":
    main()
