"""TV-L1 flow on one GPU (coclr_b200.flow and tools/make_flow_lmdb.py).  Inputs are seeded moving-texture videos of
64 frames (63 pairs) at 240 x 320 (UCF101) and 256 x 340 (K400-256): a smooth texture translating by a sub-pixel
step per frame plus a second texture patch moving the other way, with noise, JPEG-encoded (Pillow, quality 90).

For each size it reports, in one JSON line with the card name and power limit read in the same run:
  * device ms per pair of one 63-pair solve (CUDA events around warmed-up repetitions);
  * the iteration histogram per scale (iterations per warp, over pairs and warps);
  * the bytes the primal-dual iterations move, from shapes (88 bytes per pixel per iteration of an active pair: the
    u-step reads u, p, I1wx, I1wy, g, rho_c and writes u; the p-step reads u and p and writes p), over the two
    iteration kernels' time from a separate torch.profiler run, against 3.35 TB/s (H100 SXM HBM3 data sheet);
  * host encode ms per frame (Pillow, one core) and the tool's end-to-end pairs/s on a database of 4 such videos.

  python tests/tools/bench_flow.py [--reps 3] [--out FILE]
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

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))

HBM_BYTES_PER_S = 3.35e12
BYTES_PER_PIXEL_ITER = 88
FRAMES = 64
SIZES = (("ucf101", 240, 320), ("k400-256", 256, 340))


def video(h, w, seed, n=FRAMES):
    """n JPEG frames of a seeded moving texture."""
    import flow_oracle as O
    from PIL import Image
    r = np.random.RandomState(seed)
    v = r.uniform(0.3, 1.2, 2) * r.choice([-1, 1], 2)
    out = []
    for t in range(n):
        base = O.texture(h, w, seed, (v[0] * t, v[1] * t))
        patch = O.texture(h, w, seed + 1, (-v[0] * t, -0.5 * v[1] * t))
        y, x = np.mgrid[0:h, 0:w]
        mask = ((x - w / 2) ** 2 + (y - h / 2) ** 2) < (min(h, w) / 4) ** 2
        img = np.where(mask, patch, base) + r.normal(0, 2, (h, w))
        rgb = np.clip(np.stack([img, 0.8 * img + 20, 255 - img], -1), 0, 255).astype(np.uint8)
        b = io.BytesIO()
        Image.fromarray(rgb).save(b, "JPEG", quality=90)
        out.append(b.getvalue())
    return out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def bench_size(name, h, w, reps):
    from coclr_b200 import flow
    from coclr_b200.jpeg import JpegDecoder
    import make_flow_lmdb as M
    jpegs = video(h, w, 11)
    dec = JpegDecoder()
    g = flow.grey(dec(dec.parse(jpegs)))
    i0, i1 = g[:-1].contiguous(), g[1:].contiguous()
    P = i0.shape[0]
    f, iters = flow.tvl1(i0, i1)                           # warm-up
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        f2, it2 = flow.tvl1(i0, i1)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
        assert torch.equal(f2, f) and torch.equal(it2, iters)
    ms = sorted(times)[len(times) // 2]
    it = iters.cpu().numpy()                               # [P, S, 5]
    S = it.shape[1]
    sizes = [(h, w)]
    for _ in range(S - 1):
        sizes.append((int(sizes[-1][0] * 0.5 + 0.5), int(sizes[-1][1] * 0.5 + 0.5)))
    hist = {}
    edges = [1, 2, 11, 51, 101, 201, 300, 301]
    for s in range(S):
        c, _ = np.histogram(it[:, s].ravel(), bins=edges)
        hist["%dx%d" % sizes[s]] = {"mean": float(it[:, s].mean()), "max": int(it[:, s].max()),
                                    "bins [1,2,11,51,101,201,300,301)": c.tolist()}
    iter_bytes = sum(int(it[:, s].sum()) * sizes[s][0] * sizes[s][1] * BYTES_PER_PIXEL_ITER for s in range(S))

    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        flow.tvl1(i0, i1)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        key = next((k for k in ("tvl1_u_kernel", "tvl1_p_kernel", "warp_kernel", "blur_kernel", "resample_kernel")
                    if k in e.key), None)
        if key:
            us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            kern[key] = kern.get(key, 0.0) + us / 1e3
    iter_ms = kern.get("tvl1_u_kernel", 0.0) + kern.get("tvl1_p_kernel", 0.0)

    q = flow.quantise(f).cpu().numpy()
    t0 = time.perf_counter()
    for x in q:
        M.encode(x)
    enc_ms = (time.perf_counter() - t0) * 1e3 / len(q)

    import lmdb_writer
    with tempfile.TemporaryDirectory() as tmp:
        vids = {"c/v%d" % i: video(h, w, 20 + i) for i in range(4)}
        order = sorted(vids)
        lmdb_writer.write_videos(os.path.join(tmp, "rgb"), vids, order)
        stats = M.build(os.path.join(tmp, "rgb"), os.path.join(tmp, "flow"), 64, log=lambda *_: None)

    return {"size": name, "H": h, "W": w, "pairs": P, "scales": S,
            "device_ms_per_pair": ms / P, "solve_ms": ms, "solve_ms_reps": times,
            "iterations": hist, "iteration_bytes": iter_bytes, "kernel_ms": kern,
            "iteration_kernel_ms": iter_ms,
            "iteration_GBps": iter_bytes / (iter_ms * 1e-3) / 1e9 if iter_ms else None,
            "iteration_share_of_hbm": iter_bytes / (iter_ms * 1e-3) / HBM_BYTES_PER_S if iter_ms else None,
            "encode_ms_per_frame": enc_ms, "tool_pairs_per_s": stats["pairs_per_s"],
            "tool_solve_s": stats["solve_s"], "tool_encode_thread_s": stats["encode_s"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_flow.py needs a CUDA device")
    torch.cuda.set_device(0)
    res = {"card": card(), "sizes": [bench_size(n, h, w, args.reps) for n, h, w in SIZES]}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
