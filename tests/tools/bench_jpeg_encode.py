"""JPEG encoding of TV-L1 flow frames: the GPU encoder (coclr_b200.jpeg.JpegEncoder) against Pillow on one thread and
in a pool of min(16, cpu_count) threads (the flow tool's former encoder), on the same quantised flow frames of a
63-pair coclr_b200.flow.tvl1 solve at 240 x 320 (UCF101) and 256 x 340 (K400-256), quality 95, 4:4:4 as the flow
databases store them; the GPU encoder also at quality 75, 4:2:0 (Pillow's defaults).

Reported per size, in one JSON line with the card name and power limit read in the same run:
  * gpu_ms_per_frame: device time of one encode call (CUDA events around the launches; no copy back), per frame;
  * gpu_frames_per_s: frames per second of whole calls, files on the host (offsets and bytes copied back);
  * pillow_1_ms_per_frame and pillow_pool_frames_per_s;
  * kernel_ms: each encoder kernel's time from a separate torch.profiler run, and bytes_moved: what the kernels must
    read and write, from shapes (RGB frames in, coefficients, bit counts and the segment through the workspace, the
    files out), over their summed time.
The encoders run alternately after a warm-up; every GPU file is checked against Pillow's.

  python tests/tools/bench_jpeg_encode.py [--reps 5] [--out FILE]
"""
import argparse
import json
import os
import re
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))

import bench_flow as BF  # noqa: E402

SIZES = BF.SIZES


def flow_frames(h, w):
    from coclr_b200 import flow
    from coclr_b200.jpeg import JpegDecoder
    dec = JpegDecoder()
    g = flow.grey(dec(dec.parse(BF.video(h, w, 11))))
    f, _ = flow.tvl1(g[:-1].contiguous(), g[1:].contiguous())
    return flow.quantise(f)


def bytes_moved(q, files, s):
    n, h, w, _ = q.shape
    hs, vs = {0: (1, 1), 1: (2, 1), 2: (2, 2)}[s]
    blocks = -(-w // (8 * hs)) * -(-h // (8 * vs)) * (hs * vs + 2)
    seg = sum(len(f) for f in files)
    # frames in; coefficients written, read twice; bit counts written, scanned, read; segment written, read twice;
    # files written
    return n * (h * w * 3 + blocks * (128 * 3 + 8 * 4)) + 3 * seg + seg


def bench_size(name, h, w, reps):
    import ctypes as C
    import make_flow_lmdb as M
    from coclr_b200 import lib as L
    from coclr_b200.jpeg import JpegEncoder
    lib = L.load()
    q = flow_frames(h, w)
    qh = q.cpu().numpy()
    n = q.shape[0]
    res = {"size": name, "H": h, "W": w, "frames": n}
    threads = min(16, os.cpu_count() or 1)
    pool = ThreadPoolExecutor(threads)
    want = [M.encode(x) for x in qh]
    for quality, s, tag in ((M.QUALITY, M.SUBSAMPLING, "q95_444"), (75, 2, "q75_420")):
        enc = JpegEncoder(quality, s)
        out = enc(q)                                   # warm-up
        if tag == "q95_444":
            assert out == want, "GPU files differ from Pillow's"
        dev_ms, call_s, p1, pp = [], [], [], []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            p = L.JpegEncode(n, h, w, quality, s, L.dptr(q), q.stride(0), q.stride(1), L.dptr(enc._out),
                             enc._out.numel(), L.dptr(enc._offsets), L.dptr(enc._work), enc._work.numel())
            L.check(lib.coclr_jpeg_encode(C.byref(p), L.stream_ptr()), "coclr_jpeg_encode")
            b.record()
            b.synchronize()
            dev_ms.append(a.elapsed_time(b))
            t0 = time.perf_counter()
            enc(q)
            call_s.append(time.perf_counter() - t0)
            if tag == "q95_444":
                t0 = time.perf_counter()
                for x in qh:
                    M.encode(x)
                p1.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                list(pool.map(M.encode, qh))
                pp.append(time.perf_counter() - t0)
        med = lambda v: sorted(v)[len(v) // 2]         # noqa: E731
        r = {"gpu_ms_per_frame": med(dev_ms) / n, "gpu_ms_reps": dev_ms,
             "gpu_frames_per_s": n / med(call_s), "mean_file_bytes": sum(len(f) for f in out) / n}
        if tag == "q95_444":
            r.update({"pillow_1_ms_per_frame": med(p1) * 1e3 / n, "pillow_pool_threads": threads,
                      "pillow_pool_frames_per_s": n / med(pp)})
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            enc(q)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            m = re.search(r"jpeg_enc_\w+(<\w+>)?", e.key)
            if m:
                us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                kern[m.group(0)] = kern.get(m.group(0), 0.0) + us / 1e3
        total_ms = sum(kern.values())
        moved = bytes_moved(q, out, s)
        r.update({"kernel_ms": kern, "kernel_ms_total": total_ms, "bytes_moved": moved,
                  "GBps": moved / (total_ms * 1e-3) / 1e9 if total_ms else None})
        res[tag] = r
    pool.shutdown()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_jpeg_encode.py needs a CUDA device")
    torch.cuda.set_device(0)
    res = {"card": BF.card(), "cpu_count": os.cpu_count(),
           "sizes": [bench_size(n, h, w, args.reps) for n, h, w in SIZES]}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
