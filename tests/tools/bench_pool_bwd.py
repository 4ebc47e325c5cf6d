"""Max-pool backward launches of the S3D training step (coclr_maxpool_bwd), one at a time, on one GPU.

Builds the benchmark's InfoNCE model (S3D, B=32 clip pairs of 32 x 128^2 frames, K=2048), runs warm-up training steps,
then records the arguments of the query encoder's 13 coclr_maxpool_bwd launches from one step: their C, dims, window
and accumulate flag as the plan made them, and an idx from a real forward over post-ReLU data (ties at 0 included).
Each launch is then repeated on its own between CUDA events.  Per launch and in total it reports:
  * the bytes the backward has to move, from shapes: dY (4 B) and idx (1 B) per output element, dX written (4 B) or
    read and written (8 B, accumulate) per input element;
  * device ms per launch (mean over --reps after --warm repetitions);
  * that time's share of the HBM floor, bytes / 3.35 TB/s (H100 SXM HBM3 data sheet).
The card name, power limit and maximum SM clock are read in the same run.  A table goes to stderr, one JSON line to
stdout.

  python tests/tools/bench_pool_bwd.py [--reps 50] [--warm 5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def pool_bytes(o):
    n_out = o.B * o.To * o.Ho * o.Wo * o.C
    n_in = o.B * o.Ti * o.Hi * o.Wi * o.C
    return 5 * n_out + (8 if o.accumulate else 4) * n_in


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warm", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pool_bwd.py needs a CUDA device")
    from coclr_b200 import moco
    from coclr_b200.engine import EncoderEngine
    from model.pretrain import InfoNCE

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, T, HW, K = 32, 32, 128, 2048
    torch.manual_seed(0)
    model = InfoNCE("s3d", 128, K, 0.999, 0.07).to(dev).train()
    opt = moco.FlatAdam(model.encoder_q, lr=1e-3, weight_decay=1e-5)
    block = torch.randn(B, 2, 3, T, HW, HW, generator=torch.Generator().manual_seed(1000)).to(dev)

    def step():
        logits, labels = model(block)
        loss = moco.nce_cross_entropy(logits, labels)
        opt.zero_grad()
        loss.backward()
        opt.step()

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    EncoderEngine.profile = []
    try:
        step()
        torch.cuda.synchronize()
        prof = EncoderEngine.profile
    finally:
        EncoderEngine.profile = None
    launches = [a for name, a, _, _ in prof if name == "coclr_maxpool_bwd"]
    from coclr_b200 import lib as L
    lib = L.load()
    stream = L.stream_ptr()

    def fn(*a):
        rc = lib.coclr_maxpool_bwd(*a, stream)
        if rc != 0:
            raise L.CoclrError("coclr_maxpool_bwd failed with code %d" % rc)

    rows = []
    for a in launches:
        o = a[0]._obj
        for _ in range(args.warm):
            fn(*a)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            fn(*a)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.reps
        nbytes = pool_bytes(o)
        floor = nbytes / HBM_BYTES_PER_S * 1e3
        g = o.g
        rows.append({"C": o.C, "ldx": o.ldx, "x_coff": o.x_coff, "in": [o.Ti, o.Hi, o.Wi], "out": [o.To, o.Ho, o.Wo],
                     "k": [g.kt, g.kh, g.kw], "s": [g.st, g.sh, g.sw], "p": [g.pt, g.ph, g.pw],
                     "accumulate": o.accumulate, "MB": round(nbytes / 1e6, 1), "ms": round(ms, 4),
                     "floor_ms": round(floor, 4), "floor_frac": round(floor / ms, 3)})
    tot_ms = sum(r["ms"] for r in rows)
    tot_floor = sum(r["floor_ms"] for r in rows)
    gpu = card()
    print("card: %s" % gpu, file=sys.stderr)
    print("%5s %14s %14s %7s %7s %3s %8s %8s %8s %6s" % ("C", "in", "out", "k", "s", "acc", "MB", "ms", "floor",
                                                         "frac"), file=sys.stderr)
    for r in rows:
        print("%5d %14s %14s %7s %7s %3d %8.1f %8.4f %8.4f %6.3f" % (
            r["C"], "x".join(map(str, r["in"])), "x".join(map(str, r["out"])), "".join(map(str, r["k"])),
            "".join(map(str, r["s"])), r["accumulate"], r["MB"], r["ms"], r["floor_ms"], r["floor_frac"]),
            file=sys.stderr)
    print("total: %d launches %.3f ms, floor %.3f ms (%.1f %%)" % (len(rows), tot_ms, tot_floor,
                                                                   100 * tot_floor / tot_ms), file=sys.stderr)
    line = json.dumps({"card": gpu, "launches": len(rows), "total_ms": round(tot_ms, 4),
                       "floor_ms": round(tot_floor, 4), "floor_frac": round(tot_floor / tot_ms, 3),
                       "reps": args.reps, "rows": rows})
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
