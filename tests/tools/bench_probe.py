"""Times the feature linear probe at the UCF101 split-1 shape (9537 train / 3783 test rows, D = 1024, C = 101,
batch 1024, 100 epochs, eval every 5, --final_bn) with CUDA events:

  * the engine (coclr_b200.probe.fit) for one config and for the 12-config grid lr {0.1, 0.3, 1.0} x
    wd {1e-4, 1e-3, 1e-2, 1e-1};
  * the reference-shaped torch loop (tests/tools/probe_oracle.py, reference_shaped=True: per-row Dataset, pinned
    DataLoader, .item() every step) for one config, on the same GPU in the same process;
  * the two GEMMs of a training step alone (coclr_sim_fp32: logits [B, S*C] and G [S*C, D]) for S = 1 and 12, with
    their achieved FLOP/s.

    python tests/tools/bench_probe.py [--epochs 100] [--reps 3]

Prints one JSON line.  Writes nothing.
"""
import argparse
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))

N, NQ, D, C, B = 9537, 3783, 1024, 101, 1024
LRS, WDS = [0.1, 0.3, 1.0], [1e-4, 1e-3, 1e-2, 1e-1]


def features(seed=1, r=64, sep=0.35):
    g = torch.Generator().manual_seed(seed)
    means = sep * torch.randn(C, r, generator=g)
    P = torch.randn(r, D, generator=g) / r ** 0.5 * (torch.rand(D, generator=g) + 0.5)

    def split(n):
        y = torch.arange(n) % C
        return (means[y] + torch.randn(n, r, generator=g)) @ P + 0.05 * torch.randn(n, D, generator=g), y

    return split(N) + split(NQ)


def timed(fn, reps):
    """Best of reps wall times (ms) between CUDA events around fn()."""
    best = float("inf")
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b))
    return best


def gemm_ms(S, reps=50):
    from coclr_b200 import lib as L
    lib = L.load()
    dev = torch.device("cuda")
    xh = torch.randn(B, D, device=dev)
    xhT = xh.t().contiguous()
    W = torch.randn(S * C, D, device=dev)
    dlT = torch.randn(S * C, B, device=dev)
    logits = torch.empty(B, S * C, device=dev)
    G = torch.empty(S * C, D, device=dev)
    fwd = lambda: lib.coclr_sim_fp32(L.dptr(xh), L.dptr(W), L.dptr(logits), B, S * C, D, L.stream_ptr())  # noqa
    bwd = lambda: lib.coclr_sim_fp32(L.dptr(dlT), L.dptr(xhT), L.dptr(G), S * C, D, B, L.stream_ptr())  # noqa
    out = {}
    for name, f in (("logits", fwd), ("G", bwd)):
        f()
        ms = timed(lambda: [f() for _ in range(reps)], 3) / reps
        out[name] = dict(ms=ms, tflops=2.0 * B * D * S * C / ms / 1e9)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    from coclr_b200 import probe as P
    import probe_oracle as O
    dev = torch.device("cuda")
    x = [t.to(dev) for t in features()]
    kw = dict(epochs=a.epochs, eval_freq=5, final_bn=True)
    steps = a.epochs * math.ceil(N / B)
    P.fit(*x, [1.0], [1e-3], epochs=2, final_bn=True)   # load the library, warm the allocator
    res = {"shape": dict(N=N, Nq=NQ, D=D, C=C, batch=B, epochs=a.epochs, steps=steps),
           "device": torch.cuda.get_device_name(0)}
    for name, lrs, wds in (("engine_1", [1.0], [1e-3]), ("engine_12", LRS, WDS)):
        ms = timed(lambda: P.fit(*x, lrs, wds, **kw), a.reps)
        res[name] = dict(ms=ms, ms_per_step=ms / steps)
    cpu = [t.cpu() for t in x]
    ms = timed(lambda: O.fit(*cpu, [1.0], [1e-3], dtype=torch.float32, device=dev, reference_shaped=True, **kw), 1)
    res["torch_reference_shaped_1"] = dict(ms=ms, ms_per_step=ms / steps)
    res["speedup_1"] = res["torch_reference_shaped_1"]["ms"] / res["engine_1"]["ms"]
    res["speedup_12_vs_12_torch_runs"] = 12 * res["torch_reference_shaped_1"]["ms"] / res["engine_12"]["ms"]
    res["gemm_S1"], res["gemm_S12"] = gemm_ms(1), gemm_ms(12)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
