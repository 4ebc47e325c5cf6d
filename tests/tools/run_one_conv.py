"""Profiling helper (test infrastructure): runs one implicit-GEMM conv launch shape repeatedly so that ncu can
capture it.  python tests/tools/run_one_conv.py fwd|dgrad|wgrad Cin Cout kt kh kw B T H W [npass] [iters]"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from coclr_b200 import ops  # noqa: E402

mode = sys.argv[1]
Cin, Cout, kt, kh, kw, B, T, H, W = [int(v) for v in sys.argv[2:11]]
npass = int(sys.argv[11]) if len(sys.argv) > 11 else 3
iters = int(sys.argv[12]) if len(sys.argv) > 12 else 5
stride = tuple(int(v) for v in os.environ.get("STRIDE", "1,1,1").split(","))   # (B,T,H,W) are the conv INPUT dims
geom = ops.Geometry((kt, kh, kw), stride, (kt // 2, kh // 2, kw // 2))
To, Ho, Wo = geom.out_dims(T, H, W)
dev = "cuda"
r8 = lambda c: (c + 7) // 8 * 8
w = torch.randn(Cout, Cin, kt, kh, kw, device=dev) * 0.05
if mode == "s2d":
    # the space-to-depth stem as the engine launches it: (1,4,4) over 16-channel pixels, zero-padded rows (W + 4), pw = 0
    geom = ops.Geometry((1, 4, 4), (1, 1, 1), (0, 2, 0))
    To, Ho, Wo = T, H, W
    x = ops.Planes((B, T, H, W + 4, 16), 0, dev, zero=True)
    x.hi[..., 2:-2, :12].normal_(); x.lo[..., 2:-2, :12].normal_(0, 1e-3)
    w = torch.randn(Cout, 16, 1, 4, 4, device=dev) * 0.05
    pw = ops.PackedWeights(Cout, 16, 16, 16, 0, 0, dev).pack(w)
    dst = torch.empty(B, To, Ho, Wo, Cout, device=dev)
    stats = torch.zeros(2 * Cout, dtype=torch.float64, device=dev)
    run = lambda: ops.conv_igemm(x.src(0, 16, T, H, W + 4), 0, geom.c(0), B, (To, Ho, Wo), pw, dst, stats=stats, npass=npass)
elif mode == "fwd":
    x = ops.Planes((B, T, H, W, r8(Cin)), 0, dev)
    x.hi.normal_(); x.lo.normal_(0, 1e-3)
    pw = ops.PackedWeights(Cout, Cin, geom.taps, r8(Cin), 0, 0, dev).pack(w)
    dst = torch.empty(B, To, Ho, Wo, Cout, device=dev)
    stats = torch.zeros(2 * Cout, dtype=torch.float64, device=dev)
    run = lambda: ops.conv_igemm(x.src(0, r8(Cin), T, H, W), 0, geom.c(0), B, (To, Ho, Wo), pw, dst, stats=stats, npass=npass)
elif mode == "dgrad":
    dy = ops.Planes((B, To, Ho, Wo, r8(Cout)), 1, dev)
    dy.hi.normal_(); dy.lo.normal_(0, 1e-3)
    pw = ops.PackedWeights(Cout, Cin, geom.taps, r8(Cout), 1, 1, dev).pack(w)
    dst = torch.zeros(B, T, H, W, Cin, device=dev)
    run = lambda: ops.conv_igemm(dy.src(0, r8(Cout), To, Ho, Wo), 1, geom.c(1), B, (T, H, W), pw, dst, accumulate=False, npass=npass)
else:
    x = ops.Planes((B, T, H, W, r8(Cin)), 1, dev)
    x.hi.normal_(); x.lo.normal_(0, 1e-3)
    dy = ops.Planes((B, To, Ho, Wo, r8(Cout)), 1, dev)
    dy.hi.normal_(); dy.lo.normal_(0, 1e-3)
    dw = torch.zeros_like(w)
    splits = int(os.environ.get("SPLITS", "50"))
    ws = [True]     # allocated by the first call, reused afterwards

    def run():
        ws[0] = ops.conv_wgrad(x.src(0, r8(Cin), T, H, W), 1, geom.c(0), dy.src(0, r8(Cout), To, Ho, Wo), 1, B,
                               (To, Ho, Wo), Cout, Cin, dw, npass=npass, splits=splits, workspace=ws[0])
for _ in range(2):
    run()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(iters):
    run()
e1.record()
torch.cuda.synchronize()
print("%s %s: %.3f ms/launch" % (mode, sys.argv[2:11], e0.elapsed_time(e1) / iters))
