"""Bit reproducibility of the gather convolution kernel (conv_igemm.cu): the same launch, run twice on the same inputs,
writes identical outputs and identical BatchNorm statistics.  The cases are the launch kinds the TMA-staged kernel
declines: (1,3,3) convs over 8x8 and 4x4 frames, a (3,1,1) conv whose channel count is not a multiple of 64, a
16-channel input, a spatially strided ResNet-50 conv2, and a strided data gradient added into a channel slice."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# (name, Cin, Cout, k, s, p, B, T, H, W)
CASES = [
    ("s3d_m4f_sp_160_320", 160, 320, (1, 3, 3), (1, 1, 1), (0, 1, 1), 4, 8, 8, 8),
    ("s3d_m5c_sp_192_384", 192, 384, (1, 3, 3), (1, 1, 1), (0, 1, 1), 4, 8, 4, 4),
    ("s3d_tm_208_208", 208, 208, (3, 1, 1), (1, 1, 1), (1, 0, 0), 4, 4, 4, 4),
    ("sp_16_32", 16, 32, (1, 3, 3), (1, 1, 1), (0, 1, 1), 2, 4, 16, 16),
    ("r50_conv2_s2", 128, 128, (1, 3, 3), (1, 2, 2), (0, 1, 1), 2, 2, 16, 16),
]


def _planes(ops, x, bf16, coff=8):
    """NCDHW fp32 -> hi/lo planes with the channels at [coff, coff + C) of a wider buffer."""
    B, Cc, T, H, W = x.shape
    Cp = (Cc + 7) // 8 * 8
    rows = F.pad(x, (0, 0, 0, 0, 0, 0, 0, Cp - Cc)).permute(0, 2, 3, 4, 1).contiguous()
    pl = ops.Planes((B, T, H, W, Cp + coff + 8), bf16, "cuda", lo=True)
    pl.hi.zero_()
    pl.lo.zero_()
    ops.split_into(rows, pl, 0, Cp, None, None, False, out_coff=coff)
    return pl, Cp, coff


def _launch(cv, diag, key):
    from coclr_b200 import lib as L
    lib = L.load()
    kernel = "tma" if lib.coclr_conv_tma_plan(C.byref(cv), (C.c_int * 8)()) else "gather"
    diag["kernel/" + key] = kernel
    assert kernel == "gather", key
    L.check(lib.coclr_conv_igemm(C.byref(cv), L.num_sms(), L.stream_ptr()), "coclr_conv_igemm")


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("bf16", [0, 1])
def test_gather_forward_is_bit_reproducible(case, bf16, diag):
    from coclr_b200 import ops
    name, Cin, Cout, k, s, p, B, T, H, W = case
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.randn(B, Cin, T, H, W, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, *k, device="cuda", generator=g) * 0.05
    geom = ops.Geometry(k, s, p)
    To, Ho, Wo = geom.out_dims(T, H, W)
    pl, Cp, coff = _planes(ops, x, bf16)
    pw = ops.PackedWeights(Cout, Cin, geom.taps, Cp, 0, bf16, "cuda").pack(w.contiguous())
    outs = []
    for run in range(2):
        dst = torch.full((B, To, Ho, Wo, Cout + 40), -3.0, device="cuda")
        stats = torch.zeros(2 * Cout, dtype=torch.float64, device="cuda")
        _launch(ops.make_conv(pl.src(coff, Cp, T, H, W), bf16, geom.c(0), B, (To, Ho, Wo), pw, dst, 32,
                              stats_sum=stats[:Cout], stats_sq=stats[Cout:], npass=3), diag, "repro/%s/%d" % (name, run))
        torch.cuda.synchronize()
        outs.append((dst, stats))
    (d0, s0), (d1, s1) = outs
    assert torch.equal(d0, d1), name
    assert torch.equal(s0, s1), name
    # and the launch computed the convolution and its statistics
    ref = F.conv3d(x.double(), w.double(), stride=s, padding=p).permute(0, 2, 3, 4, 1)
    got = d0[..., 32:32 + Cout].double()
    err = float((got - ref).abs().max() / ref.abs().max())
    diag["repro/%s/bf%d" % (name, bf16)] = err
    assert err < (2e-5 if not bf16 else 2e-4)
    for st, ex in ((s0[:Cout], got.sum(dim=(0, 1, 2, 3))), (s0[Cout:], (got ** 2).sum(dim=(0, 1, 2, 3)))):
        assert float((st - ex).abs().max() / ex.abs().max()) < 1e-5, name


def test_gather_dgrad_accumulate_is_bit_reproducible(diag):
    """dX += the data gradient of a stride-2 1x1x1 conv over odd frames, into a channel slice of a wider buffer."""
    from coclr_b200 import ops
    Cin, Cout, k, s, p, B, T, H, W = 64, 256, (1, 1, 1), (1, 2, 2), (0, 0, 0), 1, 2, 7, 9
    g = torch.Generator(device="cuda").manual_seed(13)
    w = torch.randn(Cout, Cin, *k, device="cuda", generator=g) * 0.05
    geom = ops.Geometry(k, s, p)
    To, Ho, Wo = geom.out_dims(T, H, W)
    dy = torch.randn(B, Cout, To, Ho, Wo, device="cuda", generator=g)
    pl, Cop, coff = _planes(ops, dy, 1)
    pw = ops.PackedWeights(Cout, Cin, geom.taps, Cop, 1, 1, "cuda").pack(w.contiguous())
    base = torch.randn(B, T, H, W, Cin + 16, device="cuda", generator=g)
    outs = []
    for run in range(2):
        dst = base.clone()
        _launch(ops.make_conv(pl.src(coff, Cop, To, Ho, Wo), 1, geom.c(1), B, (T, H, W), pw, dst, 8, accumulate=True,
                              npass=3), diag, "repro/dgrad_acc/%d" % run)
        torch.cuda.synchronize()
        outs.append(dst)
    assert torch.equal(outs[0], outs[1])
    assert torch.equal(outs[0][..., :8], base[..., :8]) and torch.equal(outs[0][..., 8 + Cin:], base[..., 8 + Cin:])
