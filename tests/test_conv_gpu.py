"""GPU parity of the wgmma implicit-GEMM convolution (forward, dgrad, wgrad), the BatchNorm-apply/ReLU/split
kernel that feeds it, and max-pooling, against torch.nn.functional evaluated in float64 -- the ops the reference
reaches through nn.Conv3d / nn.BatchNorm3d / nn.MaxPool3d (backbone/s3dg.py:11-17,39-48,105).  Tolerances:
3-pass fp16 split precision must be fp32-grade (2e-5 of the output scale), 3-pass bf16 2e-4; the single-pass
mode is only checked for sanity (3e-2).  Every launch records in `diag` which kernel took it (TMA-staged or cp.async
gather); the float64 checks hold whichever it is."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# (name, Cin, Cout, k, s, p, B, T, H, W)
CASES = [
    ("pw_64_64", 64, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 4, 8, 8),
    ("pw_192_96_ragged", 192, 96, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1, 3, 5, 7),
    ("pw_832_384", 832, 384, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 2, 4, 4),
    ("pw_480_16", 480, 16, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 2, 8, 8),
    ("sp_64_192", 64, 192, (1, 3, 3), (1, 1, 1), (0, 1, 1), 2, 2, 16, 16),
    ("sp_24_64", 24, 64, (1, 3, 3), (1, 1, 1), (0, 1, 1), 2, 4, 8, 8),
    ("sp_144_288", 144, 288, (1, 3, 3), (1, 1, 1), (0, 1, 1), 1, 4, 8, 8),
    ("tm_192_192", 192, 192, (3, 1, 1), (1, 1, 1), (1, 0, 0), 2, 8, 8, 8),
    ("tm_48_48", 48, 48, (3, 1, 1), (1, 1, 1), (1, 0, 0), 2, 4, 6, 6),
    ("stem_sp", 3, 64, (1, 7, 7), (1, 2, 2), (0, 3, 3), 2, 2, 32, 32),
    ("stem_tm", 64, 64, (7, 1, 1), (2, 1, 1), (3, 0, 0), 1, 8, 16, 16),
    # ResNet2d3d-50 bottlenecks (backbone/resnet_2d3d.py:46-131): the spatially strided conv2 and downsample.0, whose
    # data gradient takes the frame-parity branch of the gather kernel, and the 1024- to 2048-channel layers, whose
    # BatchNorm statistics are flushed after every N tile (n_tiles * BN > 512)
    ("r50_conv2_s2", 128, 128, (1, 3, 3), (1, 2, 2), (0, 1, 1), 2, 2, 16, 16),
    ("r50_conv2_s2_odd", 64, 96, (1, 3, 3), (1, 2, 2), (0, 1, 1), 1, 3, 9, 7),    # edge rows / columns: some taps only
    ("r50_conv2_s2_4to2", 512, 512, (1, 3, 3), (1, 2, 2), (0, 1, 1), 2, 2, 4, 4),   # layer4: 4x4 -> 2x2 frames
    ("r50_ds_s2", 256, 512, (1, 1, 1), (1, 2, 2), (0, 0, 0), 2, 2, 16, 16),
    ("r50_ds_s2_odd", 64, 256, (1, 1, 1), (1, 2, 2), (0, 0, 0), 1, 2, 7, 9),      # half the dX pixels get no gradient
    ("r50_ds_s2_wide", 1024, 2048, (1, 1, 1), (1, 2, 2), (0, 0, 0), 2, 4, 24, 24),  # 144 tiles: CTAs flush several
    ("r50_conv3_wide", 512, 2048, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 2, 2, 2),
    ("r50_conv1_3d", 1024, 512, (3, 1, 1), (1, 1, 1), (1, 0, 0), 2, 4, 4, 4),    # Bottleneck3d conv1
]
# the RGB stem conv has no data gradient (its input is the clip)
DGRAD_CASES = [c for c in CASES if c[0] != "stem_sp"]


def _conv_run(cv, diag, key):
    """Launch one coclr_conv_t and record which kernel takes it."""
    from coclr_b200 import lib as L
    lib = L.load()
    diag["kernel/" + key] = "tma" if lib.coclr_conv_tma_plan(C.byref(cv), (C.c_int * 8)()) else "gather"
    L.check(lib.coclr_conv_igemm(C.byref(cv), L.num_sms(), L.stream_ptr()), "coclr_conv_igemm")


def _wgrad_kernel(src, geom_c, dy_src, B, dst_dims, Cout, Cin_real, npass, bf16):
    """Which kernel ops.conv_wgrad (which passes a large enough workspace) runs these operands on."""
    from coclr_b200 import lib as L
    wg = L.Wgrad(src, geom_c, dy_src, B, *dst_dims, Cout, Cin_real, None, npass, bf16, bf16, 1, None)
    return "tma" if L.load().coclr_wgrad_tma_plan(C.byref(wg), None) else "gather"


def _r8(c):
    return (c + 7) // 8 * 8


def _rows(x, ld=None, coff=0):
    """NCDHW -> channels-last fp32 rows [B,T,H,W,ld] with the tensor's channels at [coff, coff+C)."""
    B, Cc, T, H, W = x.shape
    ld = ld or Cc
    out = torch.full((B, T, H, W, ld), 7.0, dtype=torch.float32, device=x.device)  # poison unused channels
    out[..., coff:coff + Cc] = x.permute(0, 2, 3, 4, 1)
    return out.contiguous()


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def _dump(name, got, ref):
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    os.makedirs(out, exist_ok=True)
    if got.numel() <= 2_000_000:
        np.save(os.path.join(out, "fail_%s_got.npy" % name), got.detach().float().cpu().numpy())
        np.save(os.path.join(out, "fail_%s_ref.npy" % name), ref.detach().float().cpu().numpy())


def _setup(case, seed=0):
    from coclr_b200 import ops
    name, Cin, Cout, k, s, p, B, T, H, W = case
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, Cin, T, H, W, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, *k, device="cuda", generator=g) * 0.05
    geom = ops.Geometry(k, s, p)
    return ops, geom, x, w


def _planes_of(ops, x_ncdhw, bf16, scale=None, shift=None, relu=False, ld_extra=8, coff=8, lo=True, twin=False):
    """Run the split kernel: NCDHW fp32 -> hi/lo planes with the channels at [coff, coff+Cp) of a wider buffer."""
    B, Cc, T, H, W = x_ncdhw.shape
    Cp = _r8(Cc)
    rows = _rows(F.pad(x_ncdhw, (0, 0, 0, 0, 0, 0, 0, Cp - Cc)))
    pl = ops.Planes((B, T, H, W, Cp + coff + ld_extra), bf16, "cuda", lo=lo)
    pl.hi.fill_(3.0)
    if lo:
        pl.lo.fill_(3.0)
    sc = F.pad(scale, (0, Cp - Cc)).contiguous() if scale is not None else None
    sh = F.pad(shift, (0, Cp - Cc)).contiguous() if shift is not None else None
    tw = ops.Planes((B, T, H, W, Cp + coff + ld_extra), 1, "cuda", lo=lo) if twin else None
    ops.split_into(rows, pl, 0, Cp, sc, sh, relu, out_coff=coff, twin=tw)
    if twin:
        return pl, Cp, coff, tw
    return pl, Cp, coff


@pytest.mark.parametrize("bf16", [0, 1])
def test_affine_split(bf16, diag):
    from coclr_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(2, 24, 3, 5, 7, device="cuda", generator=g) * 3
    scale = torch.rand(24, device="cuda", generator=g) + 0.5
    shift = torch.randn(24, device="cuda", generator=g)
    pl, Cp, coff = _planes_of(ops, x, bf16, scale, shift, True)
    torch.cuda.synchronize()
    ref = torch.relu(x * scale.view(1, -1, 1, 1, 1) + shift.view(1, -1, 1, 1, 1)).permute(0, 2, 3, 4, 1)
    got = pl.value()[..., coff:coff + 24]
    err = _rel(got, ref)
    diag["split/bf%d" % bf16] = err
    assert err < (2e-6 if not bf16 else 2e-5)
    assert float((pl.hi[..., :coff].float() - 3).abs().max()) == 0.0   # neighbours untouched


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("npass,bf16", [(3, 0), (3, 1), (1, 1)])
def test_conv_forward(case, npass, bf16, diag):
    ops, geom, x, w = _setup(case)
    name, Cin, Cout, k, s, p, B, T, H, W = case
    To, Ho, Wo = geom.out_dims(T, H, W)
    g = torch.Generator(device="cuda").manual_seed(1)
    scale = torch.rand(Cin, device="cuda", generator=g) + 0.5
    shift = torch.randn(Cin, device="cuda", generator=g) * 0.3
    xin = torch.relu(x * scale.view(1, -1, 1, 1, 1) + shift.view(1, -1, 1, 1, 1))
    ref = F.conv3d(xin.double(), w.double(), stride=s, padding=p)
    pl, Cp, coff = _planes_of(ops, x, bf16, scale, shift, True, lo=(npass > 1))
    pw = ops.PackedWeights(Cout, Cin, geom.taps, Cp, 0, bf16, "cuda").pack(w.contiguous())
    ld_out = Cout + 40
    dst = torch.full((B, To, Ho, Wo, ld_out), -3.0, device="cuda")
    stats = torch.zeros(2 * Cout, dtype=torch.float64, device="cuda")
    _conv_run(ops.make_conv(pl.src(coff, Cp, T, H, W), bf16, geom.c(0), B, (To, Ho, Wo), pw, dst, 32,
                            stats_sum=stats[:Cout], stats_sq=stats[Cout:], npass=npass),
              diag, "fwd/%s/p%d" % (name, npass))
    torch.cuda.synchronize()
    got = dst[..., 32:32 + Cout].permute(0, 4, 1, 2, 3)
    err = _rel(got, ref)
    tol = 2e-5 if npass == 3 and not bf16 else (2e-4 if npass == 3 else 3e-2)
    diag["fwd/%s/p%d_bf%d" % (name, npass, bf16)] = err
    if not err < tol:
        _dump("fwd_%s_p%d_bf%d" % (name, npass, bf16), got, ref)
    assert err < tol, "forward %s rel err %.3e" % (name, err)
    assert float((dst[..., :32] + 3.0).abs().max()) == 0.0
    assert float((dst[..., 32 + Cout:] + 3.0).abs().max()) == 0.0
    s1 = got.double().sum(dim=(0, 2, 3, 4))
    s2 = (got.double() ** 2).sum(dim=(0, 2, 3, 4))
    e1 = float((stats[:Cout] - s1).abs().max() / s1.abs().max().clamp_min(1e-30))
    e2 = float((stats[Cout:] - s2).abs().max() / s2.abs().max().clamp_min(1e-30))
    diag["fwd_stats/%s/p%d_bf%d" % (name, npass, bf16)] = max(e1, e2)
    assert e1 < 1e-5 and e2 < 1e-5


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv_accumulate(case, diag):
    """dst += result (bf16 planes x bf16 weights; wgmma needs one format for both operands)."""
    ops, geom, x, w = _setup(case, seed=3)
    name, Cin, Cout, k, s, p, B, T, H, W = case
    To, Ho, Wo = geom.out_dims(T, H, W)
    ref = F.conv3d(x.double(), w.double(), stride=s, padding=p)
    pl, Cp, coff = _planes_of(ops, x, 1)
    pw = ops.PackedWeights(Cout, Cin, geom.taps, Cp, 0, 1, "cuda").pack(w.contiguous())
    base = torch.randn(B, To, Ho, Wo, Cout, device="cuda")
    dst = base.clone()
    _conv_run(ops.make_conv(pl.src(coff, Cp, T, H, W), 1, geom.c(0), B, (To, Ho, Wo), pw, dst, accumulate=True, npass=3),
              diag, "acc/%s" % name)
    torch.cuda.synchronize()
    got = (dst - base).permute(0, 4, 1, 2, 3)
    err = _rel(got, ref)
    diag["acc/%s" % name] = err
    assert err < 2e-4


@pytest.mark.parametrize("case", DGRAD_CASES, ids=[c[0] for c in DGRAD_CASES])
@pytest.mark.parametrize("npass", [3, 1])
def test_conv_dgrad(case, npass, diag):
    ops, geom, x, w = _setup(case, seed=5)
    name, Cin, Cout, k, s, p, B, T, H, W = case
    To, Ho, Wo = geom.out_dims(T, H, W)
    g = torch.Generator(device="cuda").manual_seed(7)
    dy = torch.randn(B, Cout, To, Ho, Wo, device="cuda", generator=g)
    xd = x.double().requires_grad_(True)
    y = F.conv3d(xd, w.double(), stride=s, padding=p)
    (ref,) = torch.autograd.grad(y, xd, dy.double())
    pl, Cop, coff = _planes_of(ops, dy, 1, lo=(npass > 1))
    pw = ops.PackedWeights(Cout, Cin, geom.taps, Cop, 1, 1, "cuda").pack(w.contiguous())
    dst = torch.zeros(B, T, H, W, Cin, device="cuda")
    _conv_run(ops.make_conv(pl.src(coff, Cop, To, Ho, Wo), 1, geom.c(1), B, (T, H, W), pw, dst, npass=npass),
              diag, "dgrad/%s/p%d" % (name, npass))
    torch.cuda.synchronize()
    got = dst.permute(0, 4, 1, 2, 3)
    err = _rel(got, ref)
    diag["dgrad/%s/p%d" % (name, npass)] = err
    tol = 2e-4 if npass == 3 else 3e-2
    if not err < tol:
        _dump("dgrad_%s_p%d" % (name, npass), got, ref)
    assert err < tol


def test_conv_dgrad_accumulate(diag):
    """dX += the data gradient of a spatially strided conv, into a channel slice of a wider buffer: the input of a
    bottleneck with a downsample branch receives the gradients of conv1 and of downsample.0.  The pixels of odd rows and
    columns receive nothing from the stride-2 1x1x1 conv and must keep what they hold."""
    case = next(c for c in CASES if c[0] == "r50_ds_s2_odd")
    ops, geom, x, w = _setup(case, seed=15)
    name, Cin, Cout, k, s, p, B, T, H, W = case
    To, Ho, Wo = geom.out_dims(T, H, W)
    g = torch.Generator(device="cuda").manual_seed(17)
    dy = torch.randn(B, Cout, To, Ho, Wo, device="cuda", generator=g)
    xd = x.double().requires_grad_(True)
    (ref,) = torch.autograd.grad(F.conv3d(xd, w.double(), stride=s, padding=p), xd, dy.double())
    pl, Cop, coff = _planes_of(ops, dy, 1)
    pw = ops.PackedWeights(Cout, Cin, geom.taps, Cop, 1, 1, "cuda").pack(w.contiguous())
    base = torch.randn(B, T, H, W, Cin + 16, device="cuda", generator=g)
    dst = base.clone()
    _conv_run(ops.make_conv(pl.src(coff, Cop, To, Ho, Wo), 1, geom.c(1), B, (T, H, W), pw, dst, 8, accumulate=True,
                            npass=3), diag, "dgrad_acc/%s" % name)
    torch.cuda.synchronize()
    got = (dst[..., 8:8 + Cin].double() - base[..., 8:8 + Cin].double()).permute(0, 4, 1, 2, 3)
    err = _rel(got, ref)
    diag["dgrad_acc/%s" % name] = err
    assert torch.equal(dst[..., :8], base[..., :8]) and torch.equal(dst[..., 8 + Cin:], base[..., 8 + Cin:])
    assert torch.equal(dst[:, :, 1::2], base[:, :, 1::2]) and torch.equal(dst[:, :, :, 1::2], base[:, :, :, 1::2])
    assert err < 2e-4


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("npass,splits", [(3, 1), (3, 5), (1, 2)])
def test_conv_wgrad(case, npass, splits, diag):
    """dY as bf16 planes x the bf16 twin of the activation planes, no out_scale.  The training step's backbone runs its
    weight gradients on fp16 planes of dY * s with out_scale = 1/s instead: test_wgrad_tma_gpu.py and
    test_conv_bwd_scaled_gpu.py test that format."""
    ops, geom, x, w = _setup(case, seed=9)
    name, Cin, Cout, k, s, p, B, T, H, W = case
    To, Ho, Wo = geom.out_dims(T, H, W)
    g = torch.Generator(device="cuda").manual_seed(11)
    dy = torch.randn(B, Cout, To, Ho, Wo, device="cuda", generator=g)
    scale = torch.rand(Cin, device="cuda", generator=g) + 0.5
    shift = torch.randn(Cin, device="cuda", generator=g) * 0.3
    xin = torch.relu(x * scale.view(1, -1, 1, 1, 1) + shift.view(1, -1, 1, 1, 1)).double()
    wd = w.double().requires_grad_(True)
    y = F.conv3d(xin, wd, stride=s, padding=p)
    (ref,) = torch.autograd.grad(y, wd, dy.double())
    _, Cp, coff, pl = _planes_of(ops, x, 0, scale, shift, True, lo=(npass > 1), twin=True)
    dpl, Cop, dcoff = _planes_of(ops, dy, 1, lo=(npass > 1))
    dw = torch.zeros_like(w)
    src, dsrc = pl.src(coff, Cp, T, H, W), dpl.src(dcoff, Cop, To, Ho, Wo)
    diag["kernel/wgrad/%s/p%d" % (name, npass)] = _wgrad_kernel(src, geom.c(0), dsrc, B, (To, Ho, Wo), Cout, Cin, npass, 1)
    ops.conv_wgrad(src, 1, geom.c(0), dsrc, 1, B, (To, Ho, Wo), Cout, Cin, dw, npass=npass, splits=splits)
    torch.cuda.synchronize()
    err = _rel(dw, ref)
    diag["wgrad/%s/p%d_s%d" % (name, npass, splits)] = err
    tol = 2e-4 if npass == 3 else 3e-2
    if not err < tol:
        _dump("wgrad_%s_p%d_s%d" % (name, npass, splits), dw.reshape(Cout, -1), ref.reshape(Cout, -1))
    assert err < tol


@pytest.mark.parametrize("T", [4, 5], ids=["T_even", "T_odd"])
@pytest.mark.parametrize("npass,bf16", [(3, 0), (1, 1)])
def test_r50_stem_space_to_depth(npass, bf16, T, diag):
    """The ResNet2d3d-50 stem (backbone/resnet_2d3d.py:138: (5,7,7) conv, stride (2,2,2), padding (2,3,3)) as the engine
    launches it: a (5,4,4) conv with stride (2,1,1) and padding (2,2,0) over the space-to-depth planes (16 channels per
    pixel, 12 real; rows zero-padded by 2 pixels on each side, engine.S2D_PAD).  Forward with BatchNorm statistics, and
    the weight gradient in the (5,4,4) layout the engine scatters back to the (5,7,7) weight.  Truth: the same
    effective conv in float64, cropped to the H/2 x W/2 destination pixels."""
    from coclr_b200 import ops
    B, H2, W2, Cout = 2, 8, 12, 64
    g = torch.Generator(device="cuda").manual_seed(53 + T)
    x = torch.randn(B, 16, T, H2, W2, device="cuda", generator=g)
    x[:, 12:] = 0.0                                           # 4*Cin = 12 real channels
    w = torch.randn(Cout, 16, 5, 4, 4, device="cuda", generator=g) * 0.05
    geom = ops.Geometry((5, 4, 4), (2, 1, 1), (2, 2, 0))
    To = geom.out_dims(T, H2, W2)[0]
    ref = F.conv3d(x.double(), w.double(), stride=(2, 1, 1), padding=(2, 2, 2))[..., :H2, :W2]
    pl, Cp, coff = _planes_of(ops, F.pad(x, (2, 2)), bf16, ld_extra=0, coff=0, lo=(npass > 1))
    src = pl.src(0, 16, T, H2, W2 + 4)
    pw = ops.PackedWeights(Cout, 16, geom.taps, 16, 0, bf16, "cuda").pack(w.contiguous())
    dst = torch.full((B, To, H2, W2, Cout), -3.0, device="cuda")
    stats = torch.zeros(2 * Cout, dtype=torch.float64, device="cuda")
    _conv_run(ops.make_conv(src, bf16, geom.c(0), B, (To, H2, W2), pw, dst, 0, stats_sum=stats[:Cout],
                            stats_sq=stats[Cout:], npass=npass), diag, "fwd/r50_stem_T%d/p%d" % (T, npass))
    torch.cuda.synchronize()
    got = dst.permute(0, 4, 1, 2, 3)
    err = _rel(got, ref)
    s1 = got.double().sum(dim=(0, 2, 3, 4))
    s2 = (got.double() ** 2).sum(dim=(0, 2, 3, 4))
    e1 = float((stats[:Cout] - s1).abs().max() / s1.abs().max())
    e2 = float((stats[Cout:] - s2).abs().max() / s2.abs().max())
    # weight gradient against float64 autograd on the exact plane values
    dy = torch.randn(B, Cout, To, H2, W2, device="cuda", generator=g)
    dpl, Cop, dcoff = _planes_of(ops, dy, bf16, lo=(npass > 1))
    dsrc = dpl.src(dcoff, Cop, To, H2, W2)
    xv = pl.value()[..., :12].permute(0, 4, 1, 2, 3).double()              # [B, 12, T, H2, W2 + 4]
    dv = dpl.value()[..., dcoff:dcoff + Cout].permute(0, 4, 1, 2, 3).double()
    wd = torch.zeros(Cout, 12, 5, 4, 4, device="cuda", dtype=torch.float64, requires_grad=True)
    (ref_dw,) = torch.autograd.grad(F.conv3d(xv, wd, stride=(2, 1, 1), padding=(2, 2, 0))[..., :H2, :W2], wd, dv)
    dw = torch.zeros(Cout, 12, 5, 4, 4, device="cuda")
    diag["kernel/wgrad/r50_stem_T%d/p%d" % (T, npass)] = _wgrad_kernel(src, geom.c(0), dsrc, B, (To, H2, W2), Cout, 12,
                                                                        npass, bf16)
    ops.conv_wgrad(src, bf16, geom.c(0), dsrc, bf16, B, (To, H2, W2), Cout, 12, dw, npass=npass)
    torch.cuda.synchronize()
    e_w = _rel(dw, ref_dw)
    diag["r50_stem/T%d/p%d_bf%d" % (T, npass, bf16)] = [err, max(e1, e2), e_w]
    assert err < (2e-5 if npass == 3 else 3e-2), "forward rel err %.3e" % err
    assert e1 < 1e-5 and e2 < 1e-5, (e1, e2)
    assert e_w < (2e-5 if npass == 3 else 3e-2), "weight gradient rel err %.3e" % e_w


POOLS = [((1, 3, 3), (1, 2, 2), (0, 1, 1)), ((3, 3, 3), (1, 1, 1), (1, 1, 1)), ((3, 3, 3), (2, 2, 2), (1, 1, 1)),
         ((2, 2, 2), (2, 2, 2), (0, 0, 0)), ((1, 2, 3), (1, 1, 2), (0, 1, 1))]


@pytest.mark.parametrize("acc", [1, 0], ids=["accumulate", "overwrite"])
@pytest.mark.parametrize("dims,Cc", [((6, 9, 10), 24), ((4, 8, 12), 24), ((5, 16, 16), 32), ((3, 12, 8), 48), ((2, 64, 64), 16)],
                         ids=["ragged", "x4", "smem16", "smem8_raggedH", "smem64"])
@pytest.mark.parametrize("k,s,p", POOLS, ids=["133s2", "333s1", "333s2", "222s2", "generic"])
def test_maxpool_fwd_bwd(k, s, p, dims, Cc, acc, diag):
    """The 16-channel-multiple cases on 8/16/64-wide frames take the shared-memory kernels (3x3x3/s1 rolling frame ring,
    (1,3,3)/s2 tile); the others the register-only kernels."""
    import ctypes as C
    from coclr_b200 import ops, lib as L
    g = torch.Generator(device="cuda").manual_seed(13)
    B = 2
    T, H, W = dims
    x = torch.randn(B, Cc, T, H, W, device="cuda", generator=g)
    x = torch.relu(x)                     # post-ReLU inputs as in the network: many exact ties at 0
    pl, Cp, coff = _planes_of(ops, x, 0) if acc else _planes_of(ops, x, 0, ld_extra=0, coff=0)
    xv = pl.value()[..., coff:coff + Cc].permute(0, 4, 1, 2, 3).double().requires_grad_(True)   # exact plane values
    ref = F.max_pool3d(xv, k, s, p)
    geom = ops.Geometry(k, s, p)
    To, Ho, Wo = geom.out_dims(T, H, W)
    out = ops.Planes((B, To, Ho, Wo, Cp), 0, "cuda")
    idx = torch.empty(B * To * Ho * Wo * Cp, dtype=torch.uint8, device="cuda")
    dyt = torch.randn(B, To, Ho, Wo, Cp, device="cuda", generator=g)
    dx = torch.full((B, T, H, W, pl.ld), 0.5, device="cuda")
    tw = ops.Planes((B, To, Ho, Wo, Cp), 1, "cuda")
    pp = L.Pool(L.dptr(pl.hi), L.dptr(pl.lo), pl.ld, coff, L.dptr(out.hi), L.dptr(out.lo), Cp, 0,
                L.dptr(tw.hi), L.dptr(tw.lo), L.dptr(idx),
                B, Cp, T, H, W, To, Ho, Wo, geom.c(0), L.dptr(dyt), L.dptr(dx), acc)
    L.check(L.load().coclr_maxpool_fwd(C.byref(pp), L.stream_ptr()), "coclr_maxpool_fwd")
    L.check(L.load().coclr_maxpool_bwd(C.byref(pp), L.stream_ptr()), "coclr_maxpool_bwd")
    torch.cuda.synchronize()
    got = out.value()[..., :Cc].permute(0, 4, 1, 2, 3)
    assert torch.equal(got.double(), ref.detach())
    assert _rel(tw.value()[..., :Cc].permute(0, 4, 1, 2, 3), ref.detach()) < 2e-5
    (gref,) = torch.autograd.grad(ref, xv, dyt[..., :Cc].permute(0, 4, 1, 2, 3).double())
    gdx = (dx[..., coff:coff + Cc] - (0.5 if acc else 0.0)).permute(0, 4, 1, 2, 3)
    e = _rel(gdx, gref)
    diag["pool/%s" % (str(k) + str(s))] = e
    assert e < 1e-6


@pytest.mark.parametrize("Cc,res,relu", [(48, None, 1), (2048, "fp16", 1), (2048, "bf16", 1), (2048, None, 0)],
                         ids=["C48", "C2048_res_fp16", "C2048_res_bf16", "C2048_linear"])
@pytest.mark.parametrize("training", [1, 0])
def test_fused_bn_finalize_apply_split(training, Cc, res, relu, diag):
    """coclr_affine_split with the BatchNorm finalize fused in, against F.batch_norm (+ residual) (+ relu) in float64
    (train and eval mode, running-stat update included) -- nn.BatchNorm3d semantics of backbone/s3dg.py:16.  C = 2048
    fills the kernel's shared-memory scale table; the residual (a bottleneck's relu(bn3(y) + r), backbone/resnet_2d3d.py:
    118-123) comes from planes of the output's 16-bit format; relu = 0 is the downsample BatchNorm."""
    from coclr_b200 import ops, lib as L
    g = torch.Generator(device="cuda").manual_seed(21)
    B, T, H, W = (2, 3, 6, 5) if Cc == 48 else (2, 2, 3, 2)
    bf16 = int(res == "bf16")
    x = torch.randn(B, Cc, T, H, W, device="cuda", generator=g) * 2 + 0.5
    gamma = torch.rand(Cc, device="cuda", generator=g) + 0.5
    beta = torch.randn(Cc, device="cuda", generator=g)
    rm = torch.randn(Cc, device="cuda", generator=g) * 0.1
    rv = torch.rand(Cc, device="cuda", generator=g) + 0.5
    rm_ref, rv_ref = rm.double(), rv.double()
    ref = F.batch_norm(x.double(), rm_ref, rv_ref, gamma.double(), beta.double(), bool(training), 0.1, 1e-5)
    rpl, rcoff = None, 0
    if res is not None:
        rpl, _, rcoff = _planes_of(ops, torch.randn(B, Cc, T, H, W, device="cuda", generator=g), bf16)
        ref = ref + rpl.value()[..., rcoff:rcoff + Cc].permute(0, 4, 1, 2, 3).double()    # exact plane values
    if relu:
        ref = torch.relu(ref)
    ref = ref.permute(0, 2, 3, 4, 1)
    rows = _rows(x)
    M = rows.numel() // Cc
    xs = rows.double().reshape(M, Cc)
    ssum, ssq = xs.sum(0).contiguous(), (xs * xs).sum(0).contiguous()
    scale, shift, mean, rstd = (torch.zeros(Cc, device="cuda") for _ in range(4))
    pl = ops.Planes((B, T, H, W, Cc), bf16, "cuda")
    bn = L.BnFinalize(L.dptr(ssum), L.dptr(ssq), M, L.dptr(gamma), L.dptr(beta), L.dptr(rm), L.dptr(rv), 0.1, 1e-5,
                      training, L.dptr(scale), L.dptr(shift), L.dptr(mean), L.dptr(rstd), Cc)
    sp = L.Split(L.dptr(rows), Cc, 0, Cc, M, None, None, relu, L.dptr(pl.hi), L.dptr(pl.lo), Cc, 0, bf16, None, None, bn,
                 L.dptr(rpl.hi) if rpl else None, L.dptr(rpl.lo) if rpl else None, rpl.ld if rpl else 0, rcoff)
    lib = L.load()
    L.check(lib.coclr_affine_split(C.byref(sp), L.num_sms(), L.stream_ptr()), "coclr_affine_split")
    torch.cuda.synchronize()
    e = _rel(pl.value(), ref)
    diag["fused_bn/train%d_C%d_%s_relu%d" % (training, Cc, res, relu)] = e
    assert e < (2e-5 if bf16 else 5e-6)
    assert _rel(rm, rm_ref) < 1e-6 and _rel(rv, rv_ref) < 1e-6
    if training:
        assert _rel(mean, xs.mean(0)) < 1e-6
    if Cc == 2048:   # wider than the kernel's shared-memory scale table; refused before any launch
        sp.C = sp.bn.C = sp.ld = sp.out_ld = 2056
        assert lib.coclr_affine_split(C.byref(sp), L.num_sms(), L.stream_ptr()) == -1    # COCLR_E_ARG


def _clear_of_kink(y, gamma, beta, r=None, gap=1e-3):
    """Move the elements of y [M, C] whose ReLU input bn(y) (+ r) lies within `gap` of 0 to about 2 gap on their side
    of it (the batch statistics shift a little with them, hence the loop): the kernel's fp32 ReLU mask must agree with
    float64's on every element."""
    for _ in range(20):
        yd = y.double()
        rstd = (yd.var(0, unbiased=False) + 1e-5).rsqrt()
        z = (yd - yd.mean(0)) * rstd * gamma.double() + beta.double()
        if r is not None:
            z = z + r
        near = z.abs() < gap
        if not bool(near.any()):
            return y
        step = torch.where(z < 0, -2.0 * gap, 2.0 * gap) / (gamma.double() * rstd)
        y = torch.where(near, yd + step, yd).float()
    raise AssertionError("ReLU inputs keep landing within %g of 0" % gap)


@pytest.mark.parametrize("fp16", [1, 0], ids=["fp16_scaled", "bf16"])
@pytest.mark.parametrize("C,M,spread", [(64, 4096, 1.0), (24, 777, 1e-4), (192, 2048, 1e3),
                                        (1024, 256, 1.0), (2048, 64, 1.0), (2048, 4096, 10.0)])
@pytest.mark.parametrize("relu", [1, 0], ids=["relu", "linear"])
def test_bn_relu_backward_planes(relu, fp16, C, M, spread, diag):
    """coclr_bn_bwd against autograd of relu(batch_norm(y)) in float64 (NativeBatchNormBackward0 + ReluBackward0 of the
    reference's graph): dgamma / dbeta and the dY operand planes -- bf16 hi/lo, or fp16 hi/lo of dY * s with the
    power-of-two s the kernel derives from the data (dy_scale), for gradient magnitudes from 1e-4 to 1e3 (`spread`)
    and channels of very different scale inside one tensor.  relu = 0 is the downsample BatchNorm of a ResNet
    bottleneck; C = 1024 is one channel tile with one row per pass, C = 2048 two tiles under one dy_scale.  dgamma /
    dbeta are gradient buffers: the kernel adds to what they hold."""
    import ctypes as C_
    from coclr_b200 import ops, lib as L
    g = torch.Generator(device="cuda").manual_seed(C + M)
    y = torch.randn(M, C, device="cuda", generator=g) * 1.5 + 0.3
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5
    beta = torch.randn(C, device="cuda", generator=g) * 0.2
    chan = torch.logspace(-3, 0, C, device="cuda")                      # per-channel gradient magnitudes over 3 decades
    dA = torch.randn(M, C, device="cuda", generator=g) * chan * spread
    if relu:
        y = _clear_of_kink(y, gamma, beta)
    yd = y.double().requires_grad_(True)
    gd, bd = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    out = F.batch_norm(yd, None, None, gd, bd, True, 0.1, 1e-5)
    if relu:
        out = torch.relu(out)
    ref_dy, ref_dg, ref_db = torch.autograd.grad(out, [yd, gd, bd], dA.double())
    mean = y.double().mean(0)
    var = y.double().var(0, unbiased=False)
    rstd = (var + 1e-5).rsqrt()
    scale = (gamma.double() * rstd).float()
    shift = (beta.double() - mean * gamma.double() * rstd).float()
    mean32, rstd32 = mean.float().contiguous(), rstd.float().contiguous()    # keep alive: the kernel gets raw pointers
    sums = torch.zeros(2 * C, dtype=torch.float64, device="cuda")
    amax = torch.zeros(2 * C, device="cuda")
    dscale = torch.ones(2, device="cuda")
    dgam0 = torch.randn(C, device="cuda", generator=g) * float(ref_dg.abs().max())
    dbet0 = torch.randn(C, device="cuda", generator=g) * float(ref_db.abs().max())
    dgam, dbet = dgam0.clone(), dbet0.clone()
    pl = ops.Planes((M, C), 0 if fp16 else 1, "cuda")
    bb = L.BnBwd(L.dptr(y), L.dptr(dA), C, 0, C, M, L.dptr(scale), L.dptr(shift), L.dptr(mean32), L.dptr(rstd32),
                 relu, L.dptr(sums), L.dptr(dgam), L.dptr(dbet), L.dptr(pl.hi), L.dptr(pl.lo),
                 None, None, 0, 0, 0, None, 0, 0, 0, fp16, L.dptr(amax), L.dptr(dscale))
    L.check(L.load().coclr_bn_bwd(C_.byref(bb), L.num_sms(), L.stream_ptr()), "coclr_bn_bwd")
    torch.cuda.synchronize()
    got = pl.value().double() * (float(dscale[1]) if fp16 else 1.0)
    e_dy = _rel(got, ref_dy)
    # per-channel error relative to that channel's own scale: small channels must not drown in the tensor-wide scale
    per_c = ((got - ref_dy).abs().amax(0) / ref_dy.abs().amax(0).clamp_min(1e-300)).max()
    diag["bn_bwd/relu%d_fp16%d_C%d_M%d_s%g" % (relu, fp16, C, M, spread)] = [e_dy, float(per_c), float(dscale[0])]
    assert _rel(dgam.double() - dgam0.double(), ref_dg) < 1e-4 and _rel(dbet.double() - dbet0.double(), ref_db) < 1e-4
    if fp16:
        s = float(dscale[0])
        assert s > 0 and abs(np.log2(s) - round(np.log2(s))) < 1e-6          # a power of two
        top = float(pl.value().abs().max())
        assert 2.0 ** 8 < top <= 2.0 ** 14, top                                # the range bound is not wildly pessimistic
        assert e_dy < 2e-6 and float(per_c) < 2e-5, (e_dy, float(per_c))
    else:
        assert e_dy < 3e-5


@pytest.mark.parametrize("C,M", [(256, 1000), (2048, 200)], ids=["C256", "C2048"])
@pytest.mark.parametrize("dres_acc", [0, 1], ids=["dres_store", "dres_add"])
@pytest.mark.parametrize("res_bf16", [0, 1], ids=["res_fp16", "res_bf16"])
@pytest.mark.parametrize("fp16", [1, 0], ids=["fp16_scaled", "bf16"])
def test_bn_backward_residual(fp16, res_bf16, dres_acc, C, M, diag):
    """coclr_bn_bwd of a bottleneck's output unit relu(bn3(y) + r) (backbone/resnet_2d3d.py:75-80) against float64
    autograd w.r.t. y, gamma, beta and r.  r is read from a channel slice of wider 16-bit planes and enters the ReLU
    mask; dz = dA * [bn(y) + r > 0] is stored or added into a channel slice of a wider fp32 buffer (the gradient of the
    residual branch), whose other channels must keep what they hold.  C = 2048 runs as two channel tiles."""
    import ctypes as C_
    from coclr_b200 import ops, lib as L
    g = torch.Generator(device="cuda").manual_seed(C + M + 2 * res_bf16 + dres_acc)
    y = torch.randn(M, C, device="cuda", generator=g) * 1.5 + 0.3
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5
    beta = torch.randn(C, device="cuda", generator=g) * 0.2
    dA = torch.randn(M, C, device="cuda", generator=g) * torch.logspace(-3, 0, C, device="cuda")
    res, _, rcoff = _planes_of(ops, torch.randn(M, C, device="cuda", generator=g).t().reshape(1, C, M, 1, 1), res_bf16)
    rv = res.value()[..., rcoff:rcoff + C].reshape(M, C).double()        # exact plane values
    y = _clear_of_kink(y, gamma, beta, rv)
    yd, rd = y.double().requires_grad_(True), rv.clone().requires_grad_(True)
    gd, bd = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    out = torch.relu(F.batch_norm(yd, None, None, gd, bd, True, 0.1, 1e-5) + rd)
    ref_dy, ref_dg, ref_db, ref_dr = torch.autograd.grad(out, [yd, gd, bd, rd], dA.double())
    mean = y.double().mean(0)
    rstd = (y.double().var(0, unbiased=False) + 1e-5).rsqrt()
    scale = (gamma.double() * rstd).float()
    shift = (beta.double() - mean * gamma.double() * rstd).float()
    mean32, rstd32 = mean.float().contiguous(), rstd.float().contiguous()
    sums = torch.zeros(2 * C, dtype=torch.float64, device="cuda")
    amax = torch.zeros(2 * C, device="cuda")
    dscale = torch.ones(2, device="cuda")
    dgam, dbet = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    pl = ops.Planes((M, C), 0 if fp16 else 1, "cuda")
    dres_ld, dres_coff = C + 16, 8
    base = torch.randn(M, dres_ld, device="cuda", generator=g)
    dres = base.clone()
    bb = L.BnBwd(L.dptr(y), L.dptr(dA), C, 0, C, M, L.dptr(scale), L.dptr(shift), L.dptr(mean32), L.dptr(rstd32),
                 1, L.dptr(sums), L.dptr(dgam), L.dptr(dbet), L.dptr(pl.hi), L.dptr(pl.lo),
                 L.dptr(res.hi), L.dptr(res.lo), res.ld, rcoff, res_bf16, L.dptr(dres), dres_ld, dres_coff, dres_acc,
                 fp16, L.dptr(amax), L.dptr(dscale))
    lib = L.load()
    L.check(lib.coclr_bn_bwd(C_.byref(bb), L.num_sms(), L.stream_ptr()), "coclr_bn_bwd")
    torch.cuda.synchronize()
    got = pl.value().double() * (float(dscale[1]) if fp16 else 1.0)
    sl = slice(dres_coff, dres_coff + C)
    got_dr = dres[:, sl].double() - (base[:, sl].double() if dres_acc else 0.0)
    e_dy, e_dr, e_dg, e_db = _rel(got, ref_dy), _rel(got_dr, ref_dr), _rel(dgam, ref_dg), _rel(dbet, ref_db)
    diag["bn_bwd_res/fp16%d_res_bf16%d_acc%d_C%d" % (fp16, res_bf16, dres_acc, C)] = [e_dy, e_dr, e_dg, e_db]
    assert torch.equal(dres[:, :dres_coff], base[:, :dres_coff]) and torch.equal(dres[:, sl.stop:], base[:, sl.stop:])
    assert e_dr < 1e-6, e_dr
    assert e_dg < 1e-4 and e_db < 1e-4, (e_dg, e_db)
    assert e_dy < (2e-6 if fp16 else 3e-5), e_dy
    if C == 2048:   # argument checks; the buffers hold 2048 channels, so a call that slipped through stays inside them
        bb.relu = 0         # the residual is added before the ReLU: there is no residual unit without one
        assert lib.coclr_bn_bwd(C_.byref(bb), L.num_sms(), L.stream_ptr()) == -1    # COCLR_E_ARG
        bb.relu, bb.C = 1, 1536     # wider than one 1024-channel tile, but not whole tiles
        assert lib.coclr_bn_bwd(C_.byref(bb), L.num_sms(), L.stream_ptr()) == -1
