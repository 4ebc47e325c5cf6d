"""The backward convolutions in the format the training step runs them in (engine.Plan): the gradient planes are fp16
hi/lo of dY * s with s a power of two chosen from the data (coclr_bn_bwd, dy_fp16 = 1), the data gradient multiplies
them with fp16 mode-1 packed weights, and both the data gradient and the weight gradient receive 1/s as the device
scalar out_scale (&dy_scale[1]).  Every fp16 (pass count, tile width) instance of both convolution kernels (the
TMA-staged one and the cp.async gather one) runs a data gradient here, stored and accumulated into a channel slice of a
wider buffer, with 1/s far from 1 in both directions and per-row weight scales spread over several octaves (so that
the packer's unscale differs from column to column and from one N tile to the next).  Truth: float64 autograd of
torch's conv3d; single-pass launches are also held to the float64 product of their exact operands.  Also: weight
gradients in the same format on every kind (1x1x1, (1,3,3), (3,1,1), the temporally strided and the space-to-depth
stems) and product count of the TMA-staged weight-gradient kernel and on the gather kernel's shapes, the
BatchNorm-backward -> convolution chain as the engine wires it, and the batched weight packer against the per-layer
one."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from test_conv_gpu import _clear_of_kink, _dump, _planes_of, _rel

pytestmark = pytest.mark.gpu

# Data gradients dX[.., Cin] <- dY[.., Cout]: (name, kernel, BN, Cin, Cout, k, s, p, B, T, H, W).  kernel and BN are
# what the planner picks for the fp16 launch (the GEMM N of a data gradient is Cin); test_conv_bwd_scaled_plan_cpu.py
# checks that these reach all four tile widths of both kernels at both pass counts.
DGRAD_CASES = [
    ("tma32_pw_32_64", "tma", 32, 32, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 4, 16, 16),
    ("tma64_sp_64_192", "tma", 64, 64, 192, (1, 3, 3), (1, 1, 1), (0, 1, 1), 2, 2, 16, 16),
    ("tma64_tm_64_64", "tma", 64, 64, 64, (3, 1, 1), (1, 1, 1), (1, 0, 0), 2, 8, 8, 8),
    # the stem's temporally strided conv: frame-parity output tiles on the TMA kernel, zero_chunk_mask on the gather one
    ("tma64_stem_tm", "tma", 64, 64, 64, (7, 1, 1), (2, 1, 1), (3, 0, 0), 2, 8, 16, 16),
    ("tma96_pw_96_64", "tma", 96, 96, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 2, 8, 8),
    ("tma96_pw_192_32", "tma", 96, 192, 32, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 2, 8, 8),          # 2 N tiles
    ("tma96_tm_192_192", "tma", 96, 192, 192, (3, 1, 1), (1, 1, 1), (1, 0, 0), 2, 8, 8, 8),
    ("tma128_pw_128_64", "tma", 128, 128, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 2, 8, 8),
    ("tma128_pw_832_384", "tma", 128, 832, 384, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 2, 4, 4),      # 7 N tiles
    ("g32_sp_32_96", "gather", 32, 32, 96, (1, 3, 3), (1, 1, 1), (0, 1, 1), 2, 2, 16, 16),
    ("g32_tm_32_32", "gather", 32, 32, 32, (3, 1, 1), (1, 1, 1), (1, 0, 0), 2, 8, 16, 16),
    ("g64_sp_48_16", "gather", 64, 48, 16, (1, 3, 3), (1, 1, 1), (0, 1, 1), 2, 4, 8, 8),
    ("g64_tm_48_48", "gather", 64, 48, 48, (3, 1, 1), (1, 1, 1), (1, 0, 0), 2, 8, 8, 8),
    ("g64_r50_conv2_s2_odd", "gather", 64, 64, 96, (1, 3, 3), (1, 2, 2), (0, 1, 1), 1, 3, 9, 7),
    ("g64_r50_ds_s2_odd", "gather", 64, 64, 256, (1, 1, 1), (1, 2, 2), (0, 0, 0), 1, 2, 7, 9),
    ("g96_tm_96_96", "gather", 96, 96, 96, (3, 1, 1), (1, 1, 1), (1, 0, 0), 2, 8, 16, 16),
    ("g128_sp_320_160", "gather", 128, 320, 160, (1, 3, 3), (1, 1, 1), (0, 1, 1), 2, 4, 4, 4),     # 3 N tiles
    ("g128_tm_208_208", "gather", 128, 208, 208, (3, 1, 1), (1, 1, 1), (1, 0, 0), 2, 4, 8, 8),
    ("g128_r50_conv2_s2", "gather", 128, 128, 128, (1, 3, 3), (1, 2, 2), (0, 1, 1), 2, 2, 16, 16),
]
DGRAD_IDS = [c[0] for c in DGRAD_CASES]
# gradient magnitudes: 1/s is about 2^-35 at the small end and 2^9 at the large end
MAGS = [1e-7, 1e-2, 1e6]
DST_COFF, DST_EXTRA = 8, 16     # the data gradient goes to channels [8, 8 + Cin) of a buffer 16 channels wider


def _pow2_scale(t):
    """s = 2^(14 - e), e the frexp exponent of max |t|: the power of two bn_bwd_apply_kernel scales dY by."""
    e = math.frexp(float(t.abs().max()))[1]
    return 2.0 ** (14 - e)


def _row_octaves(Cin, device="cuda"):
    """Per input channel (a row of the mode-1 packed weight) a power of two over 9 octaves, different for neighbouring
    columns and for the columns of different N tiles."""
    return 2.0 ** ((torch.arange(Cin, device=device, dtype=torch.float64) * 5) % 9 - 4)


def _weights(Cout, Cin, k, g, exact):
    """[Cout, Cin, *k] fp32.  exact: 11-bit integers times a per-row power of two, so that the packer's fp16 hi image
    (row scaled to max |w| in [0.5, 1)) is the weight itself and the lo image is zero."""
    oct_ = _row_octaves(Cin).float().view(1, Cin, 1, 1, 1)
    if exact:
        w = torch.randint(-2047, 2048, (Cout, Cin) + tuple(k), device="cuda", generator=g).float() * 2.0 ** -11
    else:
        w = torch.randn(Cout, Cin, *k, device="cuda", generator=g) * 0.05
    return (w * oct_).contiguous()


def dgrad_conv(ops, case, dy_pl, dcoff, pw, dst, npass, bf16, accumulate, out_scale):
    """The coclr_conv_t of one data-gradient launch of `case` (shared with the dry-run plan test)."""
    name, kernel, BN, Cin, Cout, k, s, p, B, T, H, W = case
    geom = ops.Geometry(k, s, p)
    To, Ho, Wo = geom.out_dims(T, H, W)
    Cop = (Cout + 7) // 8 * 8
    return ops.make_conv(dy_pl.src(dcoff, Cop, To, Ho, Wo), bf16, geom.c(1), B, (T, H, W), pw, dst, DST_COFF,
                         accumulate=accumulate, npass=npass, out_scale=out_scale)


def _launch(cv, gather, diag, key):
    """Run one launch on the kernel the planner picks, or on the gather kernel; records which kernel ran it."""
    from coclr_b200 import lib as L
    lib = L.load()
    kernel = "gather" if gather or not lib.coclr_conv_tma_plan(C.byref(cv), None) else "tma"
    diag["kernel/" + key] = kernel
    lib.coclr_set_conv_tma(0 if gather else 1)
    try:
        L.check(lib.coclr_conv_igemm(C.byref(cv), L.num_sms(), L.stream_ptr()), "coclr_conv_igemm")
        torch.cuda.synchronize()
    finally:
        lib.coclr_set_conv_tma(1)
    return kernel


def _idle_pixels(geom, dims):
    """[T, H, W] mask of the input pixels that no output pixel reads (the odd rows and columns of a 1x1x1 stride-2
    conv): they receive no data gradient."""
    out = geom.out_dims(*dims)
    op = tuple(d - ((o - 1) * s - 2 * p + k) for d, o, s, p, k in zip(dims, out, geom.s, geom.p, geom.k))
    cover = F.conv_transpose3d(torch.ones(1, 1, *out, device="cuda", dtype=torch.float64),
                               torch.ones(1, 1, *geom.k, device="cuda", dtype=torch.float64), stride=geom.s,
                               padding=geom.p, output_padding=op)[0, 0]
    return cover == 0


def _dgrad_truth(case, dy64, w64):
    name, kernel, BN, Cin, Cout, k, s, p, B, T, H, W = case
    x = torch.zeros(B, Cin, T, H, W, device="cuda", dtype=torch.float64, requires_grad=True)
    (ref,) = torch.autograd.grad(F.conv3d(x, w64, stride=s, padding=p), x, dy64)
    return ref.permute(0, 2, 3, 4, 1)                     # channels-last, as the kernel writes it


@pytest.mark.parametrize("mag", MAGS)
@pytest.mark.parametrize("npass", [3, 1])
@pytest.mark.parametrize("case", DGRAD_CASES, ids=DGRAD_IDS)
def test_dgrad_fp16_scaled(case, npass, mag, diag):
    """Production format: dY planes = fp16 split of dY * s, out_scale = 1/s on the device, fp16 mode-1 weights.  Each
    of {planner's kernel, gather kernel} x {store, accumulate}."""
    from coclr_b200 import ops
    name, kernel, BN, Cin, Cout, k, s, p, B, T, H, W = case
    geom = ops.Geometry(k, s, p)
    To, Ho, Wo = geom.out_dims(T, H, W)
    g = torch.Generator(device="cuda").manual_seed(1000 + 10 * DGRAD_IDS.index(name) + npass)
    dy = torch.randn(B, Cout, To, Ho, Wo, device="cuda", generator=g) * mag
    w = _weights(Cout, Cin, k, g, exact=(npass == 1))
    sc = _pow2_scale(dy)
    pl, Cop, dcoff = _planes_of(ops, dy * sc, 0, lo=(npass > 1))
    out_scale = torch.tensor([1.0 / sc], device="cuda")
    pw = ops.PackedWeights(Cout, Cin, geom.taps, Cop, 1, 0, "cuda").pack(w)
    assert (pw.BN, pw.bf16) == (BN, 0)
    ref = _dgrad_truth(case, dy.double(), w.double())
    if npass == 1:
        # the single-pass kernel multiplies the hi planes alone; the weight's hi image is exact
        dyh = pl.hi[..., dcoff:dcoff + Cout].double().permute(0, 4, 1, 2, 3) / sc
        ref_ops = _dgrad_truth(case, dyh, w.double())
    top = float(ref.abs().max())
    ld = Cin + DST_EXTRA
    gb = torch.Generator(device="cuda").manual_seed(7)
    base = torch.randn(B, T, H, W, ld, device="cuda", generator=gb) * top   # of the gradient's magnitude
    sl = slice(DST_COFF, DST_COFF + Cin)
    idle = _idle_pixels(geom, (T, H, W))
    for gather in (False, True):
        for acc in (False, True):
            key = "dgrad_fp16/%s/p%d/m%g/%s/%s" % (name, npass, mag, "gather" if gather else "plan",
                                                   "acc" if acc else "store")
            dst = base.clone() if acc else torch.full((B, T, H, W, ld), 1e30, device="cuda")    # store: poisoned
            ran = _launch(dgrad_conv(ops, case, pl, dcoff, pw, dst, npass, 0, acc, out_scale), gather, diag, key)
            assert ran == ("gather" if gather else kernel), (key, ran)
            got = dst[..., sl].double() - (base[..., sl].double() if acc else 0.0)
            err = _rel(got, ref)
            errs = [err]
            if npass == 1:
                errs.append(_rel(got, ref_ops))
            diag[key] = errs
            nb = base if acc else torch.full_like(base, 1e30)
            assert torch.equal(dst[..., :DST_COFF], nb[..., :DST_COFF]), key + ": channels below the slice changed"
            assert torch.equal(dst[..., sl.stop:], nb[..., sl.stop:]), key + ": channels above the slice changed"
            if acc and bool(idle.any()):
                assert torch.equal(dst[:, idle], base[:, idle]), key + ": pixels without a gradient changed"
            tol = 2e-5 if npass == 3 else 3e-3
            if not (err < tol and (npass == 3 or errs[1] < 2e-5)):
                _dump(key.replace("/", "_"), got, ref)
            assert err < tol, (key, errs)
            if npass == 1:
                assert errs[1] < 2e-5, (key, "vs the product of the exact operands", errs)


@pytest.mark.parametrize("case", DGRAD_CASES, ids=DGRAD_IDS)
def test_dgrad_bf16_control(case, diag):
    """The same launches in the bf16 format (the projection head's), 3 passes, no out_scale."""
    from coclr_b200 import ops
    name, kernel, BN, Cin, Cout, k, s, p, B, T, H, W = case
    geom = ops.Geometry(k, s, p)
    To, Ho, Wo = geom.out_dims(T, H, W)
    g = torch.Generator(device="cuda").manual_seed(2000 + DGRAD_IDS.index(name))
    dy = torch.randn(B, Cout, To, Ho, Wo, device="cuda", generator=g)
    w = _weights(Cout, Cin, k, g, exact=False)
    pl, Cop, dcoff = _planes_of(ops, dy, 1)
    pw = ops.PackedWeights(Cout, Cin, geom.taps, Cop, 1, 1, "cuda").pack(w)
    ref = _dgrad_truth(case, dy.double(), w.double())
    dst = torch.full((B, T, H, W, Cin + DST_EXTRA), 1e30, device="cuda")
    key = "dgrad_bf16/%s" % name
    _launch(dgrad_conv(ops, case, pl, dcoff, pw, dst, 3, 1, False, None), False, diag, key)
    err = _rel(dst[..., DST_COFF:DST_COFF + Cin], ref)
    diag[key] = err
    assert err < 2e-4, (key, err)


# Weight gradients dW[Cout, Cin, *k] += X x dY: (name, kernel, width, Cin, Cout, k, s, p, B, T, H, W).  kernel and width
# are the instance the launch must reach: the TMA-staged kernel at item width N = coclr_wgrad_tma_plan info[3], or the
# gather kernel at K-column tile width wgrad_bnk(Kreal).  One TMA case per kind and product count (3 passes: 2 products
# when Cout <= 64, stacked, else 3; single pass: 1), the block kind at every N; test_conv_bwd_scaled_plan_cpu.py
# checks the labels and that every weight-gradient launch class of the training plans is among these or the other
# float64 weight-gradient tests.  A (., 4, 4) kernel is a space-to-depth stem: Cin = 12 real channels of 16-channel
# pixels, rows zero-padded by engine.S2D_PAD = 2 pixels on each side, and (T, H, W) the destination frame.
WGRAD_CASES = [
    ("tma64_pw_64_256", "tma", 64, 64, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 2, 7, 9),
    ("tma64_pw_48_32", "tma", 64, 48, 32, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 3, 5, 7),
    ("tma128_pw_128_192", "tma", 128, 128, 192, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 2, 9, 7),
    ("tma128_pw_96_48", "tma", 128, 96, 48, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1, 3, 6, 7),
    ("tma192_pw_192_96", "tma", 192, 192, 96, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 3, 7, 9),
    ("tma192_pw_192_32", "tma", 192, 192, 32, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 3, 6, 5),
    ("tma256_pw_256_128", "tma", 256, 256, 128, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 2, 5, 9),
    ("tma256_pw_480_64", "tma", 256, 480, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 2, 8, 5),
    ("tma192_sp_64_192", "tma", 192, 64, 192, (1, 3, 3), (1, 1, 1), (0, 1, 1), 2, 2, 8, 12),
    ("tma192_sp_32_48", "tma", 192, 32, 48, (1, 3, 3), (1, 1, 1), (0, 1, 1), 1, 3, 8, 8),
    ("tma192_tm_64_96", "tma", 192, 64, 96, (3, 1, 1), (1, 1, 1), (1, 0, 0), 2, 4, 6, 6),
    ("tma192_tm_48_48", "tma", 192, 48, 48, (3, 1, 1), (1, 1, 1), (1, 0, 0), 2, 5, 5, 5),
    # the stem's temporally strided (7,1,1) conv: taps 0,2,4,6 / 1,3,5 per frame parity, both at N = 256
    ("tma256_stem_tm", "tma", 256, 64, 64, (7, 1, 1), (2, 1, 1), (3, 0, 0), 2, 6, 10, 12),
    # the S3D space-to-depth stem (1,4,4): one slab serves all 16 taps
    ("tma256_stem_s2d", "tma", 256, 12, 64, (1, 4, 4), (1, 1, 1), (0, 2, 0), 2, 3, 12, 24),
    # shapes the TMA-staged kernel declines: spatially strided ResNet-50 convs, (1,3,3) on 4x4 frames, and the ResNet-50
    # space-to-depth stem (5,4,4) with temporal stride 2
    ("g128_r50_conv2_s2", "gather", 128, 128, 128, (1, 3, 3), (1, 2, 2), (0, 1, 1), 2, 2, 16, 16),
    ("g128_r50_conv2_s2_odd", "gather", 128, 64, 96, (1, 3, 3), (1, 2, 2), (0, 1, 1), 1, 3, 9, 7),
    ("g64_r50_ds_s2_odd", "gather", 64, 64, 256, (1, 1, 1), (1, 2, 2), (0, 0, 0), 1, 2, 7, 9),
    ("g128_r50_ds_s2_T3", "gather", 128, 256, 128, (1, 1, 1), (1, 2, 2), (0, 0, 0), 2, 3, 8, 8),
    ("g128_sp_4x4", "gather", 128, 96, 208, (1, 3, 3), (1, 1, 1), (0, 1, 1), 2, 4, 4, 4),
    ("g128_r50_stem_s2d", "gather", 128, 12, 64, (5, 4, 4), (2, 1, 1), (2, 2, 0), 2, 5, 8, 12),
]
WGRAD_IDS = [c[0] for c in WGRAD_CASES]


def wgrad_bnk(Kreal):
    """K-column tile width of the gather weight-gradient kernel: wgrad_bnk() in coclr_b200/csrc/conv_igemm.cu
    (multiples of 64, at most 128, balanced over the tiles)."""
    kt = (Kreal + 127) // 128
    w = (Kreal + kt - 1) // kt
    return (w + 63) // 64 * 64


def wgrad_window(case):
    """True for the space-to-depth stems (see WGRAD_CASES)."""
    return case[5][1:] == (4, 4)


def wgrad_dims(ops, case):
    """(source T, H, W) and (destination To, Ho, Wo) of a weight-gradient case."""
    name, kernel, width, Cin, Cout, k, s, p, B, T, H, W = case
    geom = ops.Geometry(k, s, p)
    if wgrad_window(case):
        return (T, H, W + 4), (geom.out_dims(T, H, W + 4)[0], H, W)
    return (T, H, W), geom.out_dims(T, H, W)


@pytest.mark.parametrize("mag", MAGS)
@pytest.mark.parametrize("npass", [3, 1])
@pytest.mark.parametrize("case", WGRAD_CASES, ids=WGRAD_IDS)
def test_wgrad_fp16_scaled(case, npass, mag, diag):
    """dW += (fp16 activation planes) x (fp16 planes of dY * s), times out_scale = 1/s, added to a dW that holds a
    nonzero value, on the kernel instance the case names (the TMA-staged kernel with a NaN-poisoned workspace)."""
    from coclr_b200 import ops, lib as L
    lib = L.load()
    name, kernel, width, Cin, Cout, k, s, p, B, T, H, W = case
    geom = ops.Geometry(k, s, p)
    (Ts, Hs, Ws), (To, Ho, Wo) = wgrad_dims(ops, case)
    g = torch.Generator(device="cuda").manual_seed(3000 + sum(map(ord, name)) + npass)
    x = torch.relu(torch.randn(B, Cin, T, H, W, device="cuda", generator=g))
    dy = torch.randn(B, Cout, To, Ho, Wo, device="cuda", generator=g) * mag
    sc = _pow2_scale(dy)
    if wgrad_window(case):
        xpad = F.pad(F.pad(x, (0, 0, 0, 0, 0, 0, 0, 16 - Cin)), (2, 2))
        xp, Cp, xcoff = _planes_of(ops, xpad, 0, ld_extra=0, coff=0, lo=(npass > 1))
    else:
        xp, Cp, xcoff = _planes_of(ops, x, 0, lo=(npass > 1))
    dp, Cop, dcoff = _planes_of(ops, dy * sc, 0, lo=(npass > 1))
    out_scale = torch.tensor([1.0 / sc], device="cuda")
    wd = torch.zeros(Cout, Cin, *k, device="cuda", dtype=torch.float64, requires_grad=True)

    def truth(xv, dyv):
        (r,) = torch.autograd.grad(F.conv3d(xv, wd, stride=s, padding=p)[..., :Ho, :Wo], wd, dyv)
        return r

    xv = xp.value()[..., xcoff:xcoff + Cin].permute(0, 4, 1, 2, 3).double()          # exact operand values
    ref = truth(xv, dy.double())
    top = float(ref.abs().max())
    base = torch.randn(Cout, Cin, *k, device="cuda", generator=g) * top
    dw = base.clone()
    wg = L.Wgrad(xp.src(xcoff, Cp, Ts, Hs, Ws), geom.c(0), dp.src(dcoff, Cop, To, Ho, Wo), B, To, Ho, Wo, Cout, Cin,
                 L.dptr(dw), npass, 0, 0, 1, L.dptr(out_scale))
    info = (C.c_int * 8)()
    if lib.coclr_wgrad_tma_plan(C.byref(wg), info) == 1:
        ran = ("tma", info[3])
        need = int(lib.coclr_wgrad_ws_floats(C.byref(wg)))
        ws = torch.full((need,), float("nan"), device="cuda")       # every element read must have been written
        wg.ws, wg.ws_floats = L.dptr(ws).value, need
    else:
        ran = ("gather", wgrad_bnk(geom.taps * Cp))
    diag["kernel/wgrad_fp16/%s/p%d" % (name, npass)] = list(ran)
    assert ran == (kernel, width), (name, ran)
    L.check(lib.coclr_conv_wgrad(C.byref(wg), L.stream_ptr()), "coclr_conv_wgrad")
    torch.cuda.synchronize()
    got = dw.double() - base.double()
    errs = [_rel(got, ref)]
    if npass == 1:
        xh = xp.hi[..., xcoff:xcoff + Cin].double().permute(0, 4, 1, 2, 3)
        dh = dp.hi[..., dcoff:dcoff + Cout].double().permute(0, 4, 1, 2, 3) / sc
        errs.append(_rel(got, truth(xh, dh)))
    key = "wgrad_fp16/%s/p%d/m%g" % (name, npass, mag)
    diag[key] = errs
    if npass == 3:
        assert errs[0] < 2e-5, (key, errs)
    else:
        assert errs[1] < 2e-5 and errs[0] < 4e-3, (key, errs)


# The chain of one BatchNorm+ReLU unit: (name, Cin, Cout, k, s, p, B, T, H, W); the first runs both convolutions on the
# TMA-staged kernels, the second on the gather kernels
CHAIN_CASES = [
    ("tma_sp_64_192", 64, 192, (1, 3, 3), (1, 1, 1), (0, 1, 1), 2, 2, 16, 16),
    ("gather_r50_conv2_s2_odd", 64, 96, (1, 3, 3), (1, 2, 2), (0, 1, 1), 1, 3, 9, 7),
]


@pytest.mark.parametrize("mag", [1e-6, 1e2])
@pytest.mark.parametrize("case", CHAIN_CASES, ids=[c[0] for c in CHAIN_CASES])
def test_bn_bwd_into_conv_backward(case, mag, diag):
    """coclr_bn_bwd (dy_fp16 = 1, relu = 1) writes the dY planes and (s, 1/s); the data gradient and the weight
    gradient read those planes with out_scale = dy_scale[1:], the view the engine passes.  Truth: float64 autograd of
    relu(batch_norm(y)) for dY, then the float64 conv transposes."""
    import ctypes as C_
    from coclr_b200 import ops, lib as L
    name, Cin, Cout, k, s, p, B, T, H, W = case
    geom = ops.Geometry(k, s, p)
    To, Ho, Wo = geom.out_dims(T, H, W)
    M = B * To * Ho * Wo
    g = torch.Generator(device="cuda").manual_seed(4000 + len(name))
    y = torch.randn(M, Cout, device="cuda", generator=g) * 1.5 + 0.3
    gamma = torch.rand(Cout, device="cuda", generator=g) + 0.5
    beta = torch.randn(Cout, device="cuda", generator=g) * 0.2
    dA = torch.randn(M, Cout, device="cuda", generator=g) * mag
    y = _clear_of_kink(y, gamma, beta)
    x = torch.relu(torch.randn(B, Cin, T, H, W, device="cuda", generator=g))
    w = torch.randn(Cout, Cin, *k, device="cuda", generator=g) * 0.05
    yd = y.double().requires_grad_(True)
    (dy64,) = torch.autograd.grad(torch.relu(F.batch_norm(yd, None, None, gamma.double(), beta.double(), True, 0.1,
                                                          1e-5)), yd, dA.double())
    dy64 = dy64.view(B, To, Ho, Wo, Cout).permute(0, 4, 1, 2, 3)
    mean = y.double().mean(0)
    rstd = (y.double().var(0, unbiased=False) + 1e-5).rsqrt()
    scale = (gamma.double() * rstd).float()
    shift = (beta.double() - mean * gamma.double() * rstd).float()
    mean32, rstd32 = mean.float().contiguous(), rstd.float().contiguous()
    sums = torch.zeros(2 * Cout, dtype=torch.float64, device="cuda")
    amax = torch.zeros(2 * Cout, device="cuda")
    dy_scale = torch.ones(2, device="cuda")
    dgam, dbet = torch.zeros(Cout, device="cuda"), torch.zeros(Cout, device="cuda")
    dpl = ops.Planes((B, To, Ho, Wo, Cout), 0, "cuda")
    bb = L.BnBwd(L.dptr(y), L.dptr(dA), Cout, 0, Cout, M, L.dptr(scale), L.dptr(shift), L.dptr(mean32), L.dptr(rstd32),
                 1, L.dptr(sums), L.dptr(dgam), L.dptr(dbet), L.dptr(dpl.hi), L.dptr(dpl.lo),
                 None, None, 0, 0, 0, None, 0, 0, 0, 1, L.dptr(amax), L.dptr(dy_scale))
    L.check(L.load().coclr_bn_bwd(C_.byref(bb), L.num_sms(), L.stream_ptr()), "coclr_bn_bwd")
    oscale = dy_scale[1:]
    dsrc = dpl.src(0, Cout, To, Ho, Wo)
    # data gradient into a channel slice of a wider buffer
    pw = ops.PackedWeights(Cout, Cin, geom.taps, Cout, 1, 0, "cuda").pack(w)
    dx = torch.full((B, T, H, W, Cin + DST_EXTRA), 1e30, device="cuda")
    cv = ops.make_conv(dsrc, 0, geom.c(1), B, (T, H, W), pw, dx, DST_COFF, npass=3, out_scale=oscale)
    kernel = _launch(cv, False, diag, "chain/%s/m%g/dgrad" % (name, mag))
    assert kernel == name.split("_")[0]
    # weight gradient against the forward activation planes
    xp, Cp, xcoff = _planes_of(ops, x, 0)
    src = xp.src(xcoff, Cp, T, H, W)
    dw = torch.zeros(Cout, Cin, *k, device="cuda")
    wg = L.Wgrad(src, geom.c(0), dsrc, B, To, Ho, Wo, Cout, Cin, None, 3, 0, 0, 1, None)
    wkernel = "tma" if L.load().coclr_wgrad_tma_plan(C.byref(wg), None) else "gather"
    diag["kernel/chain/%s/m%g/wgrad" % (name, mag)] = wkernel
    assert wkernel == kernel
    ops.conv_wgrad(src, 0, geom.c(0), dsrc, 0, B, (To, Ho, Wo), Cout, Cin, dw, npass=3, out_scale=oscale)
    torch.cuda.synchronize()
    xd = torch.zeros(B, Cin, T, H, W, device="cuda", dtype=torch.float64, requires_grad=True)
    (ref_dx,) = torch.autograd.grad(F.conv3d(xd, w.double(), stride=s, padding=p), xd, dy64)
    xv = xp.value()[..., xcoff:xcoff + Cin].permute(0, 4, 1, 2, 3).double()
    wd = torch.zeros(Cout, Cin, *k, device="cuda", dtype=torch.float64, requires_grad=True)
    (ref_dw,) = torch.autograd.grad(F.conv3d(xv, wd, stride=s, padding=p), wd, dy64)
    e_dx = _rel(dx[..., DST_COFF:DST_COFF + Cin], ref_dx.permute(0, 2, 3, 4, 1))
    e_dw = _rel(dw, ref_dw)
    e_dy = _rel(dpl.value().double() * float(dy_scale[1]), dy64.permute(0, 2, 3, 4, 1))
    diag["chain/%s/m%g" % (name, mag)] = [e_dy, e_dx, e_dw, float(dy_scale[0])]
    poison = torch.full_like(dx, 1e30)
    assert torch.equal(dx[..., :DST_COFF], poison[..., :DST_COFF])
    assert torch.equal(dx[..., DST_COFF + Cin:], poison[..., DST_COFF + Cin:])
    # dY may carry up to 2e-6 of its own (test_bn_relu_backward_planes), the convolutions add fp32 accumulation; both
    # stay below 3e-7 on an H100 SXM
    assert e_dy < 2e-6 and e_dx < 5e-6 and e_dw < 5e-6, (e_dy, e_dx, e_dw)


# coclr_pack_weights_batch against one coclr_pack_weights launch per entry: (Cout, Cin, taps, Cpad, mode, bf16)
PACK_TABLE = [
    (64, 12, 80, 16, 0, 0),       # ResNet-50 space-to-depth stem (5,4,4): Cpad > Cin, BN 64
    (64, 12, 80, 16, 0, 1),
    (32, 64, 9, 64, 0, 1),        # BN 32
    (96, 100, 7, 104, 0, 0),      # BN 96, Cpad > Cin, 7 taps
    (136, 512, 1, 512, 0, 0),     # 2 N tiles of 96 (68 + 68 real rows)
    (320, 160, 9, 160, 0, 1),     # 3 N tiles of 128 (107 + 107 + 106)
    (1024, 256, 1, 256, 0, 0),    # 8 N tiles of 128
    (832, 384, 1, 832, 1, 0),     # mode 1: N = Cin = 384, 3 N tiles
    (36, 96, 9, 40, 1, 1),        # mode 1: Cpad > Cout, BN 96
    (48, 64, 3, 48, 1, 0),        # mode 1: BN 64
    (192, 32, 1, 192, 1, 1),      # mode 1: BN 32
    (208, 208, 3, 208, 1, 0),     # mode 1: 2 N tiles of 128 (104 real rows each)
]


def test_pack_weights_batch_matches_per_layer():
    from coclr_b200 import ops, lib as L
    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(77)
    arr = (L.Pack * len(PACK_TABLE))()
    starts, singles, batched, keep = [0], [], [], []
    for i, (Cout, Cin, taps, Cpad, mode, bf16) in enumerate(PACK_TABLE):
        # rows of very different scale, and one all-zero row (its unscale stays 1)
        w = torch.randn(Cout, Cin, taps, device="cuda", generator=g)
        w = w * 2.0 ** torch.randint(-12, 13, (Cout, Cin, 1), device="cuda", generator=g).float()
        if mode == 0:
            w[0] = 0.0              # packed row 0 = output channel 0
        else:
            w[:, 0] = 0.0           # packed row 0 = input channel 0
        w = w.contiguous()
        one = ops.PackedWeights(Cout, Cin, taps, Cpad, mode, bf16, "cuda")
        one.wpk.fill_(0xAB)
        one.unscale.fill_(-1.0)
        one.pack(w)
        many = ops.PackedWeights(Cout, Cin, taps, Cpad, mode, bf16, "cuda")
        many.wpk.fill_(0xCD)
        many.unscale.fill_(-2.0)
        arr[i] = L.Pack(L.dptr(w), Cout, Cin, taps, Cpad, mode, bf16, L.dptr(many.wpk), L.dptr(many.unscale))
        starts.append(starts[-1] + many.BN * many.n_tiles)
        singles.append(one)
        batched.append(many)
        keep.append(w)
    raw = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).cuda()
    rs = torch.tensor(starts, dtype=torch.int32, device="cuda")
    L.check(lib.coclr_pack_weights_batch(L.dptr(raw), L.dptr(rs), len(PACK_TABLE), starts[-1], L.stream_ptr()),
            "coclr_pack_weights_batch")
    torch.cuda.synchronize()
    assert sorted({(b.BN, b.n_tiles > 1) for b in batched}) == [(32, False), (64, False), (96, False), (96, True),
                                                                  (128, True)]
    for entry, one, many in zip(PACK_TABLE, singles, batched):
        assert torch.equal(one.wpk, many.wpk), entry
        assert torch.equal(one.unscale, many.unscale), entry
