"""GPU checks of the TMA-staged convolution's register-only epilogue (csrc/conv_tma.cu): every consumer thread scales its
accumulator fragment and writes it into the staging blocks, whose owner warps store them and accumulate the BatchNorm
statistics, with no barrier between the two warpgroups.  The launches below hand a CTA several tiles, uneven tile counts
per CTA, several N tiles, ragged last tiles, resident and streamed weights, the space-to-depth stem, the frame-parity slab
types of the strided stem's data gradient and the bulk add-reduction.  Each is compared with the cp.async gather kernel
(outputs and statistics, tolerances as in test_conv_tma_gpu.py) and run twice for bit-identical results."""
import ctypes as C

import pytest
import torch

from test_conv_gpu import _planes_of, _rel

pytestmark = pytest.mark.gpu

# (name, Cin, Cout, k, s, p, B, T, H, W): forward with statistics
FWD = [
    # 1x1, 2 x 4 x 20 x 20 = 3200 rows: 25 tiles, the last one ragged; one tile per CTA
    ("pw_ragged_m", 64, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 4, 20, 20),
    # 1x1, 262 tiles over 132 CTAs: two tiles for most CTAs, one for the rest; resident weights
    ("pw_uneven_resident", 64, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 8, 46, 46),
    # 1x1, 384 output channels = 3 N tiles, streamed weights, ragged last M tile
    ("pw_n_tiles", 256, 384, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 5, 12, 12),
    # 480 input channels (a partial K chunk), streamed weights, many tiles per CTA
    ("pw_streamed", 480, 192, (1, 1, 1), (1, 1, 1), (0, 0, 0), 4, 8, 16, 16),
    # (1,3,3) with 20-row frames: ragged tiles in H, two N tiles of 96
    ("sp_ragged_h", 128, 192, (1, 3, 3), (1, 1, 1), (0, 1, 1), 2, 3, 20, 16),
    # (3,1,1), 12 frames of 8 x 8
    ("tm_ragged_t", 64, 64, (3, 1, 1), (1, 1, 1), (1, 0, 0), 2, 12, 8, 8),
    # the temporally strided stem conv
    ("stem_tm", 64, 64, (7, 1, 1), (2, 1, 1), (3, 0, 0), 2, 16, 16, 16),
]
# data gradients: (case, accumulate)
DGRAD = [
    (("stem_tm_dgrad", 64, 64, (7, 1, 1), (2, 1, 1), (3, 0, 0), 2, 16, 16, 16), 0),
    (("stem_tm_dgrad_acc", 64, 64, (7, 1, 1), (2, 1, 1), (3, 0, 0), 2, 16, 16, 16), 1),
    (("sp_dgrad_acc", 192, 64, (1, 3, 3), (1, 1, 1), (0, 1, 1), 2, 4, 16, 16), 1),
    (("pw_dgrad_n_tiles_acc", 384, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2, 6, 12, 12), 1),
]


def _run(cv, tma):
    from coclr_b200 import lib as L
    lib = L.load()
    lib.coclr_set_conv_tma(1 if tma else 0)
    try:
        L.check(lib.coclr_conv_igemm(C.byref(cv), L.num_sms(), L.stream_ptr()), "coclr_conv_igemm")
        torch.cuda.synchronize()
    finally:
        lib.coclr_set_conv_tma(1)


def _plan(cv):
    from coclr_b200 import lib as L
    info = (C.c_int * 8)()
    ok = L.load().coclr_conv_tma_plan(C.byref(cv), info)
    return bool(ok), list(info)


def _forward(ops, src, bf16, geom, B, dims, pw, Cout, npass, tma):
    dst = torch.full((B, *dims, Cout + 8), -3.0, device="cuda")
    stats = torch.zeros(2 * Cout, dtype=torch.float64, device="cuda")
    cv = ops.make_conv(src, bf16, geom.c(0), B, dims, pw, dst, 8, stats_sum=stats[:Cout], stats_sq=stats[Cout:],
                       npass=npass)
    if tma:
        ok, info = _plan(cv)
        assert ok, "the planner sends this launch to the gather kernel"
    _run(cv, tma)
    return dst, stats, (info if tma else None)


def _check_forward(dst, stats, ref_dst, ref_stats, Cout, tol):
    assert float((dst[..., :8] + 3.0).abs().max()) == 0.0
    assert _rel(dst[..., 8:], ref_dst[..., 8:]) < tol
    e1 = _rel(stats[:Cout], ref_stats[:Cout])
    e2 = _rel(stats[Cout:], ref_stats[Cout:])
    assert e1 < 1e-5 and e2 < 1e-5, (e1, e2)


@pytest.mark.parametrize("case", FWD, ids=[c[0] for c in FWD])
@pytest.mark.parametrize("npass,bf16", [(3, 0), (1, 1)])
def test_epilogue_forward_matches_gather(case, npass, bf16, diag):
    from coclr_b200 import ops
    name, Cin, Cout, k, s, p, B, T, H, W = case
    geom = ops.Geometry(k, s, p)
    dims = geom.out_dims(T, H, W)
    g = torch.Generator(device="cuda").manual_seed(53)
    x = torch.relu(torch.randn(B, Cin, T, H, W, device="cuda", generator=g)) + 0.5   # channel means far from zero
    w = torch.randn(Cout, Cin, *k, device="cuda", generator=g) * 0.05
    pl, Cp, coff = _planes_of(ops, x, bf16, lo=(npass > 1))
    pw = ops.PackedWeights(Cout, Cin, geom.taps, Cp, 0, bf16, "cuda").pack(w.contiguous())
    src = pl.src(coff, Cp, T, H, W)
    got = [_forward(ops, src, bf16, geom, B, dims, pw, Cout, npass, 1) for _ in range(2)]
    ref = _forward(ops, src, bf16, geom, B, dims, pw, Cout, npass, 0)
    diag["tma_epilogue_plan/%s/p%d" % (name, npass)] = got[0][2]
    tol = 2e-5 if npass == 3 and not bf16 else 3e-2
    _check_forward(got[0][0], got[0][1], ref[0], ref[1], Cout, tol)
    assert torch.equal(got[0][0], got[1][0]), "TMA kernel output differs run to run"
    # statistics: per CTA the same fp32 order every run; the fp64 atomics across CTAs may round differently
    assert _rel(got[0][1], got[1][1]) < 1e-12


def test_epilogue_window_stem_matches_gather(diag):
    """The space-to-depth stem (1,4,4) over zero-padded 16-channel rows, resident weights, several tiles per CTA."""
    from coclr_b200 import ops
    B, T, H2, W2, Cout = 4, 6, 32, 32, 64
    g = torch.Generator(device="cuda").manual_seed(59)
    x = torch.randn(B, 16, T, H2, W2, device="cuda", generator=g)
    x[:, 12:] = 0.0
    w = torch.randn(Cout, 16, 1, 4, 4, device="cuda", generator=g) * 0.05
    xpad = torch.nn.functional.pad(x, (2, 2))
    pl, Cp, coff = _planes_of(ops, xpad, 0, ld_extra=0, coff=0)
    geom = ops.Geometry((1, 4, 4), (1, 1, 1), (0, 2, 0))
    pw = ops.PackedWeights(Cout, 16, 16, 16, 0, 0, "cuda").pack(w.contiguous())
    src = pl.src(0, 16, T, H2, W2 + 4)
    got = [_forward(ops, src, 0, geom, B, (T, H2, W2), pw, Cout, 3, 1) for _ in range(2)]
    ref = _forward(ops, src, 0, geom, B, (T, H2, W2), pw, Cout, 3, 0)
    assert got[0][2][2] == 1, "window stem: weights not resident %s" % got[0][2]
    _check_forward(got[0][0], got[0][1], ref[0], ref[1], Cout, 2e-5)
    assert torch.equal(got[0][0], got[1][0])


@pytest.mark.parametrize("case,accumulate", DGRAD, ids=[c[0][0] for c in DGRAD])
def test_epilogue_dgrad_matches_gather(case, accumulate, diag):
    from coclr_b200 import ops
    name, Cin, Cout, k, s, p, B, T, H, W = case
    geom = ops.Geometry(k, s, p)
    To, Ho, Wo = geom.out_dims(T, H, W)
    g = torch.Generator(device="cuda").manual_seed(61)
    w = torch.randn(Cout, Cin, *k, device="cuda", generator=g) * 0.05
    dy = torch.randn(B, Cout, To, Ho, Wo, device="cuda", generator=g)
    pl, Cop, coff = _planes_of(ops, dy, 1)
    pw = ops.PackedWeights(Cout, Cin, geom.taps, Cop, 1, 1, "cuda").pack(w.contiguous())
    base = torch.randn(B, T, H, W, Cin + 8, device="cuda", generator=g)
    outs = []
    for tma in (1, 1, 0):
        dst = base.clone()
        cv = ops.make_conv(pl.src(coff, Cop, To, Ho, Wo), 1, geom.c(1), B, (T, H, W), pw, dst, 8,
                           accumulate=bool(accumulate), npass=3)
        if tma:
            ok, info = _plan(cv)
            assert ok, "the planner sends the dgrad of %s to the gather kernel" % name
        _run(cv, tma)
        assert torch.equal(dst[..., :8], base[..., :8])
        outs.append(dst[..., 8:] - (base[..., 8:] if accumulate else 0.0))
    assert torch.equal(outs[0], outs[1]), "TMA kernel output differs run to run"
    err = _rel(outs[0], outs[2])
    diag["tma_epilogue_dgrad/%s" % name] = err
    assert err < 2e-4, "TMA dgrad %s against the gather kernel: %.3e" % (name, err)
