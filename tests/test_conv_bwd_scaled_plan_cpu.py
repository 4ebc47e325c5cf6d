"""Host-side plans (no GPU) behind test_conv_bwd_scaled_gpu.py and test_wgrad_tma_gpu.py: their data-gradient cases
reach every fp16 (pass count, tile width) instance of both convolution kernels through the planner, their
weight-gradient cases reach every instance of both weight-gradient kernels, and every launch class that the S3D, S3D-G
and ResNet-50 training plans send to coclr_conv_igemm or coclr_conv_wgrad in `parity` and `mixed` precision is one that
a float64 unit test runs.  A convolution launch class is (kernel, passes, tile width BN, 16-bit format, transposed,
out_scale set); a weight-gradient launch class is (kernel, width, products per K step, 16-bit format, kind, out_scale
set).  A planner change that creates a class no unit test runs makes this fail."""
import ctypes as C

import pytest
import torch

from test_conv_bwd_scaled_gpu import DGRAD_CASES, dgrad_conv
import test_conv_bwd_scaled_gpu as TS
import test_conv_gpu as TC
import test_conv_igemm_repro_gpu as TR
import test_wgrad_tma_gpu as TW


def _class(lib, cv):
    kernel = "tma" if lib.coclr_conv_tma_plan(C.byref(cv), None) == 1 else "gather"
    return (kernel, cv.npass, cv.BN, "bf16" if cv.a_bf16 else "fp16", cv.g.transposed, bool(cv.out_scale))


def _dgrad_classes(ops, lib, case, npass, bf16, out_scale):
    name, kernel, BN, Cin, Cout, k, s, p, B, T, H, W = case
    geom = ops.Geometry(k, s, p)
    To, Ho, Wo = geom.out_dims(T, H, W)
    Cop = (Cout + 7) // 8 * 8
    pl = ops.Planes((B, To, Ho, Wo, Cop + 16), bf16, "cpu", lo=npass > 1)
    pw = ops.PackedWeights(Cout, Cin, geom.taps, Cop, 1, bf16, "cpu")
    dst = torch.empty(B, T, H, W, Cin + 16)
    osc = torch.ones(1) if out_scale else None
    return {_class(lib, dgrad_conv(ops, case, pl, 8, pw, dst, npass, bf16, acc, osc)) for acc in (False, True)}


def _tested_classes(ops, lib):
    """Launch classes the float64 convolution tests run (test_conv_bwd_scaled_gpu.py, test_conv_gpu.py,
    test_conv_igemm_repro_gpu.py)."""
    got = set()
    for case in DGRAD_CASES:
        for npass in (3, 1):
            got |= _dgrad_classes(ops, lib, case, npass, 0, True)
            got |= {("gather",) + c[1:] for c in _dgrad_classes(ops, lib, case, npass, 0, True)}   # forced gather
        got |= _dgrad_classes(ops, lib, case, 3, 1, False)
    # test_conv_forward; test_gather_forward_is_bit_reproducible
    fwd = [(c, (3, 0), (3, 1), (1, 1)) for c in TC.CASES] + [(c, (3, 0), (3, 1)) for c in TR.CASES]
    for (name, Cin, Cout, k, s, p, B, T, H, W), *modes in fwd:
        geom = ops.Geometry(k, s, p)
        To, Ho, Wo = geom.out_dims(T, H, W)
        Cp = (Cin + 7) // 8 * 8
        for npass, bf16 in modes:
            pl = ops.Planes((B, T, H, W, Cp + 16), bf16, "cpu", lo=npass > 1)
            pw = ops.PackedWeights(Cout, Cin, geom.taps, Cp, 0, bf16, "cpu")
            dst = torch.empty(B, To, Ho, Wo, Cout + 40)
            stats = torch.zeros(2 * Cout, dtype=torch.float64)
            got.add(_class(lib, ops.make_conv(pl.src(8, Cp, T, H, W), bf16, geom.c(0), B, (To, Ho, Wo), pw, dst, 32,
                                              stats_sum=stats[:Cout], stats_sq=stats[Cout:], npass=npass)))
    for name, Cin, Cout, k, s, p, B, T, H, W in TC.DGRAD_CASES:
        geom = ops.Geometry(k, s, p)
        To, Ho, Wo = geom.out_dims(T, H, W)
        Cop = (Cout + 7) // 8 * 8
        for npass in (3, 1):                                   # test_conv_dgrad
            pl = ops.Planes((B, To, Ho, Wo, Cop + 16), 1, "cpu", lo=npass > 1)
            pw = ops.PackedWeights(Cout, Cin, geom.taps, Cop, 1, 1, "cpu")
            dst = torch.empty(B, T, H, W, Cin)
            got.add(_class(lib, ops.make_conv(pl.src(8, Cop, To, Ho, Wo), 1, geom.c(1), B, (T, H, W), pw, dst,
                                              npass=npass)))
    return got


@pytest.fixture
def dry_run():
    from coclr_b200 import lib as L
    lib = L.load()
    L.DRY_RUN = True
    try:
        yield lib
    finally:
        L.DRY_RUN = False


def test_cases_reach_every_fp16_instance(dry_run):
    from coclr_b200 import ops
    lib = dry_run
    reached = set()
    for case in DGRAD_CASES:
        name, kernel, BN = case[:3]
        for npass in (3, 1):
            cls = _dgrad_classes(ops, lib, case, npass, 0, True)
            assert cls == {(kernel, npass, BN, "fp16", 1, True)}, (name, cls)
            reached |= {(kernel, npass, BN)}
    assert reached == {(k, n, bn) for k in ("tma", "gather") for n in (3, 1) for bn in (32, 64, 96, 128)}


@pytest.mark.parametrize("network", ["s3d", "s3dg", "r50"])
def test_every_plan_launch_class_is_tested(network, dry_run):
    """Training plans at the benchmark shape (B, T, H, W) = (32, 32, 128, 128)."""
    from coclr_b200 import ops, engine as E
    from coclr_b200.s3d_spec import s3d_stages
    from coclr_b200.r50_spec import r50_stages
    lib = dry_run
    tested = _tested_classes(ops, lib)
    for precision in ("parity", "mixed"):
        if network == "r50":
            g = E.Graph(r50_stages(3), 3, head_dim=128, feature_size=2048, bb_prefix="0.")
        else:
            g = E.Graph(s3d_stages(3, gating=network == "s3dg"), 3, head_dim=128, bb_prefix="0.")
        eng = E.EncoderEngine(E.ParamStore(g, "cpu"), g, precision)
        p = eng.plan(32, 32, 128, 128, True, True)
        classes = {_class(lib, a[0]._obj) for fn, a in p.fwd + p.bwd if fn.__name__ == "coclr_conv_igemm"}
        assert any(c[5] for c in classes), "no data gradient with out_scale in the plan"
        untested = sorted(classes - tested)
        assert not untested, (precision, untested)


# ---- weight gradients ----

def _wgrad_kind(wg):
    g = wg.g
    if g.kt * g.kh * g.kw == 1:
        return "block"
    if g.kw > 1 and g.pw == 0 and wg.src.W > wg.Wd:      # space-to-depth planes: rows padded in memory
        return "window"
    if g.st == 2 and g.kh == 1 and g.kw == 1:
        return "tstride"
    if g.kt == 1:
        return "spatial"
    if g.kh == 1 and g.kw == 1:
        return "temporal"
    return "3d"


def _wclass(lib, wg, gather=False):
    """(kernel, width, products, format, kind, out_scale set) of one coclr_conv_wgrad launch; gather: the launch with
    the TMA-staged kernel switched off (coclr_set_wgrad_tma(0)).  The TMA-staged kernel takes a shape its planner
    accepts when the call brings a large enough workspace."""
    info = (C.c_int * 8)()
    tma = (not gather and lib.coclr_wgrad_tma_plan(C.byref(wg), info) == 1 and bool(wg.ws)
           and wg.ws_floats >= lib.coclr_wgrad_ws_floats(C.byref(wg)))
    width = info[3] if tma else TS.wgrad_bnk(wg.g.kt * wg.g.kh * wg.g.kw * wg.src.C)
    prod = 1 if wg.npass == 1 else (2 if wg.Cout <= 64 else 3)
    return ("tma" if tma else "gather", width, prod, "bf16" if wg.dy_bf16 else "fp16", _wgrad_kind(wg), bool(wg.out_scale))


def _wgrad(ops, L, lib, k, s, p, B, dims, Cin, Cout, npass, bf16, out_scale, window=False, keep=None):
    """A coclr_wgrad_t over CPU planes laid out as the GPU tests lay them out: activation channels in a slice of a wider
    buffer (window: the space-to-depth stem's 16-channel pixels, rows padded by 2 on each side), dY in a slice of a wider
    buffer, a workspace of the size the shape asks for."""
    geom = ops.Geometry(k, s, p)
    T, H, W = dims
    lo = npass > 1
    if window:
        To, Ho, Wo = geom.out_dims(T, H, W + 4)[0], H, W
        xp = ops.Planes((B, T, H, W + 4, 16), bf16, "cpu", lo=lo)
        src = xp.src(0, 16, T, H, W + 4)
    else:
        To, Ho, Wo = geom.out_dims(T, H, W)
        Cp = (Cin + 7) // 8 * 8
        xp = ops.Planes((B, T, H, W, Cp + 24), bf16, "cpu", lo=lo)
        src = xp.src(8, Cp, T, H, W)
    Cop = (Cout + 7) // 8 * 8
    dp = ops.Planes((B, To, Ho, Wo, Cop + 24), bf16, "cpu", lo=lo)
    dw = torch.empty(Cout * Cin * geom.taps)
    osc = torch.ones(1) if out_scale else None
    wg = L.Wgrad(src, geom.c(0), dp.src(16, Cop, To, Ho, Wo), B, To, Ho, Wo, Cout, Cin, L.dptr(dw), npass, bf16, bf16, 1,
                 L.dptr(osc))
    need = int(lib.coclr_wgrad_ws_floats(C.byref(wg)))
    ws = torch.empty(max(need, 4))
    wg.ws, wg.ws_floats = L.dptr(ws).value, ws.numel()
    if keep is not None:
        keep += [xp, dp, dw, osc, ws]
    return wg


def _tested_wgrad_classes(ops, L, lib):
    """Weight-gradient launch classes the float64 tests run: test_wgrad_tma_gpu.py (every case on the TMA-staged and on
    the gather kernel, the strided and the space-to-depth stems), test_conv_bwd_scaled_gpu.py (test_wgrad_fp16_scaled,
    test_bn_bwd_into_conv_backward), test_conv_gpu.py (test_conv_wgrad, test_r50_stem_space_to_depth)."""
    got, keep = set(), []
    one = (1, 1, 1)
    for name, Cin, Cout, k, p, B, T, H, W in TW.CASES:                       # test_wgrad_tma_vs_float64_and_gather
        for npass in (3, 1):
            for bf16 in (0, 1):
                wg = _wgrad(ops, L, lib, k, one, p, B, (T, H, W), Cin, Cout, npass, bf16, True, keep=keep)
                got |= {_wclass(lib, wg), _wclass(lib, wg, gather=True)}
    for dims in ((1, 8, 16, 16), (2, 6, 10, 12)):                            # test_wgrad_tma_temporal_stride2
        wg = _wgrad(ops, L, lib, (7, 1, 1), (2, 1, 1), (3, 0, 0), dims[0], dims[1:], 64, 64, 3, 0, False, keep=keep)
        got |= {_wclass(lib, wg), _wclass(lib, wg, gather=True)}
    for dims in ((1, 2, 16, 16), (2, 3, 12, 24)):                            # test_wgrad_tma_space_to_depth_window
        wg = _wgrad(ops, L, lib, (1, 4, 4), one, (0, 2, 0), dims[0], dims[1:], 12, 64, 3, 0, False, window=True,
                    keep=keep)
        got |= {_wclass(lib, wg), _wclass(lib, wg, gather=True)}
    for case in TS.WGRAD_CASES:                                              # test_wgrad_fp16_scaled
        name, kernel, width, Cin, Cout, k, s, p, B, T, H, W = case
        for npass in (3, 1):
            wg = _wgrad(ops, L, lib, k, s, p, B, (T, H, W), Cin, Cout, npass, 0, True, window=TS.wgrad_window(case),
                        keep=keep)
            got.add(_wclass(lib, wg))
    for name, Cin, Cout, k, s, p, B, T, H, W in TS.CHAIN_CASES:              # test_bn_bwd_into_conv_backward
        got.add(_wclass(lib, _wgrad(ops, L, lib, k, s, p, B, (T, H, W), Cin, Cout, 3, 0, True, keep=keep)))
    for name, Cin, Cout, k, s, p, B, T, H, W in TC.CASES:                    # test_conv_wgrad
        for npass in (3, 1):
            got.add(_wclass(lib, _wgrad(ops, L, lib, k, s, p, B, (T, H, W), Cin, Cout, npass, 1, False, keep=keep)))
    for T in (4, 5):                                                         # test_r50_stem_space_to_depth
        for npass, bf16 in ((3, 0), (1, 1)):
            got.add(_wclass(lib, _wgrad(ops, L, lib, (5, 4, 4), (2, 1, 1), (2, 2, 0), 2, (T, 8, 12), 12, 64, npass,
                                        bf16, False, window=True, keep=keep)))
    return got


def test_wgrad_cases_reach_every_instance(dry_run):
    """Every wgrad_tma_kernel<N, NPROD, BF16> instance (24) and every conv_wgrad_kernel<NPROD, BNK, BF16> instance (12)
    runs in a float64 test, and each test_wgrad_fp16_scaled case reaches the kernel and width it names."""
    from coclr_b200 import ops, lib as L
    lib = dry_run
    for case in TS.WGRAD_CASES:
        name, kernel, width, Cin, Cout, k, s, p, B, T, H, W = case
        for npass in (3, 1):
            wg = _wgrad(ops, L, lib, k, s, p, B, (T, H, W), Cin, Cout, npass, 0, True, window=TS.wgrad_window(case))
            assert _wclass(lib, wg)[:2] == (kernel, width), (name, npass, _wclass(lib, wg))
    reached = {c[:4] for c in _tested_wgrad_classes(ops, L, lib)}
    want = {("tma", n, prod, f) for n in (64, 128, 192, 256) for prod in (1, 2, 3) for f in ("fp16", "bf16")}
    want |= {("gather", n, prod, f) for n in (64, 128) for prod in (1, 2, 3) for f in ("fp16", "bf16")}
    assert len(want) == 36
    assert not want - reached, sorted(want - reached)


@pytest.mark.parametrize("network", ["s3d", "s3dg", "r50"])
def test_every_plan_wgrad_class_is_tested(network, dry_run):
    """Every weight gradient of the training plans at the benchmark shape (B, T, H, W) = (32, 32, 128, 128), the
    space-to-depth stem's included, in `parity` and `mixed`."""
    from coclr_b200 import ops, lib as L, engine as E
    from coclr_b200.s3d_spec import s3d_stages
    from coclr_b200.r50_spec import r50_stages
    lib = dry_run
    tested = _tested_wgrad_classes(ops, L, lib)
    untested = {}
    for precision in ("parity", "mixed"):
        if network == "r50":
            g = E.Graph(r50_stages(3), 3, head_dim=128, feature_size=2048, bb_prefix="0.")
        else:
            g = E.Graph(s3d_stages(3, gating=network == "s3dg"), 3, head_dim=128, bb_prefix="0.")
        eng = E.EncoderEngine(E.ParamStore(g, "cpu"), g, precision)
        p = eng.plan(32, 32, 128, 128, True, True)
        assert p.s2d_wgrads, "no space-to-depth stem in the plan"
        classes = {_wclass(lib, w) for w in p.wgrads + p.s2d_wgrads}
        assert {"tma", "gather"} >= {c[0] for c in classes} and any(c[5] for c in classes)
        if classes - tested:
            untested[precision] = sorted(classes - tested)
    assert not untested, untested
