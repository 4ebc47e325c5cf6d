"""Host-side plans (no GPU) behind test_conv_bwd_scaled_gpu.py: its data-gradient cases reach every fp16 (pass count,
tile width) instance of both convolution kernels through the planner, and every launch class that the S3D, S3D-G and
ResNet-50 training plans send to coclr_conv_igemm in `parity` and `mixed` precision is one that a float64 unit test
runs.  A launch class is (kernel, passes, tile width BN, 16-bit format, transposed, out_scale set); a planner change
that creates a class no unit test runs makes this fail."""
import ctypes as C

import pytest
import torch

from test_conv_bwd_scaled_gpu import DGRAD_CASES, dgrad_conv
import test_conv_gpu as TC
import test_conv_igemm_repro_gpu as TR


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
