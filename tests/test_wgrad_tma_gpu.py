"""The TMA-staged weight-gradient kernel (coclr_b200/csrc/wgrad_tma.cu) through the C ABI (coclr_conv_wgrad), against
  (a) float64 autograd of torch's conv3d on the exact plane values (what cuDNN's wgrad computes in the reference behind
      loss.backward(), main_nce.py:330, for backbone/s3dg.py:11-13,39-42), and
  (b) the cp.async gather kernel on the same inputs (coclr_set_wgrad_tma(0)).
Shapes: every wgrad_tma_kernel<N, NPROD, BF16> instance (item width N = 64, 128, 192, 256; 1, 2 (stacked) or 3
products per K step; fp16 and bf16), over the kinds 1x1x1 / (1,3,3) / (3,1,1) at stride 1, the temporally strided
(7,1,1) stem and the space-to-depth window stem; ragged tiles in every dimension, channel counts that are not multiples
of 64, channel slices of wider (poisoned) buffers, Cout <= 64 (hi / lo stacked into one M = 128 operand) up to 512
(several cout groups), and the benchmark shapes at a small batch.  test_conv_bwd_scaled_plan_cpu.py checks that these
cases reach all 24 instances.  Also: several launches back to back on one shared, larger workspace, as the engine runs
them."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# name, Cin, Cout, k, p, B, T, H, W
CASES = [
    ("pw_64_64", 64, 64, (1, 1, 1), (0, 0, 0), 2, 4, 8, 8),
    ("pw_192_96", 192, 96, (1, 1, 1), (0, 0, 0), 2, 3, 7, 9),          # ragged flat tile
    ("pw_832_384", 832, 384, (1, 1, 1), (0, 0, 0), 4, 2, 4, 4),        # 13 channel chunks, 2 cout groups
    ("pw_480_16", 480, 16, (1, 1, 1), (0, 0, 0), 2, 2, 8, 8),
    ("pw_24_40", 24, 40, (1, 1, 1), (0, 0, 0), 1, 2, 5, 5),
    ("pw_64_256", 64, 256, (1, 1, 1), (0, 0, 0), 2, 4, 7, 9),          # N = 64 with 2 cout groups: <64, 3>
    ("pw_128_512", 128, 512, (1, 1, 1), (0, 0, 0), 2, 4, 9, 7),        # N = 128 (two n64 sub-blocks), 4 cout groups
    ("pw_128_48", 128, 48, (1, 1, 1), (0, 0, 0), 2, 2, 5, 7),          # N = 128 stacked, partial cout block
    ("pw_192_32", 192, 32, (1, 1, 1), (0, 0, 0), 2, 3, 6, 5),          # N = 192 stacked (Mixed_3b 192 -> 32)
    ("sp_64_192", 64, 192, (1, 3, 3), (0, 1, 1), 2, 2, 16, 16),        # Conv_2c.conv1
    ("sp_96_208", 96, 208, (1, 3, 3), (0, 1, 1), 2, 2, 8, 8),          # Mixed_4b.branch1.1.conv1: partial chunk, 4 blocks
    ("sp_16_48", 16, 48, (1, 3, 3), (0, 1, 1), 2, 3, 8, 8),
    ("sp_ragged", 32, 72, (1, 3, 3), (0, 1, 1), 1, 2, 6, 12),
    ("sp_wide", 64, 64, (1, 3, 3), (0, 1, 1), 1, 1, 4, 32),
    ("tm_192_192", 192, 192, (3, 1, 1), (1, 0, 0), 2, 8, 8, 8),        # Conv_2c.conv2
    ("tm_48_48", 48, 48, (3, 1, 1), (1, 0, 0), 2, 4, 6, 6),
    ("tm_ragged", 128, 320, (3, 1, 1), (1, 0, 0), 1, 6, 5, 5),
    ("tm_short", 64, 128, (3, 1, 1), (1, 0, 0), 3, 2, 4, 4),
]


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def _planes(ops, x_ncdhw, bf16, lo, coff, extra):
    """NCDHW fp32 -> hi/lo planes holding the channels at [coff, coff + C8) of a wider buffer whose other channels are
    poisoned (the concat-buffer slices the engine hands to the kernel)."""
    B, Cc, T, H, W = x_ncdhw.shape
    C8 = (Cc + 7) // 8 * 8
    rows = torch.zeros(B, T, H, W, C8, device="cuda")
    rows[..., :Cc] = x_ncdhw.permute(0, 2, 3, 4, 1)
    pl = ops.Planes((B, T, H, W, C8 + coff + extra), bf16, "cuda", lo=lo)
    pl.hi.fill_(3.0)
    if lo:
        pl.lo.fill_(3.0)
    ops.split_into(rows.view(-1, C8), pl, 0, C8, out_coff=coff)
    return pl, C8


def _operands(ops, case, npass, bf16):
    """Seeded planes of one case and the float64 truth: (xp, Cp, dp, Cop, ref, ref_hi); ref_hi (single pass only) is
    the product of the hi planes alone."""
    name, Cin, Cout, k, p, B, T, H, W = case
    lo = npass > 1
    g = torch.Generator(device="cuda").manual_seed(sum(ord(ch) for ch in name))
    x = torch.relu(torch.randn(B, Cin, T, H, W, device="cuda", generator=g))
    dy = torch.randn(B, Cout, T, H, W, device="cuda", generator=g)
    xp, Cp = _planes(ops, x, bf16, lo, 8, 16)
    dp, Cop = _planes(ops, dy, bf16, lo, 16, 8)
    xv = xp.value()[..., 8:8 + Cin].permute(0, 4, 1, 2, 3).double()        # exact operand values
    dv = dp.value()[..., 16:16 + Cout].permute(0, 4, 1, 2, 3).double()
    wd = torch.zeros(Cout, Cin, *k, device="cuda", dtype=torch.float64, requires_grad=True)
    (ref,) = torch.autograd.grad(F.conv3d(xv, wd, padding=p), wd, dv)
    ref_hi = None
    if npass == 1:
        xh = xp.hi.float()[..., 8:8 + Cin].permute(0, 4, 1, 2, 3).double()
        dh = dp.hi.float()[..., 16:16 + Cout].permute(0, 4, 1, 2, 3).double()
        (ref_hi,) = torch.autograd.grad(F.conv3d(xh, wd, padding=p), wd, dh)
    return xp, Cp, dp, Cop, ref, ref_hi


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
@pytest.mark.parametrize("npass", [3, 1])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_wgrad_tma_vs_float64_and_gather(case, npass, fmt, diag):
    from coclr_b200 import ops, lib as L
    lib = L.load()
    name, Cin, Cout, k, p, B, T, H, W = case
    bf16 = int(fmt == "bf16")
    xp, Cp, dp, Cop, ref, ref_hi = _operands(ops, case, npass, bf16)
    geom = ops.Geometry(k, (1, 1, 1), p)
    out_scale = torch.tensor([0.25], device="cuda")
    res = {}
    for mode in (2, 0):      # 2: TMA-staged kernel (with its workspace); 0: gather kernel
        lib.coclr_set_wgrad_tma(int(mode > 0))
        dw = torch.full((Cout, Cin) + k, 0.5, device="cuda")                # accumulates on top of what is there
        wg = L.Wgrad(xp.src(8, Cp, T, H, W), geom.c(0), dp.src(16, Cop, T, H, W), B, T, H, W, Cout, Cin, L.dptr(dw), npass,
                     bf16, bf16, 3, L.dptr(out_scale))
        if mode == 2:
            need = int(lib.coclr_wgrad_ws_floats(C.byref(wg)))
            assert need > 0
            ws = torch.full((need,), float("nan"), device="cuda")           # every element read must have been written
            wg.ws, wg.ws_floats = L.dptr(ws).value, need
        if mode > 0:
            info = (C.c_int * 8)()
            assert lib.coclr_wgrad_tma_plan(C.byref(wg), info) == 1, "shape not on the TMA-staged kernel"
            diag["wgrad_tma/%s/p%d/plan%d" % (name, npass, mode)] = list(info)
        L.check(lib.coclr_conv_wgrad(C.byref(wg), L.stream_ptr()), "coclr_conv_wgrad")
        torch.cuda.synchronize()
        res[mode] = (dw - 0.5) * 4.0
    lib.coclr_set_wgrad_tma(1)
    e_ws, e_gather = _rel(res[2], ref), _rel(res[0], ref)
    diag["wgrad_tma/%s/p%d/%s" % (name, npass, fmt)] = [e_ws, e_gather]
    # operands are exact; what remains is fp32 accumulation over B*T*H*W pixels (3 passes) or the dropped lo planes
    tol = 2e-5 if npass == 3 else (2e-2 if bf16 else 4e-3)
    if npass == 1:   # single pass: the reference for the kernel is the product of the hi planes alone
        assert _rel(res[2], ref_hi) < 2e-5, (_rel(res[2], ref_hi), "tma vs hi-plane product")
    assert e_ws < tol and e_gather < tol, (e_ws, e_gather)
    # the workspace epilogue is deterministic: a second run gives the same bits
    dw2 = torch.full((Cout, Cin) + k, 0.5, device="cuda")
    wg.dw = L.dptr(dw2).value
    ws.fill_(float("nan"))
    wg.ws, wg.ws_floats = L.dptr(ws).value, ws.numel()
    L.check(lib.coclr_conv_wgrad(C.byref(wg), L.stream_ptr()), "coclr_conv_wgrad")
    torch.cuda.synchronize()
    assert torch.equal((dw2 - 0.5) * 4.0, res[2])


# Launches that share one workspace, in this order: the widest first, then a stacked (3 passes) or single-block (mb = 1,
# single pass) item, a (3,1,1) conv with several cout groups, and another small item after it
SHARED_WS = ["pw_832_384", "sp_16_48", "tm_ragged", "pw_24_40"]


@pytest.mark.parametrize("npass", [3, 1])
def test_wgrad_tma_shared_workspace(npass, diag):
    """The engine gives every weight gradient of a plan ONE workspace of the largest coclr_wgrad_ws_floats and runs them
    back to back on one stream, so each launch finds the partial sums of the launches before it (wider items, other
    row counts) where it does not write.  Each dW must be bit-equal to its run on a fresh NaN-poisoned workspace of
    exactly its own size, and within the float64 bound."""
    from coclr_b200 import ops, lib as L
    lib = L.load()
    by_name = {c[0]: c for c in CASES}
    out_scale = torch.tensor([0.25], device="cuda")
    runs = []
    for name in SHARED_WS:
        case = by_name[name]
        _, Cin, Cout, k, p, B, T, H, W = case
        xp, Cp, dp, Cop, ref, ref_hi = _operands(ops, case, npass, 0)
        geom = ops.Geometry(k, (1, 1, 1), p)
        dw_own = torch.full((Cout, Cin) + k, 0.5, device="cuda")
        wg = L.Wgrad(xp.src(8, Cp, T, H, W), geom.c(0), dp.src(16, Cop, T, H, W), B, T, H, W, Cout, Cin, L.dptr(dw_own),
                     npass, 0, 0, 1, L.dptr(out_scale))
        info = (C.c_int * 8)()
        assert lib.coclr_wgrad_tma_plan(C.byref(wg), info) == 1, name
        need = int(lib.coclr_wgrad_ws_floats(C.byref(wg)))
        own = torch.full((need,), float("nan"), device="cuda")
        wg.ws, wg.ws_floats = L.dptr(own).value, need
        L.check(lib.coclr_conv_wgrad(C.byref(wg), L.stream_ptr()), "coclr_conv_wgrad")
        runs.append((name, wg, need, list(info), dw_own, ref, ref_hi, (xp, dp, own)))
    torch.cuda.synchronize()
    mbs = [r[3][4] for r in runs]
    needs = [r[2] for r in runs]
    # a smaller item (stacked, or mb = 1) follows a wider one
    assert needs[0] == max(needs) and needs[1] < needs[0] and (mbs[1] == 1) == (npass == 1), (needs, mbs)
    shared = torch.full((max(needs) + 4096,), float("nan"), device="cuda")     # poisoned once, larger than any need
    outs = []
    for name, wg, need, info, dw_own, ref, ref_hi, _ in runs:
        dw = torch.full_like(dw_own, 0.5)
        wg.dw = L.dptr(dw).value
        wg.ws, wg.ws_floats = L.dptr(shared).value, shared.numel()
        L.check(lib.coclr_conv_wgrad(C.byref(wg), L.stream_ptr()), "coclr_conv_wgrad")
        outs.append(dw)
    torch.cuda.synchronize()
    for (name, wg, need, info, dw_own, ref, ref_hi, _), dw in zip(runs, outs):
        got = (dw - 0.5) * 4.0
        err = _rel(got, ref_hi if npass == 1 else ref)
        diag["wgrad_tma/shared_ws/%s/p%d" % (name, npass)] = [err, info[3], info[4]]
        assert torch.equal(dw, dw_own), (name, "differs from its run on its own workspace")
        assert err < 2e-5, (name, err)


def test_benchmark_shapes_take_the_tma_kernel():
    """Plan query only (no launch): every stride-1 conv of S3D at the benchmark shape (B=32, T=32, 128^2) is covered."""
    from coclr_b200 import ops, lib as L
    from coclr_b200.s3d_spec import S3D_INCEPTION
    lib = L.load()
    B = 32
    shapes = [(64, 64, (1, 1, 1), 16, 32, 32), (64, 192, (1, 3, 3), 16, 32, 32), (192, 192, (3, 1, 1), 16, 32, 32)]
    dims = {"Mixed_3": (16, 16, 16), "Mixed_4": (8, 8, 8), "Mixed_5": (4, 4, 4)}
    for name, (cin, (o0, o1a, o1b, o2a, o2b, o3b)) in S3D_INCEPTION.items():
        d = dims[name[:7]]
        shapes += [(cin, o0, (1, 1, 1)) + d, (cin, o1a + o2a, (1, 1, 1)) + d, (o1a, o1b, (1, 3, 3)) + d,
                   (o1b, o1b, (3, 1, 1)) + d, (o2a, o2b, (1, 3, 3)) + d, (o2b, o2b, (3, 1, 1)) + d, (cin, o3b, (1, 1, 1)) + d]
    dummy = torch.zeros(64, dtype=torch.float16, device="cuda")
    missed = []
    for cin, cout, k, T, H, W in shapes:
        c8, o8 = (cin + 7) // 8 * 8, (cout + 7) // 8 * 8
        geom = ops.Geometry(k, (1, 1, 1), tuple(v // 2 for v in k))
        src = L.Src(L.dptr(dummy), L.dptr(dummy), c8, 0, c8, T, H, W)
        dy = L.Src(L.dptr(dummy), L.dptr(dummy), o8, 0, o8, T, H, W)
        wg = L.Wgrad(src, geom.c(0), dy, B, T, H, W, cout, cin, L.dptr(dummy), 3, 0, 0, 1, None)
        if lib.coclr_wgrad_tma_plan(C.byref(wg), None) != 1:
            missed.append((cin, cout, k, T, H, W))
    # (1,3,3) convs on 4x4 frames would pad more than half of every 8x8 tile: those stay on the gather kernel
    assert all(k == (1, 3, 3) and H == 4 for _, _, k, _, H, _ in missed), missed


def _run_modes(lib, L, make_wg, dw_shape, diag, key):
    """TMA-staged kernel (mode 2) / gather kernel (mode 0) on the same struct; returns both results"""
    res = {}
    for mode in (2, 0):
        lib.coclr_set_wgrad_tma(int(mode > 0))
        dw = torch.zeros(dw_shape, device="cuda")
        wg = make_wg(dw)
        if mode == 2:
            need = int(lib.coclr_wgrad_ws_floats(C.byref(wg)))
            assert need > 0, "shape not on the TMA-staged kernel"
            ws = torch.full((need,), float("nan"), device="cuda")
            wg.ws, wg.ws_floats = L.dptr(ws).value, need
        if mode > 0:
            info = (C.c_int * 8)()
            assert lib.coclr_wgrad_tma_plan(C.byref(wg), info) == 1
            diag[key + "/plan%d" % mode] = list(info)
        L.check(lib.coclr_conv_wgrad(C.byref(wg), L.stream_ptr()), "coclr_conv_wgrad")
        torch.cuda.synchronize()
        res[mode] = dw
    lib.coclr_set_wgrad_tma(1)
    return res


@pytest.mark.parametrize("dims", [(1, 8, 16, 16), (2, 6, 10, 12)], ids=["even", "ragged"])
def test_wgrad_tma_temporal_stride2(dims, diag):
    """The stem's (7,1,1) conv with temporal stride 2 (backbone/s3dg.py:145 Conv_1a.conv2): frames split by parity in
    the tensor map, one halo slab per parity (taps dt = 0,2,4,6 and 1,3,5)."""
    from coclr_b200 import ops, lib as L
    lib = L.load()
    B, T, H, W = dims
    Cin = Cout = 64
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.relu(torch.randn(B, Cin, T, H, W, device="cuda", generator=g))
    geom = ops.Geometry((7, 1, 1), (2, 1, 1), (3, 0, 0))
    To, Ho, Wo = geom.out_dims(T, H, W)
    dy = torch.randn(B, Cout, To, Ho, Wo, device="cuda", generator=g)
    xp, Cp = _planes(ops, x, 0, True, 8, 16)
    dp, Cop = _planes(ops, dy, 0, True, 16, 8)
    xv = xp.value()[..., 8:8 + Cin].permute(0, 4, 1, 2, 3).double()
    dv = dp.value()[..., 16:16 + Cout].permute(0, 4, 1, 2, 3).double()
    wd = torch.zeros(Cout, Cin, 7, 1, 1, device="cuda", dtype=torch.float64, requires_grad=True)
    (ref,) = torch.autograd.grad(F.conv3d(xv, wd, stride=(2, 1, 1), padding=(3, 0, 0)), wd, dv)
    mk = lambda dw: L.Wgrad(xp.src(8, Cp, T, H, W), geom.c(0), dp.src(16, Cop, To, Ho, Wo), B, To, Ho, Wo, Cout, Cin,
                            L.dptr(dw), 3, 0, 0, 3, None)
    res = _run_modes(lib, L, mk, (Cout, Cin, 7, 1, 1), diag, "wgrad_tma/stem_tm_%d" % T)
    errs = [_rel(res[m], ref) for m in (2, 0)]
    diag["wgrad_tma/stem_tm_%d" % T] = errs
    assert max(errs) < 2e-5, errs


@pytest.mark.parametrize("dims", [(1, 2, 16, 16), (2, 3, 12, 24)], ids=["even", "ragged"])
def test_wgrad_tma_space_to_depth_window(dims, diag):
    """The space-to-depth stem as the engine launches it (backbone/s3dg.py:145 Conv_1a.conv1 as a stride-1 (1,4,4) conv
    over 16-channel pixels, rows zero-padded by 2 pixels on each side, pw = 0): one slab serves all 16 taps."""
    from coclr_b200 import ops, lib as L
    lib = L.load()
    B, T, H, W = dims
    Cout, Cin = 64, 12
    g = torch.Generator(device="cuda").manual_seed(6)
    xpl = ops.Planes((B, T, H, W + 4, 16), 0, "cuda", zero=True)
    vals = torch.randn(B, T, H, W, 12, device="cuda", generator=g)
    tmp = ops.Planes((B, T, H, W, 16), 0, "cuda", zero=True)
    rows = torch.zeros(B * T * H * W, 16, device="cuda")
    rows[:, :12] = vals.view(-1, 12)
    ops.split_into(rows, tmp)
    xpl.hi[:, :, :, 2:-2] = tmp.hi
    xpl.lo[:, :, :, 2:-2] = tmp.lo
    dy = torch.randn(B, Cout, T, H, W, device="cuda", generator=g)
    dp, Cop = _planes(ops, dy, 0, True, 0, 0)
    geom = ops.Geometry((1, 4, 4), (1, 1, 1), (0, 2, 0))
    xv = xpl.value()[..., :12].permute(0, 4, 1, 2, 3).double()              # [B, 12, T, H, W + 4]
    dv = dp.value()[..., :Cout].permute(0, 4, 1, 2, 3).double()
    wd = torch.zeros(Cout, Cin, 1, 4, 4, device="cuda", dtype=torch.float64, requires_grad=True)
    y = F.conv3d(xv, wd, padding=(0, 2, 0))[:, :, :, :H, :W]                # the H x W destination pixels the engine uses
    (ref,) = torch.autograd.grad(y, wd, dv)
    mk = lambda dw: L.Wgrad(xpl.src(0, 16, T, H, W + 4), geom.c(0), dp.src(0, Cop, T, H, W), B, T, H, W, Cout, Cin,
                            L.dptr(dw), 3, 0, 0, 3, None)
    res = _run_modes(lib, L, mk, (Cout, Cin, 1, 4, 4), diag, "wgrad_tma/s2d_%d" % W)
    errs = [_rel(res[m], ref) for m in (2, 0)]
    diag["wgrad_tma/s2d_%d" % W] = errs
    assert max(errs) < 2e-5, errs
