"""Max-pool straight from a BatchNorm's conv output (coclr_affine_split as a finalize-only call, then coclr_maxpool_fwd
with coclr_pool_t.y) against the sequence it replaces -- coclr_affine_split writing the planes, then coclr_maxpool_fwd
over them -- bit for bit, and against float64: the pooled values are the exact maxima of the values the planes hold."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

POOL_133 = ((1, 3, 3), (1, 2, 2), (0, 1, 1))
POOL_333 = ((3, 3, 3), (2, 2, 2), (1, 1, 1))
POOL_222 = ((2, 2, 2), (2, 2, 2), (0, 0, 0))

# (id, (B, T, H, W, C), pool): the S3D stage pools and the ResNet stem pool at small batch, then ragged frames that
# take the register-only kernel instead of the shared-memory tile
CASES = [
    ("MaxPool_2a", (2, 2, 64, 64, 64), POOL_133),
    ("MaxPool_3a", (2, 2, 32, 32, 192), POOL_133),
    ("MaxPool_4a", (2, 8, 16, 16, 480), POOL_333),
    ("MaxPool_5a", (2, 4, 8, 8, 832), POOL_222),
    ("r50_maxpool", (2, 4, 32, 32, 64), POOL_133),
    ("ragged_133", (2, 3, 13, 11, 192), POOL_133),
    ("ragged_333", (1, 5, 9, 7, 480), POOL_333),
    ("ragged_222", (1, 5, 7, 9, 832), POOL_222),
]


def _inputs(shape, mode, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    B, T, H, W, Cc = shape
    y = torch.randn(B, T, H, W, Cc, device="cuda", generator=g) * 2 + 0.3
    gamma = torch.rand(Cc, device="cuda", generator=g) + 0.5
    beta = torch.randn(Cc, device="cuda", generator=g)
    if mode == "const_rows":        # every pixel of a frame row equal: each window is one big tie
        y = y[:, :, :, :1, :].expand(B, T, H, W, Cc).contiguous()
    elif mode == "all_negative":    # relu(bn(y)) == 0 everywhere: every window ties at 0
        beta = beta.abs() * 0 - 20.0
    return y, gamma, beta


class _Bn:
    """Statistics, parameters and outputs of one BatchNorm call (fresh copies of the running stats)."""

    def __init__(self, y, gamma, beta, rm, rv):
        from coclr_b200 import lib as L
        Cc = y.shape[-1]
        rows = y.view(-1, Cc).double()
        self.ssum, self.ssq = rows.sum(0).contiguous(), (rows * rows).sum(0).contiguous()
        self.rm, self.rv = rm.clone(), rv.clone()
        self.scale, self.shift, self.mean, self.rstd = (torch.zeros(Cc, device="cuda") for _ in range(4))
        self.c = L.BnFinalize(L.dptr(self.ssum), L.dptr(self.ssq), rows.shape[0], L.dptr(gamma), L.dptr(beta),
                              L.dptr(self.rm), L.dptr(self.rv), 0.1, 1e-5, 1, L.dptr(self.scale), L.dptr(self.shift),
                              L.dptr(self.mean), L.dptr(self.rstd), Cc)

    def split(self, y, planes):
        """coclr_affine_split with the fused finalize: planes, or (planes None) the finalize alone."""
        from coclr_b200 import lib as L
        Cc = y.shape[-1]
        sp = L.Split(L.dptr(y), Cc, 0, Cc, y.numel() // Cc, None, None, 1,
                     L.dptr(planes.hi) if planes is not None else None, L.dptr(planes.lo) if planes is not None else None,
                     Cc, 0, 0, None, None, self.c)
        L.check(L.load().coclr_affine_split(C.byref(sp), L.num_sms(), L.stream_ptr()), "coclr_affine_split")


def _pool(L, ops, x_pl, out, idx, shape, k, s, p, bn=None, y=None):
    B, T, H, W, Cc = shape
    geom = ops.Geometry(k, s, p)
    To, Ho, Wo = geom.out_dims(T, H, W)
    pl = L.Pool(L.dptr(x_pl.hi) if x_pl is not None else None, L.dptr(x_pl.lo) if x_pl is not None else None, Cc, 0,
                L.dptr(out.hi), L.dptr(out.lo), Cc, 0, None, None, L.dptr(idx), B, Cc, T, H, W, To, Ho, Wo, geom.c(0),
                None, None, 0)
    if y is not None:
        pl.y, pl.scale, pl.shift, pl.relu = L.dptr(y), L.dptr(bn.scale), L.dptr(bn.shift), 1
    return L.load().coclr_maxpool_fwd(C.byref(pl), L.stream_ptr())


def _bits_equal(a, b):
    as_int = {torch.float16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}
    return a.dtype == b.dtype and torch.equal(a.view(as_int[a.dtype]), b.view(as_int[b.dtype]))


@pytest.mark.parametrize("mode", ["random", "const_rows", "all_negative"])
@pytest.mark.parametrize("name,shape,pool", CASES, ids=[c[0] for c in CASES])
def test_pool_from_conv_output_bit_equal(name, shape, pool, mode, diag):
    from coclr_b200 import lib as L, ops
    k, s, p = pool
    B, T, H, W, Cc = shape
    To, Ho, Wo = ops.Geometry(k, s, p).out_dims(T, H, W)
    y, gamma, beta = _inputs(shape, mode, seed=[c[0] for c in CASES].index(name) * 3 + len(mode))
    rm0 = torch.randn(Cc, device="cuda") * 0.1
    rv0 = torch.rand(Cc, device="cuda") + 0.5

    # ---- the planes, then the pool over them ----
    bn_u = _Bn(y, gamma, beta, rm0, rv0)
    pre = ops.Planes(shape, 0, "cuda")
    bn_u.split(y, pre)
    out_u = ops.Planes((B, To, Ho, Wo, Cc), 0, "cuda")
    idx_u = torch.empty(B * To * Ho * Wo * Cc, dtype=torch.uint8, device="cuda")
    L.check(_pool(L, ops, pre, out_u, idx_u, shape, k, s, p), "coclr_maxpool_fwd")

    # ---- the finalize alone, then the pool from y: with idx (query encoder) and without (key encoder) ----
    outs = []
    for with_idx in (True, False):
        bn = _Bn(y, gamma, beta, rm0, rv0)
        bn.split(y, None)
        out = ops.Planes((B, To, Ho, Wo, Cc), 0, "cuda")
        idx = torch.full_like(idx_u, 255) if with_idx else None
        L.check(_pool(L, ops, None, out, idx, shape, k, s, p, bn=bn, y=y), "coclr_maxpool_fwd")
        outs.append((bn, out, idx))
    torch.cuda.synchronize()
    for bn, out, idx in outs:
        assert _bits_equal(out.hi, out_u.hi) and _bits_equal(out.lo, out_u.lo)
        assert idx is None or torch.equal(idx, idx_u)
        for a, b in ((bn.rm, bn_u.rm), (bn.rv, bn_u.rv), (bn.scale, bn_u.scale), (bn.shift, bn_u.shift),
                     (bn.mean, bn_u.mean), (bn.rstd, bn_u.rstd)):
            assert _bits_equal(a, b)
    out_f = outs[0][1]
    if mode == "all_negative":
        assert float(out_f.value().abs().max()) == 0.0

    # ---- float64: the pooled values are the maxima of the values the planes hold, and those are relu(bn(y)) ----
    xv = pre.value().permute(0, 4, 1, 2, 3).double()
    assert torch.equal(F.max_pool3d(xv, k, s, p).permute(0, 2, 3, 4, 1), out_f.value().double())
    a64 = torch.relu(F.batch_norm(y.double().permute(0, 4, 1, 2, 3), None, None, gamma.double(), beta.double(), True,
                                  0.1, 1e-5))
    ref = F.max_pool3d(a64, k, s, p).permute(0, 2, 3, 4, 1)
    err = float((out_f.value().double() - ref).abs().max() / ref.abs().max().clamp_min(1.0))
    diag["pool_from_conv_output/%s/%s" % (name, mode)] = err
    assert err < 1e-5, err


def test_pool_from_conv_output_rejects_other_windows():
    """The conv-output form takes only the windows it is instantiated for; anything else is an argument error."""
    from coclr_b200 import lib as L, ops
    k, s, p = (3, 3, 3), (1, 1, 1), (1, 1, 1)
    shape = (1, 4, 8, 8, 64)
    y, gamma, beta = _inputs(shape, "random", 1)
    bn = _Bn(y, gamma, beta, torch.zeros(64, device="cuda"), torch.ones(64, device="cuda"))
    bn.split(y, None)
    out = ops.Planes((1, 4, 8, 8, 64), 0, "cuda")
    assert _pool(L, ops, None, out, None, shape, k, s, p, bn=bn, y=y) == -1     # COCLR_E_ARG
