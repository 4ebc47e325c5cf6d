"""coclr_maxpool_bwd at the shapes the training plans run it at, and at shapes off its fast path.

The gradient of a max-pool is a sum, over the windows whose arg-max is an input element, of their dY.  The library adds
them from +0.0 in ascending tap order and adds the old dX last; an fp32 torch restatement of that order must give the
same bits, and float64 autograd of nn.MaxPool3d on the same input must agree to 1e-6.  idx comes from coclr_maxpool_fwd
over post-ReLU data, which has many exact ties at 0."""
import ctypes as C
import functools

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@functools.lru_cache(None)
def plan_pools(net):
    """(k, s, p, C, (Ti, Hi, Wi), accumulate) of every coclr_maxpool_bwd launch of `net`'s training plan for 32 x 128^2
    clips (a plan built over CPU tensors and never run; the shapes do not depend on the batch)."""
    from coclr_b200 import engine as E, lib as L
    from coclr_b200.r50_spec import r50_stages
    from coclr_b200.s3d_spec import s3d_stages
    L.DRY_RUN = True
    try:
        if net == "r50":
            g = E.Graph(r50_stages(3), 3, head_dim=128, feature_size=2048, bb_prefix="0.")
        else:
            g = E.Graph(s3d_stages(3), 3, head_dim=128, bb_prefix="0.")
        p = E.EncoderEngine(E.ParamStore(g, "cpu"), g, "parity").plan(2, 32, 128, 128, True, True)
        out = []
        for r in p.bwd:
            if r.fn.__name__ == "coclr_maxpool_bwd":
                o = r.args[0]._obj
                gm = o.g
                out.append(((gm.kt, gm.kh, gm.kw), (gm.st, gm.sh, gm.sw), (gm.pt, gm.ph, gm.pw), o.C,
                            (o.Ti, o.Hi, o.Wi), o.accumulate))
        return out
    finally:
        L.DRY_RUN = False


def restated_bwd(idx, dy, k, s, p, dims, old):
    """fp32 dX in the library's order: +0.0, then for each tap in ascending order the dY of the window whose arg-max it
    is (one window per tap and input element), then the old dX.  idx, dy: [B, To, Ho, Wo, C]."""
    B, To, Ho, Wo, Cc = dy.shape
    pad = [d + 2 * pp + kk for d, pp, kk in zip(dims, p, k)]
    acc = torch.zeros(B, *pad, Cc, device=dy.device)
    zero = torch.zeros((), device=dy.device)
    tap = 0
    for a in range(k[0]):
        for bb in range(k[1]):
            for cc in range(k[2]):
                acc[:, a:a + s[0] * To:s[0], bb:bb + s[1] * Ho:s[1], cc:cc + s[2] * Wo:s[2]] += \
                    torch.where(idx == tap, dy, zero)
                tap += 1
    T, H, W = dims
    out = acc[:, p[0]:p[0] + T, p[1]:p[1] + H, p[2]:p[2] + W]
    return out + old if old is not None else out


def run_pool(k, s, p, Cc, dims, acc, B=2, ld=None, coff=0, seed=7):
    from coclr_b200 import ops, lib as L
    g = torch.Generator(device="cuda").manual_seed(seed)
    T, H, W = dims
    ld = ld or Cc
    x = torch.relu(torch.randn(B, T, H, W, ld, device="cuda", generator=g))
    pl = ops.Planes((B, T, H, W, ld), 0, "cuda")
    pl.hi.copy_(x.half())
    pl.lo.copy_((x - pl.hi.float()).half())
    geom = ops.Geometry(k, s, p)
    To, Ho, Wo = geom.out_dims(T, H, W)
    out = ops.Planes((B, To, Ho, Wo, Cc), 0, "cuda")
    idx = torch.empty(B, To, Ho, Wo, Cc, dtype=torch.uint8, device="cuda")
    dy = torch.randn(B, To, Ho, Wo, Cc, device="cuda", generator=g)
    dx0 = torch.randn(B, T, H, W, ld, device="cuda", generator=g)
    dx = dx0.clone()
    pp = L.Pool(L.dptr(pl.hi), L.dptr(pl.lo), ld, coff, L.dptr(out.hi), L.dptr(out.lo), Cc, 0, None, None, L.dptr(idx),
                B, Cc, T, H, W, To, Ho, Wo, geom.c(0), L.dptr(dy), L.dptr(dx), acc)
    lib = L.load()
    L.check(lib.coclr_maxpool_fwd(C.byref(pp), L.stream_ptr()), "coclr_maxpool_fwd")
    L.check(lib.coclr_maxpool_bwd(C.byref(pp), L.stream_ptr()), "coclr_maxpool_bwd")
    torch.cuda.synchronize()
    got = dx[..., coff:coff + Cc]
    old = dx0[..., coff:coff + Cc] if acc else None
    # bit for bit against the restatement
    want = restated_bwd(idx.long(), dy, k, s, p, dims, old)
    assert torch.equal(got, want), float((got - want).abs().max())
    # channels outside the slice are untouched
    assert torch.equal(dx[..., :coff], dx0[..., :coff]) and torch.equal(dx[..., coff + Cc:], dx0[..., coff + Cc:])
    # float64 autograd of nn.MaxPool3d on the plane values
    xv = pl.value()[..., coff:coff + Cc].permute(0, 4, 1, 2, 3).double().requires_grad_(True)
    ref = F.max_pool3d(xv, k, s, p)
    (gref,) = torch.autograd.grad(ref, xv, dy.permute(0, 4, 1, 2, 3).double())
    gdx = (got.double() - (old.double() if acc else 0.0)).permute(0, 4, 1, 2, 3)
    e = float((gdx - gref).abs().max() / gref.abs().max())
    assert e < 1e-6, e


@pytest.mark.parametrize("i", range(13))
def test_pool_bwd_s3d_plan(i):
    """The 13 backward pools of the S3D training step: Inception branch-3 (3,3,3)/1 accumulated into the block input's
    gradient on 16^2, 8^2 and 4^2 frames, MaxPool_2a / MaxPool_3a (1,3,3)/(1,2,2), MaxPool_4a (3,3,3)/2, MaxPool_5a
    (2,2,2)/2, each with its real channel count and frames."""
    pools = plan_pools("s3d")
    assert len(pools) == 13
    k, s, p, Cc, dims, acc = pools[i]
    run_pool(k, s, p, Cc, dims, acc)


def test_pool_bwd_r50_stem():
    (pool,) = plan_pools("r50")
    k, s, p, Cc, dims, acc = pool
    run_pool(k, s, p, Cc, dims, acc)


WINDOWS = {"333s1": ((3, 3, 3), (1, 1, 1), (1, 1, 1)), "133s2": ((1, 3, 3), (1, 2, 2), (0, 1, 1)),
           "333s2": ((3, 3, 3), (2, 2, 2), (1, 1, 1))}


@pytest.mark.parametrize("acc", [1, 0], ids=["accumulate", "overwrite"])
@pytest.mark.parametrize("dims", [(5, 9, 11), (3, 7, 6), (4, 13, 24)], ids=["odd", "odd_h", "band_tail"])
@pytest.mark.parametrize("win", list(WINDOWS))
def test_pool_bwd_ragged(win, dims, acc):
    """Odd frame sizes: windows that hang over the last row / column / frame, bands of input rows cut short."""
    k, s, p = WINDOWS[win]
    run_pool(k, s, p, 32, dims, acc)


@pytest.mark.parametrize("coff", [8, 4], ids=["aligned", "unaligned"])
@pytest.mark.parametrize("win", list(WINDOWS))
def test_pool_bwd_channel_slice(win, coff):
    """A 48-channel slice of an 80-channel dX (ldx > C, x_coff != 0), accumulated: 8-aligned on the staged kernel,
    4-aligned on the generic one."""
    k, s, p = WINDOWS[win]
    run_pool(k, s, p, 48, (4, 8, 16), 1, ld=80, coff=coff)
