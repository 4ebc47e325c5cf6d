"""Which max-pools of the S3D, S3D-G and ResNet2d3d-50 plans read their input's conv output directly (launch lists
built over CPU tensors, never run)."""
import pytest
import torch


def _plan(net, precision="parity", with_backward=True):
    from coclr_b200.engine import Graph, ParamStore, EncoderEngine
    from coclr_b200.r50_spec import r50_stages
    from coclr_b200.s3d_spec import s3d_stages
    if net == "r50":
        g = Graph(r50_stages(3), 3, head_dim=128, feature_size=2048, bb_prefix="0.")
    else:
        g = Graph(s3d_stages(3, gating=net == "s3dg"), 3, head_dim=128, bb_prefix="0.")
    st = ParamStore(g, torch.device("cpu"))
    eng = EncoderEngine(st, g, precision)
    return g, st, eng, eng.plan(2, 8, 64, 64, True, with_backward)


@pytest.fixture
def dry_run():
    from coclr_b200 import lib as L
    L.DRY_RUN = True
    yield L
    L.DRY_RUN = False


@pytest.mark.parametrize("net,precision,want", [
    ("s3d", "parity", ["0.MaxPool_2a", "0.MaxPool_3a", "0.MaxPool_4a", "0.MaxPool_5a"]),
    ("s3d", "mixed", ["0.MaxPool_2a", "0.MaxPool_3a", "0.MaxPool_4a", "0.MaxPool_5a"]),
    ("s3dg", "parity", ["0.MaxPool_2a", "0.MaxPool_3a"]),     # MaxPool_4a / 5a read gated block outputs
    ("r50", "parity", ["0.maxpool"]),
    ("s3d", "fast", []),                                      # bf16 planes: the pool splits y into fp16 pairs
])
def test_fused_pools_store_no_pre_pool_planes(dry_run, net, precision, want):
    """Which pools read their input's conv output, and that such an input allocates no operand planes: its BatchNorm
    item is a finalize-only coclr_affine_split (no planes), the pool's coclr_maxpool_fwd carries y / scale / shift."""
    from coclr_b200.engine import _PoolInputView
    g, st, eng, p = _plan(net, precision)
    assert sorted(p.fused_pools) == sorted(want)
    pools = {it.name: it for kind, it in g.items if kind == "pool"}
    for kind, it in g.items:   # the Inception branch-3 pools read a tensor the branch convolutions read too
        if kind == "pool" and ".branch3." in it.name:
            assert it.name not in p.fused_pools
    fwd = [(fn.__name__, a[0]._obj) for fn, a in p.fwd if fn.__name__ in ("coclr_affine_split", "coclr_maxpool_fwd")]
    for name, it in pools.items():
        src, dst = p.acts[it.src.index], p.acts[it.dst.index]
        pool = [o for n, o in fwd if n == "coclr_maxpool_fwd" and o.y_hi == dst.pl.hi.data_ptr()]
        splits = [o for n, o in fwd if n == "coclr_affine_split" and src.data is not None and o.x == src.data.data_ptr()]
        assert len(pool) == 1, name
        if name in want:
            assert isinstance(src.pl, _PoolInputView) and src.grad is not None, name
            assert pool[0].y == src.data.data_ptr() and not pool[0].x_hi and pool[0].scale == src.scale.data_ptr()
            assert len(splits) == 1 and not splits[0].hi and splits[0].bn.scale == src.scale.data_ptr()
        else:
            assert not isinstance(src.pl, _PoolInputView) and not pool[0].y, name
            assert pool[0].x_hi == src.pl.hi.data_ptr()
