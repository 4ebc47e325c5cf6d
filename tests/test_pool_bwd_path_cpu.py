"""Which form of the max-pool backward the training plans get (coclr_maxpool_bwd_path: host logic, nothing launched).
The staged and grid-stride gathers give the same bits, so only this tells them apart: every overlapping-window pool
of the S3D, S3D-G and ResNet2d3d-50 plans must take the shared-memory staged kernel, and disjoint windows the scatter."""
import ctypes as C

import pytest

SCATTER, GATHER, STAGED = 0, 1, 2


@pytest.fixture
def dry_run():
    from coclr_b200 import lib as L
    L.DRY_RUN = True
    yield L
    L.DRY_RUN = False


def _plan(net, shape):
    from coclr_b200 import engine as E
    from coclr_b200.r50_spec import r50_stages
    from coclr_b200.s3d_spec import s3d_stages
    if net == "r50":
        g = E.Graph(r50_stages(3), 3, head_dim=128, feature_size=2048, bb_prefix="0.")
    else:
        g = E.Graph(s3d_stages(3, gating=net == "s3dg"), 3, head_dim=128, bb_prefix="0.")
    return E.EncoderEngine(E.ParamStore(g, "cpu"), g, "parity").plan(*shape, True, True)


@pytest.mark.parametrize("shape", [(2, 8, 64, 64), (32, 32, 128, 128)])
@pytest.mark.parametrize("net", ["s3d", "s3dg", "r50"])
def test_plan_pools_take_the_staged_backward(dry_run, net, shape):
    lib = dry_run.load()
    paths = []
    for r in _plan(net, shape).bwd:
        if r.fn.__name__ == "coclr_maxpool_bwd":
            o = r.args[0]._obj
            disjoint = o.g.st >= o.g.kt and o.g.sh >= o.g.kh and o.g.sw >= o.g.kw
            paths.append((lib.coclr_maxpool_bwd_path(r.args[0]), SCATTER if disjoint else STAGED))
    assert paths and all(got == want for got, want in paths), paths
    if net != "r50":
        assert [w for _, w in paths].count(STAGED) == 12


def _pool(k, s, p, Cc, dims, ldx=None, x_coff=0, acc=1):
    from coclr_b200 import lib as L, ops
    geom = ops.Geometry(k, s, p)
    To, Ho, Wo = geom.out_dims(*dims)
    return L.Pool(None, None, ldx or Cc, x_coff, None, None, Cc, 0, None, None, None, 2, Cc, *dims, To, Ho, Wo,
                  geom.c(0), None, None, acc)


@pytest.mark.parametrize("case,want", [
    (dict(Cc=40), GATHER),                         # not whole 16-channel slices
    (dict(Cc=48, ldx=80, x_coff=4), GATHER),       # dX rows not 8-aligned
    (dict(Cc=48, ldx=80, x_coff=8), STAGED),
    (dict(Cc=32, dims=(4, 8, 160)), GATHER),       # more than 256 threads for one input row
], ids=["C40", "coff4", "coff8", "W160"])
def test_staged_backward_conditions(case, want):
    from coclr_b200 import lib as L
    lib = L.load()
    for k, s, p in (((3, 3, 3), (1, 1, 1), (1, 1, 1)), ((1, 3, 3), (1, 2, 2), (0, 1, 1)), ((3, 3, 3), (2, 2, 2), (1, 1, 1))):
        args = dict(dims=(4, 8, 16))
        args.update(case)
        assert lib.coclr_maxpool_bwd_path(C.byref(_pool(k, s, p, **args))) == want, (k, case)
    # disjoint windows: the scatter form; and the generic gather when the destination is a slice it cannot memset
    assert lib.coclr_maxpool_bwd_path(C.byref(_pool((2, 2, 2), (2, 2, 2), (0, 0, 0), 32, (4, 8, 8), acc=0))) == SCATTER
    assert lib.coclr_maxpool_bwd_path(C.byref(_pool((2, 2, 2), (2, 2, 2), (0, 0, 0), 32, (4, 8, 8), ldx=48,
                                                    acc=0))) == GATHER
