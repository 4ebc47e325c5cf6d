"""The stream schedule of the S3D, S3D-G and ResNet2d3d-50 launch plans (built over CPU tensors, never run): the lane
and wait of every launch, and the kernels each launch counts for."""
import pytest


@pytest.fixture
def dry_run():
    from coclr_b200 import lib as L
    L.DRY_RUN = True
    yield L
    L.DRY_RUN = False


def _engine(net):
    from coclr_b200 import engine as E
    from coclr_b200.r50_spec import r50_stages
    from coclr_b200.s3d_spec import s3d_stages
    if net == "r50":
        g = E.Graph(r50_stages(3), 3, head_dim=128, feature_size=2048, bb_prefix="0.")
    else:
        g = E.Graph(s3d_stages(3, gating=net == "s3dg"), 3, head_dim=128, bb_prefix="0.")
    return g, E.EncoderEngine(E.ParamStore(g, "cpu"), g, "parity")


def _mixed_schedule(block, name):
    """(lane, wait of the item's first launch) of an item of Mixed block `block`, from its name."""
    from coclr_b200.engine import FORK, AT_FORK, AFTER1, JOIN
    rest = name[len(block) + 1:]
    if name == block:                         # the concat BatchNorm (+ S3D-G gating): joins the branches
        return 0, JOIN
    if rest == "branch1.0.conv":              # the shared 1x1 conv of branches 1 and 2 opens the block
        return 1, FORK
    if rest == "b12a" or rest.startswith("branch1."):
        return 1, None
    if rest.startswith("branch2."):           # needs the shared conv's output
        return 2, AFTER1 if rest == "branch2.1.conv1" else None
    if rest.startswith("branch0."):
        return 0, None
    assert rest.startswith("branch3."), name  # the pool reads the block input only
    return 3, AT_FORK if rest == "branch3.0" else None


def _forward_items(g, p):
    """[(item name, its Launch records)] in forward order, then ("head", the head's records)."""
    out, i = [], 0
    for kind, it in g.items:
        n = 1 + (len(it.gates) + 2 if kind == "bn" and it.gates else 0)   # gating: mean, one fc per branch, apply
        out.append((it.name, p.fwd[i:i + n]))
        i += n
    return out + [("head", p.fwd[i:])]


# launch totals (forward, backward kernels) of a training step's query-encoder plan at the benchmark shape
TOTALS = {"s3d": (128, 306), "s3dg": (182, 396), "r50": (113, 268)}


@pytest.mark.parametrize("shape", [(2, 8, 64, 64), (32, 32, 128, 128)])
@pytest.mark.parametrize("net", ["s3d", "s3dg", "r50"])
def test_plan_schedule(dry_run, net, shape):
    from coclr_b200.engine import AFTER0
    L = dry_run
    g, eng = _engine(net)
    p = eng.plan(*shape, True, True)
    # ---- forward: the Inception branches of each Mixed block on lanes 1..3, everything else on lane 0 ----
    blocks = [it.name for kind, it in g.items if kind == "bn" and ".Mixed_" in it.name and "." not in
              it.name.split(".Mixed_")[1]]
    assert len(blocks) == (9 if net != "r50" else 0)
    for name, recs in _forward_items(g, p):
        assert recs, name
        block = [b for b in blocks if name == b or name.startswith(b + ".")]
        lane, wait = _mixed_schedule(block[0], name) if block else (0, None)
        assert [(r.lane, r.wait) for r in recs] == [(lane, wait)] + [(lane, None)] * (len(recs) - 1), name
    if net == "r50":
        assert all(r.lane == 0 and r.wait is None for r in p.fwd)
    # ---- backward: the weight gradients that share wg_ws on one side lane, everything else on lane 0 ----
    shared = [r for r in p.bwd if r.fn.__name__ == "coclr_conv_wgrad"]
    assert [r.args[0]._obj for r in shared] == p.wgrads
    assert all(w.ws == p.wg_ws.data_ptr() for w in p.wgrads)
    assert len({r.lane for r in shared}) == 1 and shared[0].lane != 0 and all(r.wait == AFTER0 for r in shared)
    stem = [r for r in p.bwd if r.fn.__name__ == "coclr_conv_wgrad_s2d"]
    assert len(stem) == 1 and (stem[0].lane, stem[0].wait) == (0, None)
    own = stem[0].args[0]._obj
    assert p.s2d_wgrads == [own]
    lo, hi = p.wg_ws.data_ptr(), p.wg_ws.data_ptr() + 4 * p.wg_ws.numel()
    assert not (lo <= (own.ws or 0) < hi) and not (own.ws and own.ws < lo < own.ws + 4 * own.ws_floats)
    side = {id(r) for r in shared + stem}
    assert all(r.lane == 0 and r.wait is None for r in p.bwd if id(r) not in side)
    # ---- kernel counts: the library's rule for each launch's arguments ----
    assert all(r.kernels == L.kernels_of(r.fn, r.args) for r in p.fwd + p.bwd)
    assert (p.fwd_kernels, p.bwd_kernels) == (sum(r.kernels for r in p.fwd), sum(r.kernels for r in p.bwd))
    # the space-to-depth stem's weight gradient: TMA partial sums + reduction for S3D, the gather kernel for R50
    assert stem[0].kernels == (1 if net == "r50" else 2)
    if shape == (32, 32, 128, 128):
        assert (p.fwd_kernels, p.bwd_kernels) == TOTALS[net]
    pk = eng.plan(*shape, True, False)   # forward-only (key encoder)
    assert not pk.bwd and pk.bwd_kernels == 0 and pk.fwd_kernels == p.fwd_kernels
