"""tests/pinned_oracle.py (the q encoder with its ReLU and max-pool decisions passed in) against the oracle it restates,
and its decision sites against the engine's graph.  No GPU needed.

1. With the decisions taken from its own float64 forward, the restatement is oracle/coclr_oracle.py: the same output
   bits, and parameter gradients within 1e-12.
2. Passed-in decisions are the ones used: one flipped mask element or one moved tap changes the output.
3. Its decision sites are the engine's (coclr_b200.engine.Graph), one to one: every BatchNorm member with a ReLU, every
   residual unit, every max-pool, and the head's ReLU.  A graph change that adds a site the restatement does not pin
   fails here, before the GPU test reads decisions out of a plan."""
import functools

import pytest
import torch
import torch.nn.functional as F

import pinned_oracle as PO
from oracle import coclr_oracle as O

NETS = ["s3d", "s3dg", "r50"]
B, T, HW, DIM = 2, 8, 32, 128


def _state(net):
    sd = O.synth_state(O.infonce_shapes(DIM, 128, network=net), seed=0)
    return {k: v for k, v in sd.items() if k.startswith("encoder_q.")}


def _copy(sd):
    """float64 copy; parameters require grad, BatchNorm buffers are private (the oracle updates them)."""
    out = {}
    for k, v in sd.items():
        t = v.detach().clone()
        if t.is_floating_point():
            t = t.double().requires_grad_(k.endswith(".weight") or k.endswith(".bias"))
        out[k] = t
    return out


def _inputs():
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, 3, T, HW, HW, generator=g, dtype=torch.float64)
    return x + 0.5 * torch.randn(B, 3, 1, 1, 1, generator=g, dtype=torch.float64)


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


@functools.lru_cache(maxsize=None)
def _recorded(net):
    """The restatement's output value and the decisions it recorded, from one forward without a graph; tests that
    differentiate run their own forward on a fresh copy of the state."""
    dec = PO.Decisions()
    with torch.no_grad():
        q = PO.query(_copy(_state(net)), "encoder_q.", _inputs(), dec)
    return q, dec


@pytest.mark.parametrize("net", NETS)
def test_restatement_is_the_oracle(net, diag):
    sdp, x = _copy(_state(net)), _inputs()
    q = PO.query(sdp, "encoder_q.", x, PO.Decisions())
    sdo = _copy(_state(net))
    h = O.encoder(sdo, "encoder_q.", x, True)
    qo = F.normalize(h, dim=1).view(B, -1)
    assert torch.equal(q, qo)
    seed = torch.randn(B, DIM, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    q.backward(seed)
    qo.backward(seed)
    keys = O.param_keys(sdo, "encoder_q.")
    errs = {k: _rel(sdp[k].grad, sdo[k].grad) for k in keys}
    diag["pinned_cpu/%s/max_grad_rel" % net] = max(errs.values())
    assert len(keys) == len([k for k in sdp if k.endswith(".weight") or k.endswith(".bias")])
    assert max(errs.values()) < 1e-12, sorted(errs.items(), key=lambda kv: -kv[1])[:5]
    # the pooled-backbone form (LinearClassifier's backbone) against the oracle's backbone + average pool
    sdp, sdo = _copy(_state(net)), _copy(_state(net))
    backbone = O.r2d3d50 if net == "r50" else O.s3d
    fo = F.adaptive_avg_pool3d(backbone(sdo, "encoder_q.0.", x, True), (1, 1, 1)).view(B, -1)
    fp = PO.pooled(sdp, "encoder_q.0.", x, PO.Decisions())
    assert torch.equal(fp, fo)
    seed = torch.randn(fo.shape, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    fo.backward(seed)
    fp.backward(seed)
    errs = {k: _rel(sdp[k].grad, sdo[k].grad) for k in keys if sdo[k].grad is not None}
    assert len(errs) == len(keys) - 4          # all but the head's two convs
    assert max(errs.values()) < 1e-12, sorted(errs.items(), key=lambda kv: -kv[1])[:5]


@pytest.mark.parametrize("net", ["s3dg", "r50"])
def test_passed_decisions_are_used(net):
    q, dec = _recorded(net)
    sd, x = _copy(_state(net)), _inputs()
    with torch.no_grad():
        assert torch.equal(PO.query(sd, "encoder_q.", x, PO.Decisions(dict(dec.masks), dict(dec.taps))), q)
        site = "Mixed_3c.branch1.1.bn1" if net == "s3dg" else "layer1.1.bn3"
        m = dec.masks[site].clone()
        m.view(-1)[m.view(-1).nonzero()[0]] = False            # one active element switched off
        q1 = PO.query(sd, "encoder_q.", x, PO.Decisions(dict(dec.masks, **{site: m}), dict(dec.taps)))
        assert not torch.equal(q1, q)
        pool = "MaxPool_3a" if net == "s3dg" else "maxpool"
        # every window's winner moved to the window centre (inside the input for these (1,3,3)/2 pools): a single moved
        # tap may land on an element equal to the winner (windows of a ReLU output often hold several zeros)
        tp = torch.full_like(dec.taps[pool], 4)
        assert not torch.equal(tp, dec.taps[pool])
        q2 = PO.query(sd, "encoder_q.", x, PO.Decisions(dict(dec.masks), dict(dec.taps, **{pool: tp})))
        assert not torch.equal(q2, q)


def _engine_sites(net, pooled):
    from backbone.select_backbone import select_backbone
    from coclr_b200.engine import Graph
    bb, param = select_backbone(net)
    if pooled:
        g, pre = Graph(bb._stages, bb.input_channel, feature_size=param["feature_size"], pooled=True), ""
    else:
        g, pre = Graph(bb._stages, bb.input_channel, head_dim=DIM, feature_size=param["feature_size"], bb_prefix="0."), "0."
    strip = lambda n: n[len(pre):] if n.startswith(pre) else n  # noqa: E731
    masks = {strip(nm) for t in g.tensors if t.pending and t.relu for nm, _, _ in t.bn_members}
    residual = {strip(nm) for t in g.tensors if t.residual is not None for nm, _, _ in t.bn_members}
    pools = {strip(it.name) for kind, it in g.items if kind == "pool"}
    if g.head_dim is not None:
        masks.add(PO.HEAD_RELU)
    return masks, residual, pools


@pytest.mark.parametrize("pooled", [False, True], ids=["head", "pooled"])
@pytest.mark.parametrize("net", NETS)
def test_decision_sites_match_the_engine_graph(net, pooled):
    if pooled:
        sd, x = _copy(_state(net)), _inputs()
        dec = PO.Decisions()
        with torch.no_grad():
            PO.pooled(sd, "encoder_q.0.", x, dec)
    else:
        dec = _recorded(net)[1]
    masks, residual, pools = _engine_sites(net, pooled)
    assert set(dec.masks) == masks, (sorted(masks - set(dec.masks)), sorted(set(dec.masks) - masks))
    assert dec.residual == residual, (sorted(residual ^ dec.residual))
    assert set(dec.taps) == pools, (sorted(pools ^ set(dec.taps)))
    assert len(residual) == (16 if net == "r50" else 0)
    assert len(pools) == (1 if net == "r50" else 4 + 9)
