"""The module layer over the engine on the H100: a backward whose saved activations were overwritten by a later training
forward of the same shape raises, for every module that runs on the engine; gradients accumulate over backward passes
without zero_grad, the S3D-G gating fc gradients included (coclr_gate_fc_bwd adds into dW / dbias)."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))

pytestmark = pytest.mark.gpu


def _clips(B=4, T=8, HW=64, seed=7):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 3, T, HW, HW, generator=g).cuda()


def _encoder(net):
    from model.pretrain import InfoNCE
    from oracle import coclr_oracle as O
    model = InfoNCE(net, 128, 128)
    model.load_state_dict(O.with_aliases(O.synth_state(O.infonce_shapes(128, 128, network=net), seed=0)))
    return model.cuda().train().encoder_q


def _classifier(net, replicas=1, use_dropout=True):
    from model.classifier import LinearClassifier
    import classifier_oracle as O
    m = LinearClassifier(num_class=51, network=net, dropout=0.9, use_dropout=use_dropout, replicas=replicas)
    m.load_state_dict(O.classifier_state(net, 51, use_dropout, False, seed=0), strict=False)
    return m.cuda().train()


# ---------------------------------------------------------------------------------------------------------------------
# stale activations
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["encoder", "classifier_r1", "classifier_r2"])
def test_backward_of_an_overwritten_pass_raises(kind):
    from coclr_b200 import lib as L
    x = _clips()
    if kind == "encoder":
        run = _encoder("s3d").encode
    else:
        model = _classifier("s3d", replicas=1 if kind == "classifier_r1" else 2)
        run = lambda clips: model(clips)[0]    # noqa: E731
    first = run(x)
    second = run(x)
    with pytest.raises(L.CoclrError, match="overwritten"):
        first.sum().backward()
    second.sum().backward()       # the pass that owns the activations still runs
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# gradient accumulation
# ---------------------------------------------------------------------------------------------------------------------
def _grads(module):
    return {k: p.grad.clone() for k, p in module.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("kind", ["encoder", "classifier"])
def test_two_backwards_without_zero_grad_accumulate(kind):
    """Forward + backward twice on the same clips: every gradient is exactly twice the one-pass gradient."""
    x = _clips()
    if kind == "encoder":
        module = _encoder("s3dg")
        w = torch.randn(x.shape[0], 128, generator=torch.Generator().manual_seed(3)).cuda()
        step = lambda: (module.encode(x) * w).sum().backward()    # noqa: E731
    else:
        module = _classifier("s3dg", use_dropout=False)
        y = torch.arange(x.shape[0]).cuda()
        step = lambda: torch.nn.functional.cross_entropy(module(x)[0], y).backward()    # noqa: E731
    module.zero_grad(set_to_none=True)
    step()
    once = _grads(module)
    step()
    twice = _grads(module)
    torch.cuda.synchronize()
    gating = [k for k in once if ".gating_b" in k]
    assert sorted(once) == sorted(twice) and len(gating) == 2 * 4 * 9
    assert all(once[k].abs().max() > 0 for k in gating)
    for k in once:
        assert torch.equal(twice[k], 2 * once[k]), (k, float((twice[k] - 2 * once[k]).abs().max()))


def test_gate_fc_bwd_accumulates():
    from coclr_b200 import lib as L
    lib = L.load()
    g = torch.Generator().manual_seed(11)
    B, C, coff, n = 3, 96, 32, 40
    dgate, mean = (torch.randn(B, C, generator=g).cuda() for _ in range(2))
    gate = torch.rand(B, C, generator=g).cuda()
    W = torch.randn(n, n, generator=g).cuda()
    dW, db, dmean = torch.zeros(n, n, device="cuda"), torch.zeros(n, device="cuda"), torch.zeros(B, C, device="cuda")

    def call():
        L.check(lib.coclr_gate_fc_bwd(L.dptr(dgate), L.dptr(gate), L.dptr(mean), L.dptr(W), L.dptr(dW), L.dptr(db),
                                      L.dptr(dmean), B, C, coff, n, L.stream_ptr()), "coclr_gate_fc_bwd")
    call()
    once = [dW.clone(), db.clone(), dmean.clone()]
    call()
    torch.cuda.synchronize()
    assert torch.equal(dW, 2 * once[0]) and torch.equal(db, 2 * once[1])
    assert torch.equal(dmean, once[2])     # the data gradient is written, not accumulated
