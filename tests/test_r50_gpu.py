"""GPU parity of the InfoNCE step with the ResNet2d3d-50 backbone (BASELINE.json config 5, `--net r50`; SURVEY.md
row a14) through model.pretrain.InfoNCE -> C ABI, at a CPU-checkable shape (bs 4, 8 frames, 64x64, K=128), against
  (a) the golden vectors produced by the unmodified reference (tests/golden/infonce_r50.npz), and
  (b) the oracle (oracle/coclr_oracle.py) evaluated in float64 on the GPU as ground truth.
Tolerance on logits / loss / queue: 1e-3 relative (north star). Gradients: oracle-relative budget."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
pytestmark = pytest.mark.gpu

GOLD = os.path.join(ROOT, "tests", "golden", "infonce_r50.npz")


def _rel(a, b):
    a = torch.as_tensor(a).double().cpu()
    b = torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _rel_l2(a, b):
    a = torch.as_tensor(a).double().cpu()
    b = torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _build(precision="parity"):
    import make_golden as MG
    from model.pretrain import InfoNCE
    from oracle import coclr_oracle as O
    c = MG.R50_CFG
    torch.manual_seed(0)
    model = InfoNCE("r50", 128, c["K"], 0.999, 0.07, precision=precision)
    sd = O.synth_state(O.infonce_shapes(128, c["K"], network="r50"), seed=0, ptr=c["ptr"])
    model.load_state_dict(sd, strict=True)
    return model.cuda().train(), sd


def _oracle_truth(sd, block, idx, dtype, record=None):
    from oracle import coclr_oracle as O
    sdd = {}
    for k, v in sd.items():
        t = v.detach().clone().cuda()
        sdd[k] = t.to(dtype) if t.is_floating_point() else t
    for k in O.param_keys(sdd, "encoder_q."):
        sdd[k].requires_grad_(True)
    orig = O.bottleneck
    if record is not None:
        def rec(s, pre, x, stride, is3d, training):
            y = orig(s, pre, x, stride, is3d, training)
            record[pre] = y.detach()
            return y
        O.bottleneck = rec
    try:
        logits, labels = O.infonce_forward(sdd, [block.cuda().to(dtype)], idx)
    finally:
        O.bottleneck = orig
    loss = O.infonce_loss(logits[0], labels.cuda())
    loss.backward()
    return sdd, logits[0], loss


@pytest.fixture(scope="module")
def step():
    import make_golden as MG
    from coclr_b200 import moco
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    c = MG.R50_CFG
    model, sd = _build()
    block = MG.make_inputs_shifted(c["B"], c["T"], c["HW"]).cuda()
    torch.manual_seed(77)
    idx = torch.randperm(c["B"])
    torch.manual_seed(77)
    logits, labels = model(block)
    loss = moco.nce_cross_entropy(logits, labels)
    loss.backward()
    torch.cuda.synchronize()
    rec64 = {}
    truth = _oracle_truth(sd, block, idx, torch.float64, rec64)
    ref32 = _oracle_truth(sd, block, idx, torch.float32)
    return dict(model=model, sd=sd, logits=logits, labels=labels, loss=loss, truth=truth, ref32=ref32, rec64=rec64,
                block=block, cfg=c)


def test_r50_forward_matches_golden_and_truth(step, diag):
    gold = np.load(GOLD)
    logits, loss, model = step["logits"], step["loss"], step["model"]
    _, lg64, loss64 = step["truth"]
    e_gold, e_true = _rel(logits, gold["logits"]), _rel(logits, lg64)
    diag["r50/logits_vs_golden"] = e_gold
    diag["r50/logits_vs_fp64"] = e_true
    diag["r50/fp32oracle_vs_fp64"] = _rel(step["ref32"][1], lg64)
    diag["r50/loss"] = [float(loss), float(gold["loss"]), float(loss64)]
    assert logits.shape == (4, 129)
    assert e_gold < 1e-3 and e_true < 1e-3
    assert abs(float(loss) - float(gold["loss"])) < 1e-3 * max(1.0, abs(float(gold["loss"])))
    e_q = _rel(model.queue, gold["queue"])
    diag["r50/queue_vs_golden"] = e_q
    assert e_q < 1e-3
    assert int(model.queue_ptr) == int(gold["queue_ptr"][0]) == 20


def test_r50_side_effects(step, diag):
    gold = np.load(GOLD)
    msd = step["model"].state_dict()
    from make_golden import compact
    assert _rel(compact(msd["encoder_k.0.layer2.0.conv2.weight"].cpu().numpy())[0], gold["ema/encoder_k.0.layer2.0.conv2.weight"]) < 1e-6
    sd32 = step["ref32"][0]
    assert torch.equal(msd["encoder_k.0.layer2.0.conv2.weight"].cpu(), sd32["encoder_k.0.layer2.0.conv2.weight"].cpu())
    e1 = _rel(msd["encoder_q.0.layer1.0.downsample.1.running_mean"], gold["bn/encoder_q.0.layer1.0.downsample.1.running_mean"])
    e2 = _rel(msd["encoder_k.0.layer4.2.bn3.running_var"], gold["bn/encoder_k.0.layer4.2.bn3.running_var"])
    diag["r50/bn_running"] = [e1, e2]
    assert e1 < 1e-4 and e2 < 1e-3
    assert int(msd["encoder_q.0.layer3.2.bn2.num_batches_tracked"]) == 4


def test_r50_block_outputs(step, diag):
    """Output of each of the 16 bottlenecks (relu(bn3 + residual)) of encoder_q against the float64 oracle."""
    model, rec, c = step["model"], step["rec64"], step["cfg"]
    eng = model.encoder_q._engine
    plan = eng.plans[(c["B"], c["T"], c["HW"], c["HW"], True, True)]
    per = {}
    for t in eng.graph.tensors:
        if t.residual is None:
            continue
        y = plan.acts[t.index].pl.value()
        ref = rec["encoder_q." + t.name].permute(0, 2, 3, 4, 1)
        per[t.name] = _rel_l2(y, ref)
    assert len(per) == 16
    diag["r50/blocks"] = per
    assert max(per.values()) < 1e-3, per


def test_r50_gradients_oracle_relative(step, diag):
    import make_golden as MG
    model = step["model"]
    sd64, sd32 = step["truth"][0], step["ref32"][0]
    named = dict(model.named_parameters())
    out, bad = {}, []
    for k in sorted(sd64):
        if not k.startswith("encoder_q.") or not (k.endswith(".weight") or k.endswith(".bias")):
            continue
        g64 = sd64[k].grad
        e_new, e_ref = _rel_l2(named[k].grad, g64), _rel_l2(sd32[k].grad, g64)
        out[k] = [e_new, e_ref]
        if not e_new < 0.2:
            bad.append((k, e_new, e_ref))
    diag["r50/grad_err_new_vs_ref"] = out
    med_new = float(np.median([v[0] for v in out.values()]))
    med_ref = float(np.median([v[1] for v in out.values()]))
    diag["r50/grad_median_new_ref"] = [med_new, med_ref]
    assert med_new < 3 * med_ref + 1e-3, (med_new, med_ref)
    gold = np.load(GOLD)
    vs_gold = {}
    for k in MG.GRAD_KEYS_R50:
        got, _ = MG.compact(named[k].grad.cpu().numpy())
        vs_gold[k] = _rel_l2(got, gold["grad/" + k])
    diag["r50/grad_vs_golden"] = vs_gold
    assert not bad, bad[:5]


def test_r50_bare_backbone_forward(diag):
    """select_backbone('r50') used stand-alone (inference): [B,3,T,H,W] -> [B,2048,T/2,H/32,W/32], eval-mode BN."""
    from backbone.select_backbone import select_backbone
    from oracle import coclr_oracle as O
    net, param = select_backbone("r50")
    assert param["feature_size"] == 2048
    sd = {k[len("encoder_q.0."):]: v for k, v in O.synth_state(O.infonce_shapes(128, 128, network="r50"), seed=3).items()
          if k.startswith("encoder_q.0.")}
    net.load_state_dict(sd, strict=True)
    net = net.cuda().eval()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 3, 8, 64, 64, generator=g).cuda()
    with torch.no_grad():
        y = net(x)
    sdd = {k: (v.cuda().double() if v.is_floating_point() else v.cuda()) for k, v in sd.items()}
    ref = O.r2d3d50(sdd, "", x.double(), False)
    assert y.shape == (2, 2048, 4, 2, 2)
    e = _rel_l2(y, ref)
    diag["r50/bare_backbone_eval"] = e
    assert e < 1e-3
