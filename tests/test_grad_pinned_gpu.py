"""Every encoder gradient of one training step against float64, tensor by tensor, with the engine's own decisions.

The end-to-end gradient tests (test_infonce_gpu.py, test_cfg2_gpu.py, test_s3dg_gpu.py, test_r50_gpu.py,
test_classifier_gpu.py) compare against the float64 oracle as it decides for itself, and so bound medians and allow
exceptions: where the engine and float64 put a pre-ReLU value on different sides of zero, or pick different tied
elements of a max-pool window, they differentiate different functions.  Here the float64 encoder
(tests/pinned_oracle.py) is evaluated with the ReLU masks and max-pool taps read out of the engine's plan after the
step, and its backward is seeded with the engine's own cotangent (plan.dq for the pre-training step, plan.dfeat for the
fine-tune step).  What is left between the two is the engine's arithmetic, so every tensor gets a bound:

1. every parameter gradient of the encoder (all of them, counted against named_parameters) within the budget; the only
   exceptions are named, with their reason; the same float32 computation with TF32 off is the yardstick beside it;
2. layer by layer, for localisation: the fp32 dA of every BatchNorm member (for gated tensors d/d(un-gated activation),
   after coclr_gate_bwd_apply) and its dY planes x dy_scale[1] against the float64 gradients at the same points;
3. the forward: every conv output (fp32, pre-BatchNorm) and every activation plane against the pinned float64 forward;
4. plan.dq against the float64 gradient of the mean InfoNCE loss at the engine's own q, k (the B queue columns the
   step enqueued) and pre-step queue, T = 0.07, which closes the chain loss -> dq -> every gradient.

The decisions are checked as they are read: a mask is [fmaf(y, scale, shift) (+ r) > 0] as coclr_bn_bwd forms it, and
where it disagrees with [plane > 0] the value is below the planes' resolution (2^-24); each max-pool tap must pick the
window maximum of the engine's own input planes exactly, and the float64 window maximum to within twice the forward
error of that input.

Measured on one H100 80GB HBM3 (700 W power limit); relative L2 error per tensor against the pinned float64 gradient,
max / median over the tensors, this engine and the same computation in float32 torch:

  case           tensors  engine           float32 torch    layerwise max  forward max  dq      peak     wall
  s3d_cfg1       235      1.09e-4 / 6.2e-5  2.3e-4 / 1.3e-4  6.7e-5         8.2e-5       2.2e-4  1.7 GB   12 s
  s3d_cfg2 (B32) 235      1.66e-4 / 5.1e-5  2.0e-4 / 1.0e-4  5.1e-5         9.0e-5       2.0e-5  41.3 GB  3 s
  s3dg           307      6.5e-5 / 4.4e-5   1.2e-4 / 7.6e-5  4.7e-5         6.0e-5       7.8e-5  1.9 GB   2 s
  r50            163      4.7e-5 / 2.6e-5   1.3e-4 / 7.2e-5  2.6e-5         3.0e-5       6.1e-4  2.2 GB   3 s
  s3d_finetune   231      5.5e-5 / 2.9e-5   1.3e-4 / 6.3e-5  3.4e-5         5.8e-5       -       1.4 GB   2 s
  s3d_mixed      235      1.4e-2 / 3.0e-3   2.3e-4 / 1.3e-4  3.6e-3         8.2e-5       2.2e-4  1.7 GB   1 s

(s3d_cfg1's wall time includes loading the library.)  The floor is not the backward's arithmetic (fp16 hi/lo products,
~2^-22) but the forward's: the engine differentiates at its own fp32-grade activations, which at the last Inception
blocks are 5e-5 to 9e-5 off float64 (BatchNorm over 64 samples per channel at config 1), and every gradient below them
inherits that.  float32 torch, run with the same decisions and cotangent, is off by twice as much.

Budget: `parity` 1e-4 per tensor.  Seven tensors, named in GRAD_EXCEPTIONS, cannot meet it because of cancellation:
BatchNorm weight and bias gradients, sums over the batch whose terms cancel, which float32 torch gets wrong by as much.
Only those may be off by 4x float32 torch's error for the same tensor: s3d_cfg1 Mixed_5c.branch2.0.bn.weight (1.09e-4,
float32 torch 1.8e-4); s3d_cfg2 Conv_1a.bn2.bias (1.66e-4 / 1.35e-4), Mixed_3c.branch0.0.bn.bias, .branch1.1.bn2.bias,
.branch2.1.bn2.bias (1.0-1.3e-4 / 0.9-1.2e-4), Mixed_5b.branch2.1.bn2.weight and Mixed_5c.branch2.1.bn1.weight (1.0e-4
/ 1.8-2.0e-4).  `mixed` (single-pass fp16 dY, 11 bits): 4e-2 per tensor.  Layerwise dA / dY: 2e-4 (`mixed` 1e-2).
Forward: 3e-4.  Logits at the engine's q, k and queue: 1e-5 (measured 1.5-2.0e-7).  dq: DQ_ULPS below.

Max-pool taps: in the engine's own planes every tap is the window maximum exactly, in every case.  In float64 the picked
element can sit below the window maximum where two elements are within the forward error of each other: at most 2.6e-4
(s3d_cfg2 Mixed_5c.branch3.0, 3.6e-5 of that input's largest value), 0.57x the input's largest forward error; 2.2e-5 at
config 1 and in the fine-tune step, 5.6e-6 for S3D-G, 0 for ResNet-50.  The bound is 2x the input's forward error.

A wiring fault shows up at 1e-2 to 1: zeroing the mean term of Mixed_4d's gating backward in S3D-G puts 0.05-0.61 on
167 of the 307 tensors, everything from Mixed_4d down to the stem.
"""
import gc
import os
import sys
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pinned_oracle as PO
from oracle import coclr_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
pytestmark = pytest.mark.gpu

# case -> (network, form, precision, (B, T, HW))
CASES = {
    "s3d_cfg1": ("s3d", "infonce", "parity", (4, 8, 128)),
    "s3d_cfg2": ("s3d", "infonce", "parity", (32, 32, 128)),
    "s3dg": ("s3dg", "infonce", "parity", (4, 8, 128)),
    "r50": ("r50", "infonce", "parity", (4, 8, 64)),
    "s3d_finetune": ("s3d", "finetune", "parity", (4, 8, 128)),
    "s3d_mixed": ("s3d", "infonce", "mixed", (4, 8, 128)),
}
GRAD_BUDGET = {"parity": 1e-4, "mixed": 4e-2}
LAYER_BUDGET = {"parity": 2e-4, "mixed": 1e-2}
# the tensors that cannot meet the parity budget: BatchNorm weight / bias gradients, sum(dz * xhat) and sum(dz) over the
# batch, whose terms cancel, so the forward's fp32-grade error in dz and xhat is amplified past 1e-4 -- in float32 torch
# under the same decisions as much as here.  Their bound is FP32_FACTOR x that float32 run's error for the same tensor;
# every other tensor has the flat budget.  Measured (engine / float32 torch) in the comments.
FP32_FACTOR = 4
_CANCEL = "BatchNorm %s gradient: a sum over the batch whose terms cancel"
GRAD_EXCEPTIONS = {
    "s3d_cfg1": {
        "encoder_q.0.Mixed_5c.branch2.0.bn.weight": _CANCEL % "weight",      # 1.09e-4 / 1.77e-4 (64 samples per channel)
    },
    "s3d_cfg2": {
        "encoder_q.0.Conv_1a.bn2.bias": _CANCEL % "bias",                   # 1.66e-4 / 1.35e-4
        "encoder_q.0.Mixed_3c.branch0.0.bn.bias": _CANCEL % "bias",         # 1.03e-4 / 0.96e-4
        "encoder_q.0.Mixed_3c.branch1.1.bn2.bias": _CANCEL % "bias",        # 1.28e-4 / 1.18e-4
        "encoder_q.0.Mixed_3c.branch2.1.bn2.bias": _CANCEL % "bias",        # 1.07e-4 / 0.88e-4
        "encoder_q.0.Mixed_5b.branch2.1.bn2.weight": _CANCEL % "weight",    # 1.01e-4 / 1.83e-4
        "encoder_q.0.Mixed_5c.branch2.1.bn1.weight": _CANCEL % "weight",    # 1.02e-4 / 2.00e-4
    },
}
LOGITS_BUDGET = 1e-5   # the engine's logits against float64 at its own q, k and queue (measured 1.5-2.0e-7)
FWD_BUDGET = 3e-4
# the positive's logit gradient p_pos - 1 comes out of fp32 with an error of a few ulps of 1, while dq scales with
# 1 - p_pos (root mean square over the batch): dq's relative error is a few 2^-24 / (1 - p_pos), about 1e-4 at
# 1 - p_pos ~ 1e-3; measured 5-17 such units
DQ_ULPS = 48
PLANE_RES = 2.0 ** -24      # smallest fp16 subnormal: a positive value below it leaves both planes zero


def _rel_l2(a, b):
    """Relative L2 error of `a` against `b`, on the device, in float64."""
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _ncdhw(t):
    return t.permute(0, 4, 1, 2, 3)


def _planes(a, coff, c):
    """fp32 value of channels [coff, coff + c) of an activation's operand planes, channels-last."""
    pl = a.pl
    if not hasattr(pl, "hi"):              # a pool that reads the conv output itself: its planes are recomputed
        return pl.value()[..., coff:coff + c]
    v = pl.hi[..., coff:coff + c].float()
    return v + pl.lo[..., coff:coff + c].float() if pl.lo is not None else v


def _dy(a, coff, c):
    """dY = (hi + lo) x dy_scale[1]: the gradient planes coclr_bn_bwd wrote, unscaled."""
    v = a.dy.hi[..., coff:coff + c].float()
    if a.dy.lo is not None:
        v = v + a.dy.lo[..., coff:coff + c].float()
    return v * a.dy_scale[1]


# ---------------------------------------------------------------------------------------------------------------------
# one training step of the engine
# ---------------------------------------------------------------------------------------------------------------------
def _step(case):
    import make_golden as MG
    from coclr_b200 import moco
    net, form, precision, (B, T, HW) = CASES[case]
    out = dict(case=case, precision=precision, form=form, B=B)
    if form == "finetune":
        from test_classifier_gpu import _clips, _model
        model, sd = _model(net, 101, "ft")
        model.train()
        x, y = _clips(B, T, HW, 101)
        torch.manual_seed(5)
        logit, _ = model(x)
        F.cross_entropy(logit, y).backward()
        eng, pre, bb = model._engine, "backbone.", "backbone."
        named = dict(model.named_parameters())
        keys = sorted(k for k in named if k.startswith(pre))
    else:
        if net == "s3d":
            from test_infonce_gpu import _build
            if case == "s3d_cfg2":
                model, sd = _build(K=2048, ptr=2048 - B, precision=precision)
                block = torch.randn(B, 2, 3, T, HW, HW, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2024))
                seed = 99
            else:
                model, sd = _build(precision=precision)
                block, seed = MG.make_inputs(B, T).cuda(), 77
        else:
            _build = __import__("test_%s_gpu" % net)._build
            model, sd = _build(precision=precision)
            block, seed = MG.make_inputs_shifted(B, T, HW).cuda(), 77
        torch.manual_seed(seed)
        logits, labels = model(block)
        moco.nce_cross_entropy(logits, labels).backward()
        x = block[:, 0]
        eng, pre, bb = model.encoder_q._engine, "encoder_q.", "encoder_q.0."
        named = dict(model.named_parameters())
        keys = sorted(k for k in named if k.startswith(pre))
        out.update(logits=logits.detach(), queue=model.queue, ptr=int(sd["queue_ptr"]), queue0=sd["queue"].cuda())
    torch.cuda.synchronize()
    plan = eng.plans[(B, T, HW, HW, True, True)]
    out.update(model=model, sd=sd, x=x, eng=eng, plan=plan, pre=pre, bb=bb, named=named, keys=keys)
    return out


def _decisions(st):
    """ReLU masks and max-pool taps as the engine's backward used them, with the cross-checks of the module docstring."""
    eng, plan = st["eng"], st["plan"]
    g, B = eng.graph, st["B"]
    strip = len("0.") if g.head_dim is not None else 0
    masks, taps, members = {}, {}, {}
    worst_dis, n_dis = 0.0, 0
    for t in g.tensors:
        if not t.pending:
            continue
        a = plan.acts[t.index]
        for nm, coff, c in t.bn_members:
            members[nm[strip:]] = (t, coff, c)
            if not t.relu:
                continue
            z = a.data[..., coff:coff + c].double() * a.scale[coff:coff + c].double() + a.shift[coff:coff + c].double()
            if t.residual is not None:       # fp32 fma, then the fp32 add of the residual planes' hi + lo
                r = plan.acts[t.residual.index].pl
                z = z.float() + (r.hi[..., coff:coff + c].float() + r.lo[..., coff:coff + c].float())
            m = z > 0
            dis = m != (_planes(a, coff, c) > 0)
            if bool(dis.any()):
                # gated planes hold gate x relu(z): a value that small may flush to zero once scaled
                res = PLANE_RES / (float(a.gate[:, coff:coff + c].min()) if t.gates else 1.0)
                zd = float(z[dis].abs().max())
                n_dis += int(dis.sum())
                worst_dis = max(worst_dis, zd / res)
            masks[nm[strip:]] = _ncdhw(m)
            del z, m, dis
    st["pool_src"] = {}
    for kind, it in g.items:
        if kind == "pool":
            a = plan.acts[it.dst.index]
            taps[it.name[strip:]] = _ncdhw(a.idx.view(B, *a.dims, it.dst.C))
            st["pool_src"][it.name[strip:]] = plan.acts[it.src.index]
    if g.head_dim is not None:
        z = plan.h1 + eng.store.view("2.bias")
        m = z > 0
        dis = m != (plan.h1_pl.value() > 0)
        if bool(dis.any()):
            n_dis += int(dis.sum())
            worst_dis = max(worst_dis, float(z[dis].abs().max()) / PLANE_RES)
        masks[PO.HEAD_RELU] = _ncdhw(m)
    return masks, taps, members, dict(n_disagree=n_dis, worst_disagree_over_res=worst_dis)


class _Probe(PO.Decisions):
    """Pinned decisions plus the layerwise comparisons: forward values as they are computed, gradients through tensor
    hooks as autograd produces them (nothing float64 is retained past its comparison)."""

    def __init__(self, masks, taps, st, members):
        super().__init__(masks, taps)
        self.st, self.members = st, members
        self.fwd, self.bwd, self.pool_err = {}, {}, {}

    def pool(self, name, x, k, s, p):
        """The tap must be the window maximum of the engine's own input planes exactly, and in float64 within twice the
        forward error of that input (near-ties may order differently in the two forwards)."""
        out = super().pool(name, x, k, s, p)
        with torch.no_grad():
            src = self.st["pool_src"][name]
            e = _ncdhw(_planes(src, 0, src.spec.C)).double()
            exact = torch.equal(PO.pool_at(e, self.taps[name], k, s, p), F.max_pool3d(e, k, s, p))
            gap = float((F.max_pool3d(x, k, s, p) - out).abs().max())
            self.pool_err[name] = (exact, gap, float((e - x).abs().max()))
            del e
        return out

    def _hook(self, t, key, engine_fn):
        def hook(grad):
            self.bwd[key] = _rel_l2(engine_fn(), grad)
        t.register_hook(hook)

    def act(self, kind, name, t):
        plan = self.st["plan"]
        if kind == "feat":
            self.fwd["feat"] = _rel_l2(_ncdhw(plan.feat), t)
            self._hook(t, "dfeat", lambda: _ncdhw(plan.dfeat))
            return
        spec, coff, c = self.members[name]
        a = plan.acts[spec.index]
        if kind == "y":
            self.fwd["y/" + name] = _rel_l2(_ncdhw(a.data[..., coff:coff + c]), t)
            self._hook(t, "dY/" + name, lambda: _ncdhw(_dy(a, coff, c)))
        elif kind == "a":
            if not spec.gates:
                self.fwd["a/" + name] = _rel_l2(_ncdhw(_planes(a, coff, c)), t)
            self._hook(t, "dA/" + name, lambda: _ncdhw(a.grad[..., coff:coff + c]))
        elif kind == "gated":
            self.fwd["a/" + name] = _rel_l2(_ncdhw(_planes(a, coff, c)), t)


def _pinned(st, dtype, dec):
    """The pinned encoder in `dtype` from the step's starting state, seeded with the engine's cotangent; returns
    (output, {parameter key: gradient})."""
    pre, plan = st["pre"], st["plan"]
    sdd = {k: st["sd"][k].detach().to("cuda", dtype).requires_grad_(True) for k in st["keys"]}
    x = st["x"].to(dtype)
    if st["form"] == "finetune":
        out = PO.pooled(sdd, st["bb"], x, dec)
        out.backward(plan.dfeat.to(dtype))
    else:
        out = PO.query(sdd, pre, x, dec)
        out.backward(plan.dq.to(dtype))
    return out.detach(), {k: sdd[k].grad for k in st["keys"]}


def _dq_check(st):
    """plan.dq against d(mean InfoNCE loss)/dq in float64 at the engine's q, k and pre-step queue."""
    plan, B, ptr = st["plan"], st["B"], st["ptr"]
    q = plan.q.double().clone().requires_grad_(True)
    k = st["queue"][:, ptr:ptr + B].t().double()
    lg = torch.cat([(q * k).sum(1, keepdim=True), q @ st["queue0"].double()], 1) / 0.07
    F.cross_entropy(lg, torch.zeros(B, dtype=torch.long, device="cuda")).backward()
    return dict(dq=_rel_l2(plan.dq, q.grad), logits=_rel_l2(st["logits"], lg),
                one_minus_p_pos=float((1 - torch.softmax(lg.detach(), 1)[:, 0]).square().mean().sqrt()))


def _summary(errs):
    v = list(errs.values())
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:5]
    return dict(max=float(np.max(v)), median=float(np.median(v)), n=len(v), worst=worst)


def _run_case(case):
    """Everything one case measures, as plain numbers.  The engine's plan and the float64 graph live in `ctx` only and
    are freed before the next case (at B = 32 they take most of the card)."""
    t0 = time.time()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    flags = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    ctx = {}
    try:
        ctx["st"] = st = _step(case)
        ctx["masks"], ctx["taps"], members, dec_checks = _decisions(st)
        ctx["probe"] = probe = _Probe(ctx["masks"], ctx["taps"], st, members)
        out64, ctx["g64"] = _pinned(st, torch.float64, probe)
        torch.cuda.synchronize()
        fwd = dict(probe.fwd)
        fwd["out"] = _rel_l2(st["plan"].feat if st["form"] == "finetune" else st["plan"].q, out64)
        res = dict(case=case, precision=st["precision"],
                   n_params=len([k for k in st["named"] if k.startswith(st["pre"])]),
                   n_state_params=len(O.param_keys(st["sd"], st["pre"])),
                   unused=sorted((set(ctx["masks"]) | set(ctx["taps"])) - probe.used), fwd=fwd, bwd=dict(probe.bwd),
                   pool_err=dict(probe.pool_err), decisions=dec_checks)
        res["grad"] = {k: _rel_l2(st["named"][k].grad, ctx["g64"][k]) for k in st["keys"]}
        del probe, out64
        ctx.pop("probe")
        gc.collect()
        _, g32 = _pinned(st, torch.float32, PO.Decisions(ctx["masks"], ctx["taps"]))
        res["grad32"] = {k: _rel_l2(g32[k], ctx["g64"][k]) for k in st["keys"]}
        del g32
        if st["form"] == "infonce":
            res.update(_dq_check(st))
        torch.cuda.synchronize()
        res["peak_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
        res["wall_s"] = time.time() - t0
        return res
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags
        st = None
        ctx.clear()
        gc.collect()
        torch.cuda.empty_cache()


@pytest.fixture(scope="module", params=list(CASES))
def case(request, diag):
    res = _run_case(request.param)
    diag["pinned/%s" % request.param] = dict(
        grad=_summary(res["grad"]), grad_fp32=_summary(res["grad32"]), layer=_summary(res["bwd"]),
        fwd=_summary(res["fwd"]), pool=res["pool_err"], decisions=res["decisions"],
        dq=res.get("dq"), logits=res.get("logits"), one_minus_p_pos=res.get("one_minus_p_pos"),
        peak_gb=res["peak_gb"], wall_s=res["wall_s"], per_tensor=res["grad"], per_tensor_fp32=res["grad32"],
        per_layer=res["bwd"])
    return res


def test_every_parameter_gradient(case):
    """Every parameter gradient of the encoder within the flat budget of its precision; only the tensors named in
    GRAD_EXCEPTIONS for this case may instead be off by FP32_FACTOR x float32 torch's error for the same tensor."""
    errs = case["grad"]
    assert len(errs) == case["n_params"] == case["n_state_params"] > 0
    exc = GRAD_EXCEPTIONS.get(case["case"], {})
    assert set(exc) <= set(errs), sorted(set(exc) - set(errs))
    flat = GRAD_BUDGET[case["precision"]]
    bound = {k: max(flat, FP32_FACTOR * case["grad32"][k]) if k in exc else flat for k in errs}
    bad = {k: (e, bound[k], case["grad32"][k]) for k, e in errs.items() if not e < bound[k]}
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1][0])[:8]


def test_layerwise_gradients(case):
    """dA and dY of every BatchNorm member against the float64 gradients at the same points."""
    bwd = case["bwd"]
    n_members = sum(1 for k in bwd if k.startswith("dY/"))
    assert n_members > 0 and sum(1 for k in bwd if k.startswith("dA/")) == n_members
    budget = LAYER_BUDGET[case["precision"]]
    bad = {k: e for k, e in bwd.items() if not e < budget}
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:8]


def test_forward_activations(case):
    """Conv outputs, activation planes and the encoder output against the pinned float64 forward."""
    bad = {k: e for k, e in case["fwd"].items() if not e < FWD_BUDGET}
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:8]


def test_decisions_read_from_the_plan(case):
    """Every decision was used, masks agree with the planes above their resolution, taps pick the window maximum."""
    assert not case["unused"], case["unused"]
    assert case["decisions"]["worst_disagree_over_res"] <= 1.0, case["decisions"]
    bad = {k: v for k, v in case["pool_err"].items() if not (v[0] and v[1] <= 2 * v[2])}
    assert not bad, bad


def test_dq_against_the_loss(case):
    if "dq" not in case:
        pytest.skip("the fine-tune step is seeded with plan.dfeat from the classifier head (test_classifier_gpu.py)")
    # the logits from the same q, k and queue: checks that k and the pre-step queue were read as the step used them
    assert case["logits"] < LOGITS_BUDGET, case["logits"]
    bound = DQ_ULPS * 2.0 ** -24 / case["one_minus_p_pos"]
    assert case["dq"] < bound, (case["dq"], bound, case["one_minus_p_pos"])
