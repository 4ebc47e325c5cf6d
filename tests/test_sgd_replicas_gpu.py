"""SGD and DataParallel replicas on the H100: coclr_sgd_step / SpanSGD bit-identical to torch.optim.SGD, and
LinearClassifier(replicas=R) against the float64 DataParallel oracle (tests/tools/replica_oracle.py), against
single-replica passes of its chunks, and eval/main_classifier.py --gpu 0,1 end to end."""
import io
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "eval"))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _rel_l2(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ---------------------------------------------------------------------------------------------------------------------
# coclr_sgd_step
# ---------------------------------------------------------------------------------------------------------------------
def _foreach_rounding(n=1 << 16):
    """How torch's foreach `a + alpha * b` rounds: mismatches against one fused multiply-add and against a rounded
    product then a rounded add (diagnostic)."""
    g = torch.Generator(device="cuda").manual_seed(3)
    a, b = torch.randn(n, device="cuda", generator=g), torch.randn(n, device="cuda", generator=g)
    alpha = 1e-3
    got = torch._foreach_add([a], [b], alpha=alpha)[0]
    al = torch.tensor(alpha, dtype=torch.float32).double().item()
    fma = (a.double() + al * b.double()).float()
    two = a + (b * torch.tensor(alpha, dtype=torch.float32, device="cuda"))
    return int((got != fma).sum()), int((got != two).sum())


@pytest.mark.parametrize("n", [1, 3, 1001, 4099, (1 << 20) + 7])
@pytest.mark.parametrize("wd", [0.0, 1e-3])
def test_sgd_step_bit_identical_to_torch(n, wd, diag):
    from coclr_b200 import moco
    g = torch.Generator(device="cuda").manual_seed(n + int(wd * 1e6))
    p0 = torch.randn(n, device="cuda", generator=g)
    mine, grad = p0.clone(), torch.zeros(n, device="cuda")
    opt = moco.SpanSGD([dict(name="all", params=mine, grad=grad, lr=0.1)], momentum=0.9, weight_decay=wd)
    ref = p0.clone().requires_grad_(True)
    ref_opt = torch.optim.SGD([ref], lr=0.1, momentum=0.9, weight_decay=wd)
    loop = p0.clone().requires_grad_(True)
    loop_opt = torch.optim.SGD([loop], lr=0.1, momentum=0.9, weight_decay=wd, foreach=False)
    loop_same = True
    for step in range(5):
        if step == 3:                                         # lr drop, as adjust_learning_rate does
            for o in (opt, ref_opt, loop_opt):
                for grp in o.param_groups:
                    grp["lr"] *= 0.1
        gr = torch.randn(n, device="cuda", generator=g) * (10.0 if step == 0 else 1.0)
        grad.copy_(gr)
        ref.grad, loop.grad = gr.clone(), gr.clone()
        opt.step()
        ref_opt.step()
        loop_opt.step()
        torch.cuda.synchronize()
        buf = ref_opt.state[ref]["momentum_buffer"]
        assert torch.equal(mine, ref.detach()), (step, int((mine != ref.detach()).sum()))
        assert torch.equal(opt.momentum_buffer[0], buf), step
        loop_same = loop_same and torch.equal(loop.detach(), ref.detach())
    diag["sgd/foreach_false_same_bits/n%d_wd%g" % (n, wd)] = loop_same
    if n == 1001 and wd:
        diag["sgd/foreach_add_alpha_mismatch_fma_vs_mul_add"] = list(_foreach_rounding())


def _ft_model(ncls=51, seed=0, replicas=1, net="s3d", train_what="ft"):
    from model.classifier import LinearClassifier
    import classifier_oracle as O
    last = train_what == "last"
    m = LinearClassifier(num_class=ncls, network=net, dropout=0.9, use_dropout=not last, use_l2_norm=last,
                         use_final_bn=last, replicas=replicas)
    sd = O.classifier_state(net, ncls, not last, last, seed=seed)
    res = m.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(".block" in k for k in res.missing_keys)
    if last:
        for p in m.backbone.parameters():
            p.requires_grad = False
    return m.cuda(), sd


def test_sgd_two_groups_match_per_tensor_groups():
    """The ft layout: backbone span at lr / 10 and head span at lr, against torch.optim.SGD over the reference's
    per-tensor param groups (eval/main_classifier.py:134-161)."""
    import main_classifier as MC
    model, _ = _ft_model()
    args = types.SimpleNamespace(train_what="ft", lr=0.1, wd=1e-3, optim="sgd")
    opt = MC.build_optimizer(model, args)
    named = {k: p for k, p in model.named_parameters()}
    ref = {k: p.detach().clone().requires_grad_(True) for k, p in named.items()}
    groups = [{"params": [ref[k] for k in ref if k.startswith("backbone.")], "lr": 0.01},
              {"params": [ref[k] for k in ref if not k.startswith("backbone.")], "lr": 0.1}]
    ref_opt = torch.optim.SGD(groups, lr=0.1, momentum=0.9, weight_decay=1e-3)
    spans = model.flat_spans()
    g = torch.Generator(device="cuda").manual_seed(11)
    for step in range(3):
        opt.zero_grad()
        model._prepare_grads(True)
        for k, p in named.items():
            p.grad.copy_(torch.randn(p.shape, device="cuda", generator=g) * 1e-2)
            ref[k].grad = p.grad.detach().clone()
        opt.step()
        ref_opt.step()
    torch.cuda.synchronize()
    assert spans["backbone"][0].data_ptr() == model._engine.store.flat.data_ptr()
    for k, p in named.items():
        assert torch.equal(p.detach(), ref[k].detach()), k


def test_sgd_state_dict_round_trip():
    from coclr_b200 import moco
    g = torch.Generator(device="cuda").manual_seed(5)
    n1, n2 = 5003, 130
    pa, pb = [torch.randn(n, device="cuda", generator=g) for n in (n1, n2)]
    ga, gb = torch.zeros(n1, device="cuda"), torch.zeros(n2, device="cuda")
    mk = lambda a, b: moco.SpanSGD([dict(name="backbone", params=a, grad=ga, lr=0.01),  # noqa: E731
                                    dict(name="head", params=b, grad=gb, lr=0.1)], weight_decay=1e-3)
    grads = [(torch.randn(n1, device="cuda", generator=g), torch.randn(n2, device="cuda", generator=g))
             for _ in range(4)]
    opt = mk(pa, pb)
    for s in range(2):
        ga.copy_(grads[s][0]), gb.copy_(grads[s][1])
        opt.step()
    opt.param_groups[0]["lr"] *= 0.1
    f = io.BytesIO()
    torch.save(opt.state_dict(), f)
    qa, qb = pa.clone(), pb.clone()
    opt2 = mk(qa, qb)
    f.seek(0)
    opt2.load_state_dict(torch.load(f, map_location="cpu"))
    assert opt2.param_groups[0]["lr"] == opt.param_groups[0]["lr"]
    for s in range(2, 4):
        ga.copy_(grads[s][0]), gb.copy_(grads[s][1])
        opt.step()
        opt2.step()
    torch.cuda.synchronize()
    assert torch.equal(pa, qa) and torch.equal(pb, qb)
    assert all(torch.equal(a, b) for a, b in zip(opt.momentum_buffer, opt2.momentum_buffer))
    adam = moco.SpanAdam([dict(name="backbone", params=pa, grad=ga, lr=0.01),
                          dict(name="head", params=pb, grad=gb, lr=0.1)])
    with pytest.raises(ValueError):
        opt2.load_state_dict(adam.state_dict())


# ---------------------------------------------------------------------------------------------------------------------
# LinearClassifier(replicas=R)
# ---------------------------------------------------------------------------------------------------------------------
def _clips(B, T, HW, ncls, seed=99):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 3, T, HW, HW, generator=g) + 1.5 * torch.randn(B, 3, 1, 1, 1, generator=g)
    ramp = torch.linspace(-1, 1, HW).view(1, 1, 1, 1, HW)
    x = x + torch.randn(B, 3, 1, 1, 1, generator=g) * ramp
    return x.cuda(), torch.randint(0, ncls, (B,), generator=g).cuda()


def _set_modes(m, train_what):
    if train_what == "last":
        m.eval()
        m.final_bn.train()
    else:
        m.train()


def _running(m):
    st = m._engine.store
    out = [st.running_mean.clone(), st.running_var.clone(), st.nbt.clone()]
    if m.use_final_bn:
        out += [m.final_bn.running_mean.clone(), m.final_bn.running_var.clone(), m.final_bn.num_batches_tracked.clone()]
    return out


def _oracle(sd, x, y, R, train_what, dtype, mask):
    import replica_oracle as RO
    last = train_what == "last"
    sdd = {k: (v.cuda().to(dtype) if v.is_floating_point() else v.cuda().clone()) for k, v in sd.items()}
    for k in sdd:
        if (k.endswith(".weight") or k.endswith(".bias")) and (not last or not k.startswith("backbone.")):
            sdd[k].requires_grad_(True)
    logit, _ = RO.dataparallel_forward(sdd, x.to(dtype), R, not last, last, last, mask, 0.9)
    loss = F.cross_entropy(logit, y)
    loss.backward()
    return sdd, logit, loss


BUDGET = {"s3d": 1.5, "s3dg": 4}   # gradient median error against the fp32 oracle's, as test_classifier_gpu.py allows


CASES = [("s3d", "ft", 2, 4), ("s3d", "ft", 3, 5), ("s3d", "all", 2, 4), ("s3d", "last", 2, 5), ("s3d", "last", 3, 8),
         ("s3dg", "ft", 2, 4)]


@pytest.mark.parametrize("net,train_what,R,B", CASES)
def test_replicas_against_dataparallel_oracle(net, train_what, R, B, diag):
    import main_classifier as MC
    from model.classifier import replica_chunks
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    T, HW, ncls = 8, 64, 51
    tag = "replicas/%s_%s_R%d_B%d/" % (net, train_what, R, B)
    model, sd = _ft_model(ncls, replicas=R, net=net, train_what=train_what)
    _set_modes(model, train_what)
    x, y = _clips(B, T, HW, ncls)
    torch.manual_seed(5)
    logit, _ = model(x)
    mask = None if model.dropout_mask is None else model.dropout_mask.clone()
    loss = F.cross_entropy(logit, y)
    model.zero_grad(set_to_none=True)
    loss.backward()
    torch.cuda.synchronize()
    named = dict(model.named_parameters())
    grads = {k: p.grad.detach().clone() for k, p in named.items() if p.grad is not None}
    msd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    after = _running(model)

    # float64 DataParallel oracle, fed the dropout mask
    sd64, lg64, loss64 = _oracle(sd, x, y, R, train_what, torch.float64, mask)
    sd32, _, _ = _oracle(sd, x, y, R, train_what, torch.float32, mask)
    e = _rel(logit, lg64)
    diag[tag + "logits_vs_fp64"] = e
    assert e < 1e-3
    assert abs(float(loss.detach()) - float(loss64.detach())) < 1e-3 * max(1.0, abs(float(loss64.detach())))
    bb = {k: [_rel_l2(g, sd64[k].grad), _rel_l2(sd32[k].grad, sd64[k].grad)] for k, g in grads.items()
          if k.startswith("backbone.")}
    trained = [k for k in sd64 if sd64[k].requires_grad]
    assert sorted(grads) == sorted(trained)
    if bb:
        med_new = float(np.median([v[0] for v in bb.values()]))
        med_ref = float(np.median([v[1] for v in bb.values()]))
        diag[tag + "grad_median_new_ref"] = [med_new, med_ref]
        assert med_new < BUDGET[net] * med_ref + 1e-3, (med_new, med_ref)
        # the S3D-G gating fc gradients, summed over the replicas like every other gradient
        for k, (e_new, e_ref) in bb.items():
            if ".fc." in k:
                assert e_new < BUDGET[net] * e_ref + 5e-2, (k, e_new, e_ref)
    for k in grads:
        if not k.startswith("backbone."):
            e = _rel(grads[k], sd64[k].grad)
            diag[tag + "grad/" + k] = e
            assert e < 1e-3, (k, e)
    stat_keys = (["final_bn.running_mean", "final_bn.running_var"] if train_what == "last" else
                 ["backbone.Conv_1a.bn1.running_mean", "backbone.Mixed_4d.branch1.1.bn2.running_var",
                  "backbone.Mixed_5c.branch0.0.bn.running_mean"])
    for k in stat_keys:
        e = _rel(msd[k], sd64[k])
        diag[tag + k] = e
        assert e < (1e-4 if k.startswith("final_bn") else 1e-3), (k, e)
    for k in sd64:
        if k.endswith("num_batches_tracked"):
            assert int(msd[k]) == int(sd64[k]), k

    # each chunk's logits and the running statistics against single-replica passes from the same state
    single, _ = _ft_model(ncls, replicas=1, net=net, train_what=train_what)
    _set_modes(single, train_what)
    torch.manual_seed(5)
    for r, (r0, r1) in enumerate(replica_chunks(B, R)):
        lg_r, _ = single(x[r0:r1])
        if r == 0:
            chunk0 = _running(single)
        assert torch.equal(lg_r, logit[r0:r1]), (r, _rel(lg_r, logit[r0:r1]))
    for a, b in zip(after, chunk0):
        assert torch.equal(a, b)

    # one SGD step and one Adam step from these gradients against float64 steps on the oracle's
    flat = {k: pg[0].clone() for k, pg in model.flat_spans().items()}
    lr = {k: (0.01 if train_what == "ft" else 0.1) if k.startswith("backbone.") else 0.1 for k in grads}
    for optim in ("sgd", "adam"):
        for k, (p, _) in model.flat_spans().items():
            p.copy_(flat[k])
        args = types.SimpleNamespace(train_what=train_what, lr=0.1, wd=1e-3, optim=optim)
        opt = MC.build_optimizer(model, args)
        opt.step()
        torch.cuda.synchronize()
        now = dict(model.named_parameters())
        for k in grads:
            p0 = sd[k].double().cuda()
            g64 = sd64[k].grad.double() + 1e-3 * p0
            if optim == "sgd":
                ref = p0 - lr[k] * g64
            else:
                ref = p0 - lr[k] * g64 / (g64.abs() + 1e-8)    # Adam's first step: lr * sign(g) (up to eps)
            moved = (ref - p0).abs().max()
            off = int(((now[k].detach().double() - ref).abs() > 0.1 * moved).sum())
            diag[tag + optim + "/" + k] = off / ref.numel()
            # Adam's first step moves every element by about lr whatever the gradient's size, so a gradient element
            # near zero may flip its sign: a few such elements are allowed (with 2-clip chunks the BatchNorm bias
            # gradients of the early layers have many)
            assert off <= max(2, 0.05 * ref.numel()), (optim, k, off, ref.numel())


def test_replicas_one_is_bit_identical():
    x, y = _clips(4, 8, 64, 51)
    out = []
    for kw in ({}, {"replicas": 1}):
        from model.classifier import LinearClassifier
        import classifier_oracle as O
        m = LinearClassifier(num_class=51, network="s3d", dropout=0.9, **kw)
        m.load_state_dict(O.classifier_state("s3d", 51, True, False, seed=0), strict=False)
        m = m.cuda().train()
        torch.manual_seed(5)
        logit, feat = m(x)
        F.cross_entropy(logit, y).backward()
        torch.cuda.synchronize()
        out.append([logit, feat, m.dropout_mask] + [p.grad.clone() for p in m.parameters()] + _running(m))
    assert all(torch.equal(a, b) for a, b in zip(*out))


def test_last_with_one_row_chunk_raises_before_any_launch():
    model, _ = _ft_model(replicas=2, train_what="last")
    _set_modes(model, "last")
    model._engine_for(torch.device("cuda"))
    before = _running(model)
    with pytest.raises(ValueError):
        model(torch.randn(3, 3, 8, 64, 64, device="cuda"))        # chunks of 2 and 1
    assert not model._engine.plans
    assert all(torch.equal(a, b) for a, b in zip(before, _running(model)))


@pytest.mark.parametrize("train_what", ["ft", "last"])
def test_validate_under_replicas_is_one_pass(train_what):
    x, _ = _clips(5, 8, 64, 51)
    out = []
    for R in (1, 3):
        model, _ = _ft_model(replicas=R, train_what=train_what)
        model.eval()
        with torch.no_grad():
            out.append(model(x))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


def test_readme_shape_ft_two_replicas(diag):
    """ft at the README's shape: 2 x 32 clips of 32 x 128^2 on one card, against the float64 oracle (chunk by chunk:
    with the loss a mean over all 64 clips, the per-chunk backward of loss_r = CE_sum(chunk r) / 64 sums to the same
    gradients)."""
    from classifier_oracle import classifier_forward
    from oracle.coclr_oracle import _bn_scratch
    torch.backends.cudnn.allow_tf32 = False
    R, B, T, HW, ncls = 2, 64, 32, 128, 101
    model, sd = _ft_model(ncls, replicas=R)
    model.train()
    x, y = _clips(B, T, HW, ncls)
    torch.manual_seed(5)
    torch.cuda.reset_peak_memory_stats()
    logit, _ = model(x)
    mask = model.dropout_mask.clone()
    loss = F.cross_entropy(logit, y)
    model.zero_grad(set_to_none=True)
    loss.backward()
    torch.cuda.synchronize()
    diag["replicas/readme_ft_R2x32/peak_GiB"] = torch.cuda.max_memory_allocated() / 2 ** 30
    keys = ["backbone.Conv_1a.conv1.weight", "backbone.Mixed_4c.branch2.1.conv2.weight",
            "backbone.Mixed_5c.branch3.1.bn.weight", "final_fc.1.weight", "final_fc.1.bias"]
    named = dict(model.named_parameters())
    grads = {k: named[k].grad.detach().clone() for k in keys}
    lg_new = logit.detach().clone()
    del logit, loss
    model._engine.plans.clear()
    torch.cuda.empty_cache()
    sdd = {k: (v.cuda().double() if v.is_floating_point() else v.cuda().clone()) for k, v in sd.items()}
    for k in keys:
        sdd[k].requires_grad_(True)
    lgs = []
    for r, (xr, yr, mr) in enumerate(zip(torch.chunk(x, R), torch.chunk(y, R), torch.chunk(mask, R))):
        s = sdd if r == 0 else _bn_scratch(sdd, "")
        lg, _ = classifier_forward(s, xr.double(), True, dropout_mask=mr, p=0.9)
        (F.cross_entropy(lg, yr, reduction="sum") / B).backward()
        lgs.append(lg.detach())
        del lg
    e = _rel(lg_new, torch.cat(lgs))
    diag["replicas/readme_ft_R2x32/logits_vs_fp64"] = e
    assert e < 1e-3
    for k in keys:
        e = _rel_l2(grads[k], sdd[k].grad)
        diag["replicas/readme_ft_R2x32/grad/" + k] = e
        # backbone: fp32 arithmetic through train-mode BatchNorm; the fp32 cuDNN oracle itself is a few 1e-2 off the
        # float64 gradients at the small shapes above
        assert e < (5e-2 if k.startswith("backbone.") else 1e-3), (k, e)


# ---------------------------------------------------------------------------------------------------------------------
# CLI
# ---------------------------------------------------------------------------------------------------------------------
def _cli(tmp, *extra):
    cmd = [sys.executable, os.path.join(ROOT, "eval", "main_classifier.py"), "--synthetic", "--net", "s3d",
           "--dataset", "hmdb51", "--batch_size", "4", "--seq_len", "8", "--img_dim", "64", "--steps-per-epoch", "3",
           "--print_freq", "1", "--gpu", "0,1"] + list(extra)
    r = subprocess.run(cmd, cwd=tmp, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:]
    return r.stdout


@pytest.mark.parametrize("train_what,optim", [("last", "sgd"), ("ft", "adam")])
def test_cli_two_replicas_train_resume(train_what, optim, tmp_path):
    flags = ["--train_what", train_what, "--optim", optim]
    out = _cli(tmp_path, *flags, "--epochs", "2")
    assert "=> Effective BatchSize = 8" in out and "Acc@1" in out
    paths = [os.path.join(d, f) for d, _, fs in os.walk(tmp_path) for f in fs if f == "epoch1.pth.tar"]
    assert len(paths) == 1
    assert ("_SGD_bs8_" if optim == "sgd" else "_Adam_bs8_") in paths[0]
    ck = torch.load(paths[0], map_location="cpu", weights_only=False)
    assert ck["epoch"] == 1
    assert ("momentum_buffer" in ck["optimizer"]) == (optim == "sgd")
    assert ("exp_avg" in ck["optimizer"]) == (optim == "adam")
    out = _cli(tmp_path, *flags, "--epochs", "3", "--resume", paths[0])
    assert "Training from ep 2 to ep 3 finished" in out
    assert os.path.exists(paths[0].replace("epoch1", "epoch2"))
