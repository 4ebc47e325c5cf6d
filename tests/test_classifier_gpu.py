"""LinearClassifier on the H100: the classifier-head kernels (csrc/classifier.cu) against float64 torch over a grid of
shapes and options, and whole fine-tune / linear-probe / eval steps of the module against the float64 oracle
(tests/tools/classifier_oracle.py), plus eval/main_classifier.py --synthetic end to end."""
import ctypes as C
import itertools
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
# head kernels
# ---------------------------------------------------------------------------------------------------------------------
def _head_run(feat, W, bias, gamma, beta, rm, rv, dl, l2, bn, bn_train, p, seed):
    """One forward + backward of the head kernels; returns every output as a dict of fresh tensors."""
    from coclr_b200 import lib as L
    B, fs = feat.shape
    ncls = W.shape[0]
    dev = feat.device
    z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)  # noqa: E731
    o = dict(xn=z(B, fs), inv=z(B), xb=z(B, fs), mean=z(fs), rstd=z(fs), mask=torch.zeros(B, fs, dtype=torch.uint8, device=dev),
             xd=z(B, fs), logits=z(B, ncls), dW=z(ncls, fs), db=z(ncls), dg=z(fs), dbeta=z(fs), dx=z(B, fs),
             dfeat=z(B, fs), rm=rm.clone(), rv=rv.clone())
    h = L.ClsHead(B=B, fs=fs, ncls=ncls, l2norm=int(l2), bn=int(bn), bn_training=int(bn_train), dropout=int(p > 0), p=p,
                  momentum=0.1, eps=1e-5, seed=seed, offset=0)
    for f, t in (("feat", feat), ("xn", o["xn"]), ("inv_norm", o["inv"]), ("xb", o["xb"]), ("mean", o["mean"]),
                 ("rstd", o["rstd"]), ("gamma", gamma), ("beta", beta), ("running_mean", o["rm"]),
                 ("running_var", o["rv"]), ("mask", o["mask"]), ("xd", o["xd"]), ("W", W), ("bias", bias),
                 ("logits", o["logits"]), ("dlogits", dl), ("dW", o["dW"]), ("dbias", o["db"]), ("dgamma", o["dg"]),
                 ("dbeta", o["dbeta"]), ("dx", o["dx"]), ("dfeat", o["dfeat"])):
        setattr(h, f, L.dptr(t))
    lib = L.load()
    L.check(lib.coclr_cls_head_fwd(C.byref(h), L.stream_ptr()), "coclr_cls_head_fwd")
    L.check(lib.coclr_cls_head_bwd(C.byref(h), L.stream_ptr()), "coclr_cls_head_bwd")
    o["dW1"] = o["dW"].clone()
    L.check(lib.coclr_cls_head_bwd(C.byref(h), L.stream_ptr()), "coclr_cls_head_bwd")   # accumulates
    torch.cuda.synchronize()
    return o


@pytest.mark.parametrize("B,fs,ncls", list(itertools.product([2, 4, 32, 33], [1024, 2048], [51, 101, 400])))
def test_head_kernels_against_float64(B, fs, ncls, diag):
    g = torch.Generator(device="cuda").manual_seed(B * 7919 + fs + ncls)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)  # noqa: E731
    feat = (rn(B, fs) + 0.5 * rn(1, fs)).abs() * 0.3      # non-negative like an average-pooled ReLU output
    W, bias = rn(ncls, fs) / fs ** 0.5, rn(ncls) * 0.05
    gamma, beta = torch.rand(fs, device="cuda", generator=g) + 0.5, rn(fs) * 0.1
    rm, rv = rn(fs) * 0.01, torch.rand(fs, device="cuda", generator=g) * 0.01 + 0.005
    dl = rn(B, ncls)
    worst = {}
    for l2, bn, p in itertools.product([0, 1], [0, 1], [0.0, 0.5, 0.9]):
        for bn_train in ([0, 1] if bn else [0]):
            o = _head_run(feat, W, bias, gamma, beta, rm, rv, dl, l2, bn, bn_train, p, seed=1234)
            o2 = _head_run(feat, W, bias, gamma, beta, rm, rv, dl, l2, bn, bn_train, p, seed=1234)
            for k in ("logits", "dW", "db", "dg", "dbeta", "dfeat", "rm", "rv", "mask"):
                assert torch.equal(o[k], o2[k]), ("not reproducible", k)
            assert torch.equal(o["dW"], 2 * o["dW1"])
            # float64 truth, fed the kernels' dropout mask
            d = lambda t: t.double().clone().requires_grad_(True)  # noqa: E731
            f64, W64, b64, g64, be64 = d(feat), d(W), d(bias), d(gamma), d(beta)
            rm64, rv64 = rm.double().clone(), rv.double().clone()
            x = F.normalize(f64, p=2, dim=1) if l2 else f64
            if bn:
                x = F.batch_norm(x, rm64, rv64, g64, be64, bool(bn_train), 0.1, 1e-5)
            if p > 0:
                m = o["mask"].double()
                x = x * m / (1 - p)
                n, keep = m.numel(), float(m.sum())
                sd = (n * p * (1 - p)) ** 0.5
                assert abs(keep - n * (1 - p)) < 6 * sd, (keep, n, p)
            lg = F.linear(x, W64, b64)
            (lg * dl.double()).sum().backward()
            errs = {"logits": _rel(o["logits"], lg), "dW": _rel(o["dW1"], W64.grad), "db": _rel(o["db"] / 2, b64.grad)}
            if bn:
                errs.update(dgamma=_rel(o["dg"] / 2, g64.grad), dbeta=_rel(o["dbeta"] / 2, be64.grad),
                            rm=_rel(o["rm"], rm64), rv=_rel(o["rv"], rv64))
            # dfeat against the magnitude of the terms it is made of: with B = 2 a train-mode BatchNorm makes the true
            # gradient vanish (its output no longer depends on the input), leaving only rounding
            scale = (dl.double().abs() @ W.double().abs()).max()
            if bn:
                scale = scale * float((gamma.double() * torch.as_tensor(o["rstd"]).double()).abs().max())
            if l2:
                scale = scale * float(o["inv"].double().max())
            errs["dfeat"] = float((o["dfeat"].double() - f64.grad).abs().max() / max(float(f64.grad.abs().max()),
                                                                                     1e-3 * float(scale)))
            key = "l2=%d bn=%d/%d p=%.1f" % (l2, bn, bn_train, p)
            worst[key] = max(errs.values())
            assert max(errs.values()) < 1e-5, (key, errs)
    diag["cls_head/B%d_fs%d_n%d" % (B, fs, ncls)] = max(worst.values())


def test_head_rejects_train_mode_batchnorm_with_one_clip():
    from model.classifier import LinearClassifier
    m = LinearClassifier(num_class=11, network="s3d", use_dropout=False, use_final_bn=True).cuda().eval()
    m.final_bn.train()
    with torch.no_grad(), pytest.raises(ValueError):
        m(torch.randn(1, 3, 8, 64, 64, device="cuda"))


# ---------------------------------------------------------------------------------------------------------------------
# module steps against the float64 oracle
# ---------------------------------------------------------------------------------------------------------------------
def _clips(B, T, HW, ncls, seed=99):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 3, T, HW, HW, generator=g) + 1.5 * torch.randn(B, 3, 1, 1, 1, generator=g)
    ramp = torch.linspace(-1, 1, HW).view(1, 1, 1, 1, HW)
    x = x + torch.randn(B, 3, 1, 1, 1, generator=g) * ramp
    return x.cuda(), torch.randint(0, ncls, (B,), generator=g).cuda()


def _model(net, ncls, train_what, seed=0):
    from model.classifier import LinearClassifier
    import classifier_oracle as O
    last = train_what == "last"
    m = LinearClassifier(num_class=ncls, network=net, dropout=0.9, use_dropout=not last, use_l2_norm=last,
                         use_final_bn=last)
    sd = O.classifier_state(net, ncls, not last, last, seed=seed)
    res = m.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(".block" in k for k in res.missing_keys)
    if last:
        for p in m.backbone.parameters():
            p.requires_grad = False
    return m.cuda(), sd


def _oracle(sd, x, y, dtype, backbone_training, bn_training, l2, mask=None, p=0.9, train_params=None):
    import classifier_oracle as O
    sdd = {k: (v.cuda().to(dtype) if v.is_floating_point() else v.cuda().clone()) for k, v in sd.items()}
    for k in sdd:
        if (k.endswith(".weight") or k.endswith(".bias")) and (train_params is None or train_params(k)):
            sdd[k].requires_grad_(True)
    logit, feat = O.classifier_forward(sdd, x.to(dtype), backbone_training, bn_training, l2, mask, p)
    loss = F.cross_entropy(logit, y)
    loss.backward()
    return sdd, logit, loss


def _adam_ref(sdd, sd, keys, lr, wd):
    """One torch.optim.Adam step (coupled L2) from zero moments on float64 copies of the parameters."""
    out = {}
    for k in keys:
        p = sd[k].double().cuda().clone().requires_grad_(True)
        p.grad = sdd[k].grad.double().clone()
        opt = torch.optim.Adam([p], lr=lr[k], weight_decay=wd)
        opt.step()
        out[k] = p.detach()
    return out


def _finetune_step(net, B, T, HW, ncls):
    import main_classifier as MC
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model, sd = _model(net, ncls, "ft")
    model.train()
    args = types.SimpleNamespace(train_what="ft", lr=1e-3, wd=1e-3)
    opt = MC.build_optimizer(model, args)
    x, y = _clips(B, T, HW, ncls)
    torch.manual_seed(5)
    logit, feat = model(x)
    mask = model.dropout_mask.clone()
    loss = F.cross_entropy(logit, y)
    opt.zero_grad()
    loss.backward()
    named = dict(model.named_parameters())
    grads = {k: p.grad.detach().clone() for k, p in named.items() if p.grad is not None}
    opt.step()
    torch.cuda.synchronize()
    msd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    t64 = _oracle(sd, x, y, torch.float64, True, True, False, mask)
    r32 = _oracle(sd, x, y, torch.float32, True, True, False, mask)
    return dict(model=model, sd=sd, logit=logit, grads=grads, msd=msd, t64=t64, r32=r32, named=named)


BUDGET = {"s3d": 1.5, "s3dg": 4, "r50": 3}     # gradient median error against the fp32 oracle's, as in the pre-training suites


@pytest.fixture(scope="module")
def ft_s3d():
    return _finetune_step("s3d", 4, 8, 128, 101)


def _check_grads(step, net, diag):
    sd64, sd32 = step["t64"][0], step["r32"][0]
    out = {}
    for k, g in step["grads"].items():
        if k.startswith("backbone."):
            out[k] = [_rel_l2(g, sd64[k].grad), _rel_l2(sd32[k].grad, sd64[k].grad)]
    med_new = float(np.median([v[0] for v in out.values()]))
    med_ref = float(np.median([v[1] for v in out.values()]))
    diag["cls_ft/%s/grad_median_new_ref" % net] = [med_new, med_ref]
    assert len(out) == len([k for k in sd64 if k.startswith("backbone.") and sd64[k].requires_grad])
    assert med_new < BUDGET[net] * med_ref + 1e-3, (med_new, med_ref)
    for k in ("final_fc.1.weight", "final_fc.1.bias"):
        e = _rel(step["grads"][k], sd64[k].grad)
        diag["cls_ft/%s/grad/%s" % (net, k)] = e
        assert e < 1e-3, (k, e)


def test_finetune_step_s3d(ft_s3d, diag):
    st = ft_s3d
    e = _rel(st["logit"], st["t64"][1])
    diag["cls_ft/s3d/logits_vs_fp64"] = e
    assert e < 1e-3
    _check_grads(st, "s3d", diag)
    sd64, msd = st["t64"][0], st["msd"]
    for k in ("backbone.Conv_1a.bn1.running_mean", "backbone.Mixed_4d.branch1.1.bn2.running_var",
              "backbone.Mixed_5c.branch0.0.bn.running_mean"):
        e = _rel(msd[k], sd64[k])
        diag["cls_ft/s3d/" + k] = e
        assert e < 1e-3, (k, e)
    assert int(msd["backbone.Conv_2b.bn.num_batches_tracked"]) == 4
    # parameters after the two-lr Adam step: backbone at lr / 10, head at lr
    keys = ["backbone.Conv_1a.conv1.weight", "backbone.Mixed_4c.branch2.1.conv2.weight", "backbone.Mixed_5c.branch3.1.bn.weight",
            "final_fc.1.weight", "final_fc.1.bias"]
    lr = {k: (1e-4 if k.startswith("backbone.") else 1e-3) for k in keys}
    ref = _adam_ref(sd64, st["sd"], keys, lr, 1e-3)
    for k in keys:
        moved = (ref[k] - st["sd"][k].double().cuda()).abs().max()
        e = float((msd[k].double() - ref[k]).abs().max() / moved)
        diag["cls_ft/s3d/adam/" + k] = e
        # Adam's first step moves every element by about lr; a gradient element near zero may flip its sign, so the
        # check is against the size of the step and allows a few such elements
        frac = float(((msd[k].double() - ref[k]).abs() > 0.1 * moved).double().mean())
        assert frac < 0.02, (k, e, frac)


@pytest.mark.parametrize("net,ncls", [("s3dg", 51), ("r50", 400)])
def test_finetune_forward_and_gradients(net, ncls, diag):
    st = _finetune_step(net, 2, 8, 64, ncls)
    e = _rel(st["logit"], st["t64"][1])
    diag["cls_ft/%s/logits_vs_fp64" % net] = e
    assert e < 1e-3
    _check_grads(st, net, diag)


def test_linear_probe_step(diag):
    import main_classifier as MC
    model, sd = _model("s3d", 101, "last")
    model.eval()
    model.final_bn.train()
    args = types.SimpleNamespace(train_what="last", lr=1e-3, wd=1e-3)
    opt = MC.build_optimizer(model, args)
    bb_before = {k: v.detach().clone() for k, v in model.backbone.state_dict().items()}
    x, y = _clips(4, 8, 128, 101)
    logit, feat = model(x)
    loss = F.cross_entropy(logit, y)
    opt.zero_grad()
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    eng = model._engine
    assert all(not k[5] for k in eng.plans), "the frozen backbone must not get a backward plan"
    for k, v in model.backbone.state_dict().items():
        assert torch.equal(v, bb_before[k]), k
    sd64, lg64, _ = _oracle(sd, x, y, torch.float64, False, True, True, train_params=lambda k: not k.startswith("backbone."))
    e = _rel(logit, lg64)
    diag["cls_probe/logits_vs_fp64"] = e
    assert e < 1e-3
    msd = model.state_dict()
    for k in ("final_bn.running_mean", "final_bn.running_var"):
        e = _rel(msd[k], sd64[k])
        diag["cls_probe/" + k] = e
        assert e < 1e-4, (k, e)
    assert int(msd["final_bn.num_batches_tracked"]) == 4
    keys = ["final_fc.0.weight", "final_fc.0.bias", "final_bn.weight", "final_bn.bias"]
    for k in keys:
        e = _rel(model.final_fc[0].weight.grad if k == "final_fc.0.weight" else dict(model.named_parameters())[k].grad,
                 sd64[k].grad)
        diag["cls_probe/grad/" + k] = e
        assert e < 1e-3, (k, e)
    ref = _adam_ref(sd64, sd, keys, {k: 1e-3 for k in keys}, 1e-3)
    for k in keys:
        moved = (ref[k] - sd[k].double().cuda()).abs().max()
        frac = float(((msd[k].double() - ref[k]).abs() > 0.1 * moved).double().mean())
        assert frac < 0.02, (k, frac)


def test_eval_forward(diag):
    model, sd = _model("s3d", 101, "ft")
    model.eval()
    x, _ = _clips(4, 8, 128, 101)
    with torch.no_grad():
        logit, feat = model(x)
    sdd = {k: (v.cuda().double() if v.is_floating_point() else v.cuda()) for k, v in sd.items()}
    import classifier_oracle as O
    lg64, f64 = O.classifier_forward(sdd, x.double(), False)
    e = _rel(logit, lg64)
    diag["cls_eval/logits_vs_fp64"] = e
    assert e < 1e-3 and _rel(feat, f64) < 1e-3
    assert model.dropout_mask is None


# ---------------------------------------------------------------------------------------------------------------------
# CLI
# ---------------------------------------------------------------------------------------------------------------------
def _cli(tmp, *extra):
    cmd = [sys.executable, os.path.join(ROOT, "eval", "main_classifier.py"), "--synthetic", "--net", "s3d",
           "--dataset", "hmdb51", "--batch_size", "4", "--seq_len", "8", "--img_dim", "64", "--steps-per-epoch", "3",
           "--print_freq", "1"] + list(extra)
    r = subprocess.run(cmd, cwd=tmp, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:]
    return r.stdout


@pytest.mark.parametrize("train_what", ["last", "ft"])
def test_cli_train_validate_resume(train_what, tmp_path):
    out = _cli(tmp_path, "--train_what", train_what, "--epochs", "1")
    assert "Acc@1" in out
    paths = [os.path.join(d, f) for d, _, fs in os.walk(tmp_path) for f in fs if f == "epoch0.pth.tar"]
    assert len(paths) == 1
    ck = torch.load(paths[0], map_location="cpu", weights_only=False)
    assert set(ck) == {"epoch", "state_dict", "best_acc", "optimizer", "iteration"}
    assert ck["epoch"] == 0 and ck["iteration"] == 4
    assert ("final_fc.0.weight" if train_what == "last" else "final_fc.1.weight") in ck["state_dict"]
    out = _cli(tmp_path, "--train_what", train_what, "--epochs", "2", "--resume", paths[0])
    assert "Training from ep 1 to ep 2 finished" in out
    assert os.path.exists(paths[0].replace("epoch0", "epoch1"))


def test_cli_pretrain_loads_backbone(tmp_path):
    from model.pretrain import InfoNCE
    torch.manual_seed(1)
    pre = InfoNCE("s3d", 128, 256)
    with torch.no_grad():
        w = pre.encoder_q[0].Conv_1a.conv1.weight
        w.copy_(torch.randn_like(w))
    path = os.path.join(tmp_path, "pre.pth.tar")
    torch.save({"epoch": 7, "state_dict": pre.state_dict()}, path)
    out = _cli(tmp_path, "--train_what", "last", "--epochs", "1", "--pretrain", path)
    assert "loaded pretrained checkpoint" in out and "final_fc.0.weight" in out
    ck_path = [os.path.join(d, f) for d, _, fs in os.walk(tmp_path) for f in fs if f == "epoch0.pth.tar"][0]
    ck = torch.load(ck_path, map_location="cpu", weights_only=False)
    assert torch.equal(ck["state_dict"]["backbone.Conv_1a.conv1.weight"], w.detach())
