"""The feature linear probe on the H100 (coclr_b200.probe.fit, csrc/probe.cu) against the stock-torch oracle
(tests/tools/probe_oracle.py) in float64 on the device, under the same plan (same initial weights, same batches).

Features are low-rank (64 latent dims under a little full-rank noise) with overlapping classes, so the accuracies sit
between 0.3 and 0.8 rather than at 1.0 and many rows have small margins.

Per config, every state-dict tensor is bounded in relative L2 error by 4x the error of float32 torch (same plan, same
device) against float64, or a floor of FLOOR, whichever is larger; per-epoch train losses, eval losses and the final
probabilities likewise.  Train and eval hit counts must equal float64's, except for rows whose float64 top-1 margin is
below twice the measured logit error (the largest logit difference between the engine's final model and float64's on
the test set); the exempt counts are recorded in the `diag` fixture.  A 3 x 4 sweep is bit-identical, config by config,
to the 12 single runs and to a second sweep.  The CLI runs end to end on `main_classifier.py --retrieval` features.

Measured on one H100 80GB HBM3 at 700 W (lr 1.0, wd 1e-3; relative L2 error of the engine / of float32 torch):
  ucf101_bn       (9537/3783, D 1024, C 101, 100 epochs)  fc.weight 7.8e-7 / 5.8e-7, bn.bias 1.4e-6 / 1.1e-6,
                  running stats 2.1e-7 / 2.2e-7, prob 5.0e-6 / 5.6e-6 abs, losses 1.4e-7; final val acc 0.52
  ucf101          (no BN, rows scaled 1/32)                fc.weight 5.1e-7 / 5.0e-7, prob 2.6e-7 / 2.3e-7; acc 0.51
  r50_bn          (D 2048, 30 epochs)                      fc.weight 1.4e-6 / 5.5e-7, bn.bias 3.7e-6 / 1.4e-6,
                  prob 7.6e-6 / 2.0e-6; acc 0.52
  hmdb51_bn_norm  (3570/1530, C 51, 50 epochs)             fc.weight 8.2e-7 / 4.5e-7, prob 4.3e-6 / 9.7e-7; acc 0.44
  last_row_norm   (2049 rows: a last batch of one row)     fc.weight 2.7e-7 / 2.3e-7, prob 1.0e-6 / 3.5e-7; acc 0.78
Every bound held with the 1e-5 floor or 4x float32 torch.  Logit errors of the final models were 3.4e-7 to 6.5e-6; the
exempt rows were at most 3 per epoch in training and none in evaluation, and no hit count differed from float64's,
exempt rows included.
"""
import json
import os
import pickle
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "eval"))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))

import probe_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

FLOOR = 1e-5
# name -> (N, Nq, D, C, sep, fit kwargs).  "ucf101" (no BN) scales the features by 1/32 to rows of norm ~1.2: on the
# raw rows (norm ~38) SGD at lr 1.0 without BN is chaotic, and float32 torch itself ends 14-70% away from float64.
CASES = {
    "ucf101_bn": (9537, 3783, 1024, 101, 0.35, dict(epochs=100, eval_freq=5, final_bn=True)),
    "ucf101": (9537, 3783, 1024, 101, 0.35, dict(epochs=100, eval_freq=5), 1 / 32),
    "r50_bn": (9537, 3783, 2048, 101, 0.35, dict(epochs=30, eval_freq=5, schedule=(20, 25), final_bn=True)),
    "hmdb51_bn_norm": (3570, 1530, 1024, 51, 0.3, dict(epochs=50, eval_freq=5, schedule=(30, 40), final_bn=True,
                                                        normalize=True)),
    "last_row_norm": (2049, 500, 1024, 20, 0.6, dict(epochs=20, eval_freq=3, schedule=(10,), normalize=True)),
}


def features(N, Nq, D, C, sep, seed=1, r=64):
    g = torch.Generator().manual_seed(seed)
    means = sep * torch.randn(C, r, generator=g)
    P = torch.randn(r, D, generator=g) / r ** 0.5 * (torch.rand(D, generator=g) + 0.5)
    offset = 0.5 * torch.randn(D, generator=g)

    def split(n):
        y = torch.arange(n) % C
        y = y[torch.randperm(n, generator=g)]
        return (means[y] + torch.randn(n, r, generator=g)) @ P + offset + 0.05 * torch.randn(n, D, generator=g), y

    return split(N) + split(Nq)


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def series_err(a, b):
    a, b = torch.tensor(a, dtype=torch.float64), torch.tensor(b, dtype=torch.float64)
    return float(((a - b).abs() / b.abs().clamp_min(1e-30)).max())


@pytest.mark.parametrize("name", list(CASES))
def test_fit_vs_float64(name, diag):
    from coclr_b200 import probe as P
    N, Nq, D, Cn, sep, kw = CASES[name][:6]
    x = features(N, Nq, D, Cn, sep)
    if len(CASES[name]) > 6:
        x = (x[0] * CASES[name][6], x[1], x[2] * CASES[name][6], x[3])
    dev = torch.device("cuda")
    xd = [t.to(dev) for t in x]
    lr, wd = 1.0, 1e-3
    eng = P.fit(*xd, [lr], [wd], **kw)[0]
    kw_o = dict(kw)
    kw_o.setdefault("schedule", (60, 80))
    p = P.plan(N, Nq, D, Cn, [lr], kw["epochs"], 1024, kw_o["schedule"], kw["eval_freq"])
    run = lambda dtype, rec=None: O.run(*xd, lr, wd, p, kw_o["schedule"], kw.get("final_bn", False),  # noqa: E731
                                        kw.get("normalize", False), dtype=dtype, device=dev, record=rec)
    rec = {}
    r64 = run(torch.float64, rec)
    r32 = run(torch.float32)
    d = dict(val_acc_final=eng.final_acc, train_acc_last=eng.train_acc[-1])
    failures = []
    sd_e, sd_32, sd_64 = eng.state_dict(), r32.state_dict(), r64.state_dict()
    assert sorted(sd_e) == sorted(sd_64)
    for k in sd_64:
        if k.endswith("num_batches_tracked"):
            assert int(sd_e[k]) == int(sd_64[k])
            continue
        e, e32 = rel(sd_e[k], sd_64[k]), rel(sd_32[k], sd_64[k])
        d["state/" + k] = (e, e32)
        if e > max(4 * e32, FLOOR):
            failures.append((k, e, e32))
    for what, ea, a32, a64 in (("train_loss", eng.train_loss, r32.train_loss, r64.train_loss),
                               ("val_loss", eng.val_loss + [eng.final_loss], r32.val_loss + [r32.final_loss],
                                r64.val_loss + [r64.final_loss])):
        e, e32 = series_err(ea, a64), series_err(a32, a64)
        d[what] = (e, e32)
        if e > max(4 * e32, FLOOR):
            failures.append((what, e, e32))
    ep = float((eng.prob.double() - r64.prob.double()).abs().max())
    ep32 = float((r32.prob.double() - r64.prob.double()).abs().max())
    d["prob_abs"] = (ep, ep32)
    if ep > max(4 * ep32, FLOOR):
        failures.append(("prob", ep, ep32))
    # logit error of the final models on the test set, evaluated in float64
    xq = xd[2].double()
    if kw.get("normalize"):
        xq = torch.nn.functional.normalize(xq)

    def logits(sd):
        h = xq
        if "bn.weight" in sd:
            h = (h - sd["bn.running_mean"].to(dev).double()) / (sd["bn.running_var"].to(dev).double() + 1e-5).sqrt()
            h = h * sd["bn.weight"].to(dev).double() + sd["bn.bias"].to(dev).double()
        return h @ sd["fc.weight"].to(dev).double().t() + sd["fc.bias"].to(dev).double()

    lerr = float((logits(sd_e) - logits(sd_64)).abs().max())
    d["logit_err"] = lerr
    exempt_train = [int((m < 2 * lerr).sum()) for m in rec["train_margin"]]
    exempt_val = [int((m < 2 * lerr).sum()) for m in rec["val_margin"]]
    d["exempt_train_rows_max_per_epoch"], d["exempt_val_rows_max"] = max(exempt_train), max(exempt_val)
    d["hit_diff_train"] = [a - b for a, b in zip(eng.train_hits, r64.train_hits) if a != b]
    d["hit_diff_val"] = [a - b for a, b in zip(eng.val_hits + [eng.final_hits], r64.val_hits + [r64.final_hits])
                         if a != b]
    for e, (a, b) in enumerate(zip(eng.train_hits, r64.train_hits)):
        if abs(a - b) > exempt_train[e]:
            failures.append(("train_hits[%d]" % e, a, b, exempt_train[e]))
    for v, (a, b) in enumerate(zip(eng.val_hits + [eng.final_hits], r64.val_hits + [r64.final_hits])):
        if abs(a - b) > exempt_val[v]:
            failures.append(("val_hits[%d]" % v, a, b, exempt_val[v]))
    diag["probe/" + name] = d
    assert not failures, failures
    # the comparison is not vacuous: float32 stays near float64 and few rows are exempt
    assert max(v[1] for k, v in d.items() if k.startswith("state/")) < 1e-4
    assert max(exempt_train) <= 0.01 * N and max(exempt_val) <= 0.01 * Nq
    assert 0.15 <= eng.final_acc <= 0.85, eng.final_acc


def test_sweep_is_bitwise_the_single_runs_and_repeatable(diag):
    from coclr_b200 import probe as P
    x = [t.cuda() for t in features(9537, 3783, 1024, 101, 0.35)]
    lrs, wds = [0.1, 0.3, 1.0], [1e-4, 1e-3, 1e-2, 1e-1]
    kw = dict(epochs=12, eval_freq=5, schedule=(6, 10), final_bn=True)
    sweep = P.fit(*x, lrs, wds, **kw)
    again = P.fit(*x, lrs, wds, **kw)
    assert [(r.lr, r.wd) for r in sweep] == P.grid(lrs, wds)
    for i, (lr, wd) in enumerate(P.grid(lrs, wds)):
        one = P.fit(*x, [lr], [wd], **kw)[0]
        for other in (one, again[i]):
            for k, v in sweep[i].state_dict().items():
                assert torch.equal(v, other.state_dict()[k]), (lr, wd, k)
            assert torch.equal(sweep[i].prob, other.prob), (lr, wd)
            assert sweep[i].train_loss == other.train_loss and sweep[i].val_acc == other.val_acc
    diag["probe/sweep_best_acc"] = [(r.lr, r.wd, r.best_acc, r.best_epoch) for r in sweep]


def _run(cwd, script, *args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "eval", script)] + list(args), cwd=cwd,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:]
    return r.stdout


def test_cli_end_to_end(tmp_path, diag):
    from model.pretrain import InfoNCE
    from oracle import coclr_oracle as OO
    from coclr_b200 import probe as P
    pre = InfoNCE("s3d", 128, 256)
    pre.load_state_dict(OO.with_aliases(OO.synth_state(OO.infonce_shapes(128, 256), seed=0, ptr=0)))
    ckpt = os.path.join(tmp_path, "model", "epoch3.pth.tar")
    os.makedirs(os.path.dirname(ckpt))
    torch.save({"epoch": 3, "state_dict": pre.state_dict()}, ckpt)
    _run(tmp_path, "main_classifier.py", "--synthetic", "--net", "s3d", "--dataset", "ucf101", "--batch_size", "4",
         "--seq_len", "8", "--img_dim", "64", "--synthetic-videos", "24", "--test", ckpt, "--retrieval")
    d = os.path.join(tmp_path, "model", "feature")
    out = _run(tmp_path, "feature_linear_probe.py", "--test", ckpt, "--final_bn", "--epochs", "20")
    lines = out.strip().split("\n")
    assert lines[0] == "Use final BN layer in network"
    assert sum(1 for ln in lines if re.fullmatch(r"train: Epoch\[\d+\] loss \d+\.\d{4} acc \d\.\d{4}", ln)) == 20
    assert re.fullmatch(r"Final best acc: \d\.\d{4}", lines[-4]) and lines[-3] == "Save probability ... "
    path = os.path.join(d, "epoch3.pth.tar-lp-ucf101-prob.json")
    assert lines[-1] == "prob saved to %s" % path
    with open(path) as fp:
        js = json.load(fp)
    with open(os.path.join(d, "ucf101_test_vname.pkl"), "rb") as fp:
        vnames = [r[0] for r in pickle.load(fp)]
    assert list(js) == vnames
    t = lambda s, w: torch.load(os.path.join(d, "ucf101_%s_%s.pth.tar" % (s, w)))   # noqa: E731
    res = P.fit(t("train", "feature"), t("train", "label"), t("test", "feature"), t("test", "label"), [1.0], [1e-3],
                epochs=20, final_bn=True)[0]
    assert torch.equal(torch.tensor([js[v][0] for v in vnames]), res.prob)
    assert lines[-2] == "eval[{}] loss {:.4f} acc {:.4f}".format(res.best_epoch, res.final_loss, res.final_acc)
    out = _run(tmp_path, "feature_linear_probe.py", "--test", ckpt, "--final_bn", "--epochs", "20",
               "--lr", "0.1", "0.3", "1.0", "--wd", "1e-4", "1e-3", "1e-2", "1e-1")
    names = sorted(f for f in os.listdir(d) if re.fullmatch(r"epoch3\.pth\.tar-lp-ucf101-lr.*-prob\.json", f))
    assert len(names) == 12
    with open(os.path.join(d, "epoch3.pth.tar-lp-ucf101-sweep.json")) as fp:
        sweep = json.load(fp)
    assert [(s["lr"], s["wd"]) for s in sweep] == P.grid([0.1, 0.3, 1.0], [1e-4, 1e-3, 1e-2, 1e-1])
    one = [s for s in sweep if s["lr"] == 1.0 and s["wd"] == 1e-3][0]
    with open(os.path.join(d, one["prob"])) as fp:
        assert json.load(fp) == js   # the sweep's config gives the single run's bits
    assert one["best_acc"] == res.best_acc and one["best_epoch"] == res.best_epoch
    diag["probe/cli"] = dict(final_acc=res.final_acc, best_acc=res.best_acc, table=out.strip().split("\n")[:3])
