"""The two-stream merge on the H100: coclr_prob_merge and coclr_sim2_fp32 (csrc/evaluate.cu) against float64 and
against the single-stream kernels, retrieval against the unmodified reference's printed results
(tests/golden/two_stream.npz), and eval/merge_2stream_prob.py end to end in both modes."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))

import eval_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "two_stream.npz"))
SIM_CASES = sorted({k.split("/")[1] for k in GOLDEN.files if k.startswith("sim/")})
PROB_CASES = sorted({k.split("/")[1] for k in GOLDEN.files if k.startswith("prob/")})
MERGE = os.path.join(ROOT, "eval", "merge_2stream_prob.py")


def _g(case, key, kind="sim"):
    return GOLDEN["%s/%s/%s" % (kind, case, key)]


def _merge_cli(*args):
    r = subprocess.run([sys.executable, MERGE] + list(args), stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout


# ---------------------------------------------------------------------------------------------------------------------
# probability fusion
# ---------------------------------------------------------------------------------------------------------------------
def _merge_np(p1, p2, target):
    fused = (p1 + p2) / 2
    hits = [int((np.argmax(p, axis=-1) == target).sum()) for p in (p1, p2, fused)]
    return fused, hits


def _prob_inputs(Nv, C, seed):
    rng = np.random.default_rng(seed)
    p1, p2 = rng.random((Nv, C)), rng.random((Nv, C))
    target = rng.integers(0, C, Nv)
    for r in range(0, Nv, 3):                      # exact ties at the top, the target on either side
        o = int(rng.integers(0, C))
        p1[r, target[r]] = p1[r, o] = 2.0
        p2[r + 1 if r + 1 < Nv else r, o] = 3.0
    for r in range(1, Nv, 7):                      # fused-only ties
        a, b = int(target[r]), (int(target[r]) + 5) % C
        p1[r, a], p1[r, b], p2[r, a], p2[r, b] = 4.5, 3.5, 3.5, 4.5
    p1[2, 1] = np.nan                              # np.argmax takes the first NaN
    p2[4, [3, 0]] = np.nan
    target[5], target[6], target[7] = -1, C, C + 100   # outside [0, C): misses
    return p1, p2, target


@pytest.mark.parametrize("Nv,C", [(1000, 101), (257, 400), (64, 12), (9, 4), (33, 700)])
def test_prob_merge_vs_numpy(Nv, C):
    from coclr_b200 import evaluate as EV
    p1, p2, target = _prob_inputs(Nv, C, Nv + C)
    fused, acc = EV.merge_probabilities(torch.from_numpy(p1).cuda(), torch.from_numpy(p2).cuda(),
                                        torch.from_numpy(target).cuda())
    f64, hits = _merge_np(p1, p2, target)
    assert np.array_equal(fused.cpu().numpy(), f64, equal_nan=True)
    assert acc == tuple(h / Nv for h in hits), (acc, hits)
    fused2, acc2 = EV.merge_probabilities(torch.from_numpy(p1).cuda(), torch.from_numpy(p2).cuda(),
                                          torch.from_numpy(target).cuda())
    assert torch.equal(fused.nan_to_num(), fused2.nan_to_num()) and acc == acc2


@pytest.mark.parametrize("case", PROB_CASES)
def test_prob_merge_fixture_and_cli_mode_c(case, tmp_path):
    from coclr_b200 import evaluate as EV
    p1, p2, label = _g(case, "p1", "prob"), _g(case, "p2", "prob"), _g(case, "label", "prob")
    fused, acc = EV.merge_probabilities(torch.from_numpy(p1).cuda(), torch.from_numpy(p2).cuda(),
                                        torch.from_numpy(label).cuda())
    f64, hits = _merge_np(p1, p2, label)
    assert np.array_equal(fused.cpu().numpy(), f64) and acc == tuple(h / len(label) for h in hits)
    for i in (1, 2):
        (tmp_path / ("p%d.json" % i)).write_text(str(_g(case, "json%d" % i, "prob")))
    (tmp_path / "ClassInd.txt").write_text(str(_g(case, "class_text", "prob")))
    out = _merge_cli("--mode", "c", "--prob1", str(tmp_path / "p1.json"), "--prob2", str(tmp_path / "p2.json"),
                     "--dataset", str(_g(case, "dataset", "prob")), "--class-index", str(tmp_path / "ClassInd.txt"))
    assert out == "Merge classification probability\n" + str(_g(case, "stdout", "prob")), out


# ---------------------------------------------------------------------------------------------------------------------
# two-stream similarity
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Nq,Nk,D1,D2", [(3783, 9537, 1024, 1024), (517, 1001, 1024, 2048), (129, 61, 30, 18),
                                         (40, 263, 10, 7), (1, 5, 3, 4)])
def test_sim2_equals_two_calls(Nq, Nk, D1, D2, diag):
    from coclr_b200 import evaluate as EV
    g = torch.Generator().manual_seed(Nq + Nk + D1 + D2)
    f = [torch.randn(n, d, generator=g).cuda() for n, d in ((Nq, D1), (Nk, D1), (Nq, D2), (Nk, D2))]
    q1, k1, q2, k2 = (EV.center_normalize(x) for x in f)
    sim = EV.similarity2(q1, k1, q2, k2)
    assert sim.shape == (Nq, Nk)
    assert torch.equal(sim, EV.similarity(q1, k1) + EV.similarity(q2, k2))
    assert torch.equal(sim, EV.similarity2(q1, k1, q2, k2))
    sim64 = q1.double() @ k1.double().t() + q2.double() @ k2.double().t()
    e = float((sim.double() - sim64).abs().max())
    diag["two_stream/sim2/%d_%d_%d_%d" % (Nq, Nk, D1, D2)] = dict(sim_abs=e)
    assert e < 2e-5, e          # two unit-norm dot products: twice the single-stream tolerance


def _aligned(case):
    from coclr_b200 import evaluate as EV
    idx = EV.align_two_stream(*(list(_g(case, k + "/vname")) for k in ("train1", "test1", "train2", "test2")))
    tr1, te1, tr2, te2 = idx
    t = {k: torch.from_numpy(_g(case, k + "/feature")) for k in ("train1", "test1", "train2", "test2")}
    lab = {k: torch.from_numpy(_g(case, k + "/label")) for k in ("train1", "test1")}
    return (t["test1"][te1].cuda(), t["train1"][tr1].cuda(), t["test2"][te2].cuda(), t["train2"][tr2].cuda(),
            lab["test1"][te1].cuda(), lab["train1"][tr1].cuda())


@pytest.mark.parametrize("case", SIM_CASES)
def test_two_stream_retrieval_fixture(case, tmp_path, diag):
    import pickle
    from coclr_b200 import evaluate as EV
    te1, tr1, te2, tr2, ql, kl = _aligned(case)
    sim, rank, acc = EV.two_stream_retrieval(te1, tr1, te2, tr2, ql, kl)
    sim_b, rank_b, acc_b = EV.two_stream_retrieval(te1, tr1, te2, tr2, ql, kl)
    assert torch.equal(sim, sim_b) and torch.equal(rank, rank_b) and acc == acc_b
    q1, k1, _ = O.retrieval_sim(te1, tr1)
    q2, k2, _ = O.retrieval_sim(te2, tr2)
    sim64 = q1 @ k1.t() + q2 @ k2.t()
    e = float((sim.double() - sim64).abs().max())
    assert e < 2e-5, e
    Nq, Nk = sim.shape
    # the fixture's k-boundary gaps are far above the error: the reference's topk sets are float64's
    assert float(_g(case, "gaps").min()) > 50 * e
    hits64 = O.retrieval_topk(sim64, ql, kl).sum(1).tolist()
    r64, _ = O.retrieval_rank(sim64, ql, kl)
    assert O.hits_from_rank(r64, Nk).sum(1).tolist() == hits64
    assert [round(a * Nq) for a in acc] == hits64
    want = re.findall(r"^\d+NN acc = [0-9.]+$", str(_g(case, "stdout")), re.M)
    assert ["%dNN acc = %.4f" % (k, np.float32(a)) for k, a in zip(EV.RETRIEVAL_KS, acc)] == want
    diag["two_stream/retrieval/" + case] = dict(sim_abs=e, acc=acc)
    # mode s on the fixture's files prints the reference's lines
    for s, prefix in ((1, "ucf101"), (2, "ucf101-f")):
        d = tmp_path / ("s%d" % s)
        d.mkdir()
        for split in ("train", "test"):
            key = "%s%d/" % (split, s)
            torch.save(torch.from_numpy(_g(case, key + "feature")), d / ("%s_%s_feature.pth.tar" % (prefix, split)))
            torch.save(torch.from_numpy(_g(case, key + "label")), d / ("%s_%s_label.pth.tar" % (prefix, split)))
            with open(d / ("%s_%s_vname.pkl" % (prefix, split)), "wb") as fp:
                pickle.dump([[str(v)] for v in _g(case, key + "vname")], fp)
    out = _merge_cli("--mode", "s", "--prob1", str(tmp_path / "s1"), "--prob2", str(tmp_path / "s2"))
    assert out == "Merge similarity\n" + str(_g(case, "stdout")), out


def test_two_stream_retrieval_ucf101_shape(diag):
    """UCF101 split 1 (3783 test x 9537 train videos), S3D RGB + S3D flow (D = 1024 + 1024): hits equal float64's
    except for queries whose rank-deciding gap is within twice the measured error."""
    from coclr_b200 import evaluate as EV
    Nq, Nk, ncls = 3783, 9537, 101
    g = torch.Generator().manual_seed(101)
    ql, kl = torch.randint(0, ncls, (Nq,), generator=g), torch.randint(0, ncls, (Nk,), generator=g)
    lab = torch.cat([ql, kl])
    feats = []
    for _ in range(2):
        centers = torch.randn(ncls, 1024, generator=g)
        feats.append((centers[lab] + 8.0 * torch.randn(Nq + Nk, 1024, generator=g) + 0.3).cuda())
    te1, tr1, te2, tr2 = feats[0][:Nq], feats[0][Nq:], feats[1][:Nq], feats[1][Nq:]
    ql, kl = ql.cuda(), kl.cuda()
    sim, rank, acc = EV.two_stream_retrieval(te1, tr1, te2, tr2, ql, kl)
    q1, k1, _ = O.retrieval_sim(te1, tr1)
    q2, k2, _ = O.retrieval_sim(te2, tr2)
    sim64 = q1 @ k1.t() + q2 @ k2.t()
    e = float((sim.double() - sim64).abs().max())
    assert e < 2e-5, e
    r_own, _ = O.retrieval_rank(sim.double(), ql, kl)
    assert torch.equal(rank.long(), r_own)
    r64, gap = O.retrieval_rank(sim64, ql, kl)
    h64, hk = O.hits_from_rank(r64, Nk), O.hits_from_rank(rank.long(), Nk)
    bad = (h64 != hk).any(0)
    near = gap < 2 * e
    assert not (bad & ~near).any(), int((bad & ~near).sum())
    diag["two_stream/retrieval/ucf101_split1"] = dict(sim_abs=e, acc=acc, near_ties=int(near.sum()),
                                                      hit_mismatches=int(bad.sum()))


# ---------------------------------------------------------------------------------------------------------------------
# mode s end to end on the driver's own retrieval files
# ---------------------------------------------------------------------------------------------------------------------
def _retrieval_run(tmp_path, name, dataset, seed):
    from model.pretrain import InfoNCE
    from oracle import coclr_oracle as OO
    pre = InfoNCE("s3d", 128, 256)
    pre.load_state_dict(OO.with_aliases(OO.synth_state(OO.infonce_shapes(128, 256), seed=seed, ptr=0)))
    path = os.path.join(tmp_path, name, "epoch3.pth.tar")
    os.makedirs(os.path.dirname(path))
    torch.save({"epoch": 3, "state_dict": pre.state_dict()}, path)
    cmd = [sys.executable, os.path.join(ROOT, "eval", "main_classifier.py"), "--synthetic", "--net", "s3d",
           "--dataset", dataset, "--batch_size", "4", "--seq_len", "8", "--img_dim", "64", "--synthetic-videos", "24",
           "--test", path, "--retrieval"]
    r = subprocess.run(cmd, cwd=tmp_path, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:]
    return os.path.join(tmp_path, name, "feature")


def test_cli_mode_s_on_retrieval_outputs(tmp_path, diag):
    d1 = _retrieval_run(tmp_path, "rgb", "ucf101", seed=0)
    d2 = _retrieval_run(tmp_path, "flow", "ucf101-f", seed=1)
    out = _merge_cli("--mode", "s", "--dataset", "ucf101", "--prob1", d1, "--prob2", d2)
    lines = out.splitlines()
    assert lines[0] == "Merge similarity" and len(lines) == 6, out
    assert _merge_cli("--mode", "s", "--dataset", "ucf101", "--prob1", d1, "--prob2", d2) == out
    f = {}
    for s, (d, prefix) in enumerate(((d1, "ucf101"), (d2, "ucf101-f"))):
        for split in ("train", "test"):
            f[split, s] = torch.load(os.path.join(d, "%s_%s_feature.pth.tar" % (prefix, split))).cuda()
    ql = torch.load(os.path.join(d1, "ucf101_test_label.pth.tar")).cuda()
    kl = torch.load(os.path.join(d1, "ucf101_train_label.pth.tar")).cuda()
    # both streams hold the same videos in the same order: the alignment permutes both alike, which changes no hit
    q1, k1, _ = O.retrieval_sim(f["test", 0], f["train", 0])
    q2, k2, _ = O.retrieval_sim(f["test", 1], f["train", 1])
    sim64 = q1 @ k1.t() + q2 @ k2.t()
    r64, gap = O.retrieval_rank(sim64, ql, kl)
    assert float(gap.min()) > 1e-5, float(gap.min())     # no rank within fp32 error of a tie
    want = ["%dNN acc = %.4f" % (k, np.float32(float(h.double().mean())))
            for k, h in zip((1, 5, 10, 20, 50), O.hits_from_rank(r64, kl.numel()))]
    assert lines[1:] == want, (lines, want)
    diag["two_stream/cli_mode_s"] = lines[1:]
