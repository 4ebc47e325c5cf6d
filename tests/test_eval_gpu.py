"""Video-level testing on the H100: the per-video accumulation / finalize kernels and the retrieval kernels of
csrc/evaluate.cu against float64 (tests/tools/eval_oracle.py), packed extraction (coclr_b200.evaluate) against each video
run alone and against the float64 classifier oracle, and eval/main_classifier.py --test end to end."""
import ctypes as C
import json
import os
import pickle
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "eval"))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))

import eval_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu


def _accumulate(logits, feats, slot, acc):
    from coclr_b200 import lib as L
    B, Cn = logits.shape
    L.check(L.load().coclr_video_accumulate(L.dptr(logits), L.dptr(feats), L.dptr(slot), L.dptr(acc[0]),
                                            L.dptr(acc[1]), L.dptr(acc[2]), B, Cn, feats.shape[1], L.stream_ptr()),
            "coclr_video_accumulate")


def _finalize(acc, Nv, views_sum, n_views, target):
    from coclr_b200 import lib as L
    Cn, D = acc[0].shape[1], acc[1].shape[1]
    dev = acc[0].device
    out = dict(feat=torch.empty(Nv, D, device=dev), view=torch.empty(Nv, Cn, device=dev),
               prob=torch.empty(Nv, Cn, device=dev), rank=torch.empty(Nv, dtype=torch.int32, device=dev),
               hits=torch.zeros(2, dtype=torch.int32, device=dev))
    a = L.VideoFinalize(prob_sum=L.dptr(acc[0]), feat_sum=L.dptr(acc[1]), count=L.dptr(acc[2]), Nv=Nv, C=Cn, D=D,
                        n_views=n_views, feat_mean=L.dptr(out["feat"]), prob_mean=L.dptr(out["view"]),
                        views_sum=L.dptr(views_sum), prob=L.dptr(out["prob"]), target=L.dptr(target),
                        rank=L.dptr(out["rank"]), hits=L.dptr(out["hits"]))
    L.check(L.load().coclr_video_finalize(C.byref(a), L.stream_ptr()), "coclr_video_finalize")
    return out


@pytest.mark.parametrize("B,Cn,D", [(5, 101, 1024), (32, 400, 2048), (3, 7, 12)])
def test_accumulate_and_finalize_vs_float64(B, Cn, D, diag):
    """Clips of 1-7 per video packed B per pass (videos straddle passes), logits up to +-80, two views."""
    from coclr_b200.evaluate import pack_passes
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(B * 1000 + Cn)
    counts = [int(c) for c in torch.randint(1, 8, (37,), generator=g)]
    Nv = len(counts)
    target = torch.randint(0, Cn, (Nv,), generator=g)
    # labels the head has no class for (below 0, past C, past the last video's row): rank C, never a hit
    target[0], target[1], target[Nv - 1] = -1, Cn, Cn * Nv + 7
    target = target.to(dev)
    valid = (target >= 0) & (target < Cn)
    views_sum = torch.zeros(Nv, Cn, device=dev)
    per_view = []
    for view in range(2):
        logits = [(torch.rand(n, Cn, generator=g) * 2 - 1) * torch.tensor([80.0, 20.0, 3.0])[torch.randint(0, 3, (n, 1),
                  generator=g)] for n in counts]
        feats = [torch.randn(n, D, generator=g) for n in counts]
        acc = (torch.zeros(Nv, Cn, device=dev), torch.zeros(Nv, D, device=dev),
               torch.zeros(Nv, dtype=torch.int32, device=dev))
        for segments, slot in pack_passes(iter(counts), B):
            lp, fp = torch.randn(B, Cn) * 80, torch.randn(B, D)        # padding rows hold garbage
            for v, c, k, s in segments:
                lp[s:s + k], fp[s:s + k] = logits[v][c:c + k], feats[v][c:c + k]
            _accumulate(lp.to(dev), fp.to(dev), torch.tensor(slot, dtype=torch.int32, device=dev), acc)
        out = _finalize(acc, Nv, views_sum, view + 1, target)
        assert torch.equal(acc[2].cpu(), torch.tensor(counts, dtype=torch.int32))
        p64, f64 = zip(*[O.video_means(lg, ft) for lg, ft in zip(logits, feats)])
        p64, f64 = torch.stack(p64).to(dev), torch.stack(f64).to(dev)
        per_view.append(p64)
        mean64 = torch.stack(per_view).mean(0)
        e_p = float((out["view"].double() - p64).abs().max())
        e_f = float(((out["feat"].double() - f64).abs() / f64.abs().max()).max())
        e_m = float((out["prob"].double() - mean64).abs().max())
        assert e_p < 2e-6 and e_f < 2e-6 and e_m < 2e-6, (e_p, e_f, e_m)
        # rank on the kernel's own probabilities is exact; hits against float64 topk except where the target's
        # probability is within 4e-6 of another class's
        assert torch.equal(out["rank"].long(), O.class_rank(out["prob"], target))
        h64 = O.topk_hits(mean64, target)
        hk = torch.stack([out["rank"] < 1, out["rank"] < 5])
        tv = torch.where(valid, target, torch.zeros_like(target)).view(-1, 1)
        gap = (mean64 - mean64.gather(1, tv)).abs().scatter_(1, tv, float("inf")).min(1).values
        gap[~valid] = float("inf")
        assert (out["rank"][~valid] == Cn).all() and not hk_invalid_hit(out["rank"], valid)
        bad = (h64 != hk).any(0)
        assert not (bad & (gap > 4e-6)).any()
        assert out["hits"].tolist() == [int(hk[0].sum()), int(hk[1].sum())]
        diag["eval/accumulate/B%d_C%d_D%d/view%d" % (B, Cn, D, view)] = dict(
            prob_abs=e_p, feat_rel=e_f, views_mean_abs=e_m, near_tie_mismatches=int(bad.sum()))


def hk_invalid_hit(rank, valid):
    return bool(((rank < 5) & ~valid).any())


def _features(N, D, labels, g, spread):
    centers = torch.randn(int(labels.max()) + 1, D, generator=g)
    return (centers[labels] + spread * torch.randn(N, D, generator=g) + 0.3).float()


@pytest.mark.parametrize("Nq,Nk,D,ncls", [(3783, 9537, 1024, 101), (1530, 3570, 2048, 51), (517, 1001, 260, 37)])
def test_retrieval_vs_float64(Nq, Nk, D, ncls, diag):
    from coclr_b200 import evaluate as EV
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(Nq + Nk + D)
    ql, kl = torch.randint(0, ncls, (Nq,), generator=g), torch.randint(0, ncls, (Nk,), generator=g)
    lab = torch.cat([ql, kl])
    f = _features(Nq + Nk, D, lab, g, spread=6.0)     # R@1 0.1-0.5: the rankings are not trivial
    qf, kf = f[:Nq].contiguous(), f[Nq:].contiguous()
    kf[Nk - 1] = kf[3]            # exact duplicate train rows: ranked by the lower index
    kl[Nk - 1] = kl[3]
    kf[Nk // 2] = kf[Nk // 2 - 1]
    kl[Nk // 2] = kl[Nk // 2 - 1]
    qf, kf, ql, kl = qf.to(dev), kf.to(dev), ql.to(dev), kl.to(dev)
    ks = EV.RETRIEVAL_KS
    q64, k64, sim64 = O.retrieval_sim(qf, kf)
    qn, kn = EV.center_normalize(qf), EV.center_normalize(kf)
    e_q = float((qn.double() - q64).abs().max())
    e_k = float((kn.double() - k64).abs().max())
    assert e_q < 1e-6 and e_k < 1e-6, (e_q, e_k)       # rows have norm 1: absolute = relative to the row
    sim, rank, acc = EV.retrieval(qf, ql, kf, kl)
    sim2, rank2, acc2 = EV.retrieval(qf, ql, kf, kl)
    assert torch.equal(sim, sim2) and torch.equal(rank, rank2) and acc == acc2
    e_sim = float((sim.double() - sim64).abs().max())
    assert e_sim < 1e-5, e_sim
    # duplicate columns are bit-identical, and the kernel's rank is exactly the ordering rule on its own sim
    assert torch.equal(sim[:, Nk - 1], sim[:, 3]) and torch.equal(sim[:, Nk // 2], sim[:, Nk // 2 - 1])
    r_own, _ = O.retrieval_rank(sim.double(), ql, kl)
    assert torch.equal(rank.long(), r_own)
    dup_best = kl[Nk // 2] == ql
    r64, gap = O.retrieval_rank(sim64, ql, kl)
    h64, hk = O.hits_from_rank(r64, Nk, ks), O.hits_from_rank(rank.long(), Nk, ks)
    bad = (h64 != hk).any(0)
    near = gap < 2 * e_sim
    assert not (bad & ~near).any(), int((bad & ~near).sum())
    assert int(near.sum()) <= 3 + Nq // 100, int(near.sum())
    ref_acc = [float(h.float().mean()) for h in O.retrieval_topk(sim64, ql, kl, [k for k in ks if k <= Nk])]
    diag["eval/retrieval/%d_%d_%d" % (Nq, Nk, D)] = dict(
        norm_abs=max(e_q, e_k), sim_abs=e_sim, near_ties=int(near.sum()), hit_mismatches=int(bad.sum()),
        acc=acc, acc_fp64_topk=ref_acc, dup_best_queries=int(dup_best.sum()))
    assert all(abs(a - b) <= int(bad.sum()) / Nq + 1e-6 for a, b in zip(acc, ref_acc))


def test_retrieval_small_gallery_unmatched_queries_any_d(diag):
    """Nk below the largest k, queries whose label no train item has, D not a multiple of 4 and inputs that are
    views at an odd offset: no query without a same-label item counts as a hit, for any k."""
    from coclr_b200 import evaluate as EV
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(17)
    Nq, Nk, D = 40, 24, 10
    ql, kl = torch.randint(0, 9, (Nq,), generator=g), torch.randint(0, 6, (Nk,), generator=g)
    f = _features(Nq + Nk + 1, D, torch.cat([ql, kl, kl[:1]]), g, spread=1.0).to(dev)
    qf, kf = f[1:Nq + 1], f[Nq + 1:]                   # views at an offset of 1 and Nq + 1 rows
    ql, kl = ql.to(dev), kl.to(dev)
    unmatched = ~(ql.view(-1, 1) == kl.view(1, -1)).any(1)
    assert unmatched.any()
    sim, rank, acc = EV.retrieval(qf, ql, kf, kl)
    _, _, sim64 = O.retrieval_sim(qf, kf)
    e_sim = float((sim.double() - sim64).abs().max())
    assert e_sim < 1e-5, e_sim
    assert torch.equal(EV.similarity(qf, kf), EV.similarity(qf.contiguous().clone(), kf.clone()))
    r_own, _ = O.retrieval_rank(sim.double(), ql, kl)
    assert torch.equal(rank.long(), r_own) and (rank[unmatched] == Nk).all()
    want = O.hits_from_rank(r_own, Nk, EV.RETRIEVAL_KS).double().mean(1).tolist()
    assert all(abs(a - w) < 1e-12 for a, w in zip(acc, want)), (acc, want)
    assert abs(acc[-1] - (Nq - int(unmatched.sum())) / Nq) < 1e-12     # k = 50 > Nk: the queries that have a match
    diag["eval/retrieval/small_gallery"] = dict(sim_abs=e_sim, acc=acc, unmatched=int(unmatched.sum()))


# ---------------------------------------------------------------------------------------------------------------------
# extraction
# ---------------------------------------------------------------------------------------------------------------------
SEQ, HW = 8, 64


def _classifier(seed=0):
    from model.classifier import LinearClassifier
    import classifier_oracle as CO
    m = LinearClassifier(num_class=51, network="s3d", dropout=0.9, use_dropout=False, use_l2_norm=True,
                         use_final_bn=True)
    sd = CO.classifier_state("s3d", 51, False, True, seed=seed)
    m.load_state_dict(sd, strict=False)
    return m.cuda().eval(), sd


def _videos(counts, seed=11):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i, n in enumerate(counts):
        T = n * SEQ + (i * 3) % SEQ
        v = (0.5 + 0.25 * torch.randn(3, 1, HW, HW, generator=g) + 0.1 * torch.randn(3, T, HW, HW, generator=g))
        out.append((v.clamp(0, 1).cuda(), i % 5, "v%02d" % i))
    return out


def _alone_clips(video):
    from coclr_b200.evaluate import IMAGENET_MEAN, IMAGENET_STD
    n = video.shape[1] // SEQ
    mean = torch.tensor(IMAGENET_MEAN, device=video.device).view(3, 1, 1, 1)
    std = torch.tensor(IMAGENET_STD, device=video.device).view(3, 1, 1, 1)
    x = (video[:, :n * SEQ] - mean) / std
    return x.view(3, n, SEQ, HW, HW).permute(1, 0, 2, 3, 4).contiguous()


def test_packed_extraction_equals_each_video_alone(diag):
    from coclr_b200.evaluate import evaluate
    counts = [1, 7, 3, 2, 5, 1, 4, 6, 2]
    vids = _videos(counts)
    model, _ = _classifier()
    res = evaluate(model, vids, SEQ, batch_size=5)
    res2 = evaluate(model, vids, SEQ, batch_size=5)
    assert torch.equal(res.feature, res2.feature) and torch.equal(res.prob, res2.prob)
    assert res.vname == [n for _, _, n in vids] and res.label.tolist() == [lab for _, lab, _ in vids]
    ef, ep, bit = 0.0, 0.0, True
    for i, (v, _, _) in enumerate(vids):
        with torch.no_grad():
            lg, ft = model(_alone_clips(v))
        p, f = F.softmax(lg.double(), -1).mean(0), ft.double().mean(0)
        ef = max(ef, float((res.feature[i].double() - f).abs().max() / f.abs().max()))
        ep = max(ep, float((res.prob[i].double() - p).abs().max()))
        # the same clip through a pass of the same shape, alone (padding): bit-identical to its packed result
        alone = evaluate(model, [vids[i]], SEQ, batch_size=5)
        bit = bit and torch.equal(alone.feature[0], res.feature[i]) and torch.equal(alone.prob[0], res.prob[i])
    # labels outside the head's 51 classes: the same features and probabilities, rank 51, never a hit
    relabelled = [(v, [-1, 51, 400][i % 3] if i % 2 else lab, n) for i, (v, lab, n) in enumerate(vids)]
    odd = evaluate(model, relabelled, SEQ, batch_size=5)
    assert torch.equal(odd.feature, res.feature) and torch.equal(odd.prob, res.prob)
    assert odd.label.tolist() == [lab for _, lab, _ in relabelled]
    assert odd.rank[1::2].tolist() == [51] * len(vids[1::2]) and torch.equal(odd.rank[0::2], res.rank[0::2])
    assert odd.top5 == float((res.rank[0::2] < 5).sum()) / len(vids)
    diag["eval/packed_vs_alone"] = dict(feat_rel=ef, prob_abs=ep, bit_identical_same_pass_shape=bit)
    assert ef < 1e-5 and ep < 1e-5, (ef, ep)


def test_extraction_vs_oracle(diag):
    from coclr_b200.evaluate import evaluate
    import classifier_oracle as CO
    counts = [2, 1, 3, 1]
    vids = _videos(counts, seed=5)
    model, sd = _classifier(seed=2)
    res = evaluate(model, vids, SEQ, batch_size=4)
    sdd = {k: (v.cuda().double() if v.is_floating_point() else v.cuda()) for k, v in sd.items()}
    ef, ep = 0.0, 0.0
    for i, (v, _, _) in enumerate(vids):
        lg, ft = CO.classifier_forward(sdd, _alone_clips(v).double(), False, use_l2_norm=True)
        p, f = O.video_means(lg, ft)              # ft is l2-normalised (use_l2_norm), as the engine's feat3d
        ef = max(ef, float((res.feature[i].double() - f).abs().max() / f.abs().max()))
        ep = max(ep, float((res.prob[i].double() - p).abs().max() / p.abs().max()))
    diag["eval/extraction_vs_fp64"] = dict(feat_rel=ef, prob_rel=ep)
    assert ef < 1e-3 and ep < 1e-3, (ef, ep)


# ---------------------------------------------------------------------------------------------------------------------
# CLI
# ---------------------------------------------------------------------------------------------------------------------
def _cli(cwd, *extra):
    cmd = [sys.executable, os.path.join(ROOT, "eval", "main_classifier.py"), "--synthetic", "--net", "s3d",
           "--dataset", "hmdb51", "--batch_size", "4", "--seq_len", str(SEQ), "--img_dim", str(HW),
           "--synthetic-videos", "24"] + list(extra)
    r = subprocess.run(cmd, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:]
    return r.stdout


def test_cli_retrieval(tmp_path, diag):
    from model.pretrain import InfoNCE
    from oracle import coclr_oracle as OO
    pre = InfoNCE("s3d", 128, 256)
    pre.load_state_dict(OO.with_aliases(OO.synth_state(OO.infonce_shapes(128, 256), seed=0, ptr=0)))
    path = os.path.join(tmp_path, "model", "epoch3.pth.tar")
    os.makedirs(os.path.dirname(path))
    torch.save({"epoch": 3, "state_dict": pre.state_dict()}, path)
    out = _cli(tmp_path, "--test", path, "--retrieval")
    assert "Computing test set feature" in out and "Computing train set feature" in out
    d = os.path.join(tmp_path, "model", "feature")
    feats = {}
    for split in ("test", "train"):
        f = torch.load(os.path.join(d, "hmdb51_%s_feature.pth.tar" % split))
        lab = torch.load(os.path.join(d, "hmdb51_%s_label.pth.tar" % split))
        with open(os.path.join(d, "hmdb51_%s_vname.pkl" % split), "rb") as fp:
            vn = pickle.load(fp)
        assert f.device.type == "cpu" and f.dtype == torch.float32 and f.shape == (24, 1024)
        assert lab.dtype == torch.int64 and lab.shape == (24,)
        assert len(vn) == 24 and all(isinstance(v, list) and len(v) == 1 and isinstance(v[0], str) for v in vn)
        feats[split] = (f, lab)
    sim = torch.load(os.path.join(d, "hmdb51_sim.pth.tar"))
    assert sim.shape == (24, 24)
    printed = [float(x) for x in re.findall(r"^\d+NN acc = ([0-9.]+)$", out, re.M)]
    assert len(printed) == 5
    _, _, sim64 = O.retrieval_sim(feats["test"][0], feats["train"][0])
    r64, _ = O.retrieval_rank(sim64, feats["test"][1], feats["train"][1])
    ref = [float(h.float().mean()) for h in O.hits_from_rank(r64, 24)]
    assert ["%.4f" % a for a in printed] == ["%.4f" % a for a in ref], (printed, ref)
    assert ref[0] > 0.5                    # 8 classes: well above chance
    diag["eval/cli_retrieval_acc"] = printed
    out2 = _cli(tmp_path, "--test", path, "--retrieval")
    assert "Computing" not in out2
    assert re.findall(r"^\d+NN acc = .*$", out2, re.M) == re.findall(r"^\d+NN acc = .*$", out, re.M)


def _nearest_centroid_head(m):
    """A head that classifies the driver's synthetic videos: identity final BN, fc rows = the centred class means of
    the train split's per-video features (so the test accuracies are well above chance and a disagreement shows)."""
    import main_classifier as MC
    from coclr_b200.evaluate import evaluate
    args = MC.parse_args(["--synthetic", "--seq_len", str(SEQ), "--img_dim", str(HW), "--dataset", "hmdb51",
                          "--synthetic-videos", "24"])
    args.num_class = 51
    with torch.no_grad():
        m.final_bn.running_mean.zero_()
        m.final_bn.running_var.fill_(1.0)
        m.final_bn.weight.fill_(1.0)
        m.final_bn.bias.zero_()
        res = evaluate(m, MC.SyntheticVideos(args, "train", torch.device("cuda")), SEQ, 4)
        f = res.feature.double()
        mu = f.mean(0)
        W = torch.zeros(51, f.shape[1], dtype=torch.float64, device=f.device)
        for c in res.label.unique().tolist():
            W[c] = F.normalize(f[res.label == c].mean(0) - mu, dim=0) * 200
        m.final_fc[-1].weight.copy_(W.float())
        m.final_fc[-1].bias.copy_((-(W @ mu)).float())


@pytest.mark.parametrize("mode", ["center_crop", "five_crop", "ten_crop"])
def test_cli_crops(mode, tmp_path, diag):
    from model.classifier import LinearClassifier
    import classifier_oracle as CO
    m = LinearClassifier(num_class=51, network="s3d", dropout=0.9, use_dropout=False, use_l2_norm=True,
                         use_final_bn=True)
    m.load_state_dict(CO.classifier_state("s3d", 51, False, True, seed=4), strict=False)
    m = m.cuda()
    _nearest_centroid_head(m)
    path = os.path.join(tmp_path, "epoch9.pth.tar")
    torch.save({"epoch": 9, "state_dict": m.state_dict()}, path)
    out = _cli(tmp_path, "--test", path, "--" + mode)
    titles = {"center_crop": ["ten"], "five_crop": ["ten"], "ten_crop": ["center", "five", "ten"]}[mode]
    printed = re.findall(r"^Mean: Acc@1: ([0-9.]+) Acc@5: ([0-9.]+)$", out, re.M)
    assert len(printed) == len(titles)
    for t, (a1, a5) in zip(titles, printed):
        with open(os.path.join(tmp_path, "epoch9.pth.tar-prob-%s.json" % t)) as fp:
            stat = json.load(fp)
        assert len(stat) == 24
        prob = torch.tensor([stat[v]["mean_prob"] for v in stat], dtype=torch.float64).squeeze(1)
        target = torch.tensor([int(re.search(r"/c(\d+)/", v).group(1)) for v in stat])
        h = O.topk_hits(prob, target)
        assert (a1, a5) == ("%.4f" % float(h[0].double().mean()), "%.4f" % float(h[1].double().mean()))
    assert float(printed[0][0]) > 0.3      # 8 classes: well above chance
    diag["eval/cli_%s" % mode] = printed
