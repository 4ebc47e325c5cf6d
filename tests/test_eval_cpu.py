"""Video-level testing without a GPU: driver flags, the pass packing planner, the rank-based hit@k against the
reference's topk / any formula, output file names and formats, and the argument checks of coclr_b200.evaluate."""
import os
import pickle
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "eval"))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))

import main_classifier as MC  # noqa: E402
import eval_oracle as O  # noqa: E402
from coclr_b200 import evaluate as EV  # noqa: E402


@pytest.mark.parametrize("flags", [["--test", "x", "--retrieval"], ["--test", "x", "--center_crop"],
                                   ["--test", "x", "--five_crop"], ["--test", "x", "--ten_crop"]])
def test_check_supported_accepts_synthetic_tests(flags):
    MC.check_supported(MC.parse_args(flags + ["--synthetic"]))
    with pytest.raises(NotImplementedError):
        MC.check_supported(MC.parse_args(flags))


def test_check_supported_still_refuses_sgd_and_multi_gpu_with_synthetic():
    for flags in (["--optim", "sgd"], ["--gpu", "0,1"]):
        with pytest.raises(NotImplementedError):
            MC.check_supported(MC.parse_args(["--synthetic", "--test", "x", "--retrieval"] + flags))


def test_missing_checkpoint_raises(tmp_path):
    args = MC.parse_args(["--synthetic", "--test", str(tmp_path / "none.pth.tar"), "--retrieval"])
    with pytest.raises(FileNotFoundError):
        MC.load_test_checkpoint(None, args)


@pytest.mark.parametrize("B", [1, 5, 32])
def test_pack_passes_covers_every_clip_once(B):
    g = torch.Generator().manual_seed(B)
    counts = [int(c) for c in torch.randint(1, 8, (40,), generator=g)] + list(range(1, 8))
    seen = []
    passes = list(EV.pack_passes(iter(counts), B))
    for i, (segments, slot) in enumerate(passes):
        assert len(slot) == B
        filled = [False] * B
        for v, c, k, s in segments:
            assert k >= 1 and slot[s:s + k] == [v] * k
            for j in range(k):
                assert not filled[s + j]
                filled[s + j] = True
                seen.append((v, c + j))
        pad = [b for b in range(B) if slot[b] == -1]
        assert pad == [b for b in range(B) if not filled[b]]
        assert not pad or (i == len(passes) - 1 and pad == list(range(B - len(pad), B)))
    # every clip exactly once, videos and their clips in order (so a straddling video keeps its clip order)
    assert seen == [(v, c) for v, n in enumerate(counts) for c in range(n)]
    assert len(passes) == -(-sum(counts) // B)
    if B > 1:
        assert any(segments[-1][3] + segments[-1][2] == B and passes[i + 1][0][0][0] == segments[-1][0]
                   for i, (segments, _) in enumerate(passes[:-1])), "no video straddles a pass"


def test_rank_hits_match_reference_topk_on_tie_free_data():
    g = torch.Generator().manual_seed(3)
    Nq, Nk, ncls = 300, 700, 25
    sim = torch.rand(Nq, Nk, generator=g, dtype=torch.float64) * 2 - 1
    assert sim.flatten().unique().numel() == sim.numel()
    ql, kl = torch.randint(0, ncls, (Nq,), generator=g), torch.randint(0, ncls, (Nk,), generator=g)
    ks = (1, 5, 10, 20, 50)
    rank, _ = O.retrieval_rank(sim, ql, kl)
    assert torch.equal(O.hits_from_rank(rank, Nk, ks), O.retrieval_topk(sim, ql, kl, ks))
    assert O.hits_from_rank(rank, Nk, ks).float().mean(1).min() > 0.02
    # and a query whose label no train item has never hits, not even for k >= Nk
    ql[0] = ncls
    rank, _ = O.retrieval_rank(sim, ql, kl)
    assert rank[0] == Nk and not O.retrieval_topk(sim, ql, kl, ks)[:, 0].any()
    assert not O.hits_from_rank(rank, Nk, (Nk, Nk + 1))[:, 0].any()
    assert torch.equal(O.hits_from_rank(rank, Nk, (Nk,)), O.retrieval_topk(sim, ql, kl, (Nk,)))


def test_class_rank_matches_topk_accuracy_on_tie_free_data():
    g = torch.Generator().manual_seed(4)
    prob = torch.softmax(torch.randn(500, 101, generator=g, dtype=torch.float64) * 3, 1)
    t = torch.randint(0, 101, (500,), generator=g)
    r = O.class_rank(prob, t)
    assert torch.equal(torch.stack([r < 1, r < 5]), O.topk_hits(prob, t, (1, 5)))
    # a target the head has no class for is ranked behind every class: a miss, as calc_topk_accuracy scores it
    t[:3] = torch.tensor([-1, 101, 400])
    r = O.class_rank(prob, t)
    assert r[:3].tolist() == [101] * 3 and torch.equal(torch.stack([r < 1, r < 5]), O.topk_hits(prob, t, (1, 5)))


def test_crop_schedule_and_file_names():
    test = os.path.join("exp", "model", "epoch9.pth.tar")
    titles = {}
    for flag in ("--center_crop", "--five_crop", "--ten_crop"):
        views, title = MC.crop_schedule(MC.parse_args(["--test", test, flag]))
        titles[flag] = [(f, a, list(after)) for f, a, after in views]
        # the final summary is written as -prob-ten.json whatever the mode (reference :515)
        assert views[-1][2][-1] == "ten"
    assert titles["--center_crop"] == [(0, 5, ["ten"])]
    assert titles["--five_crop"] == [(0, 5, []), (0, 1, []), (0, 2, []), (0, 3, []), (0, 4, ["ten"])]
    assert titles["--ten_crop"] == [(0, 5, ["center"]), (0, 1, []), (0, 2, []), (0, 3, []), (0, 4, ["five"]),
                                    (1, 5, []), (1, 1, []), (1, 2, []), (1, 3, []), (1, 4, ["ten"])]
    assert MC.prob_json_path(test, "ten") == os.path.join("exp", "model", "epoch9.pth.tar-prob-ten.json")
    args = MC.parse_args(["--test", test, "--retrieval", "--dataset", "hmdb51"])
    p = MC.retrieval_paths(args)
    assert p["dir"] == os.path.join("exp", "model", "feature")
    assert p["test", "feature"] == os.path.join("exp", "model", "feature", "hmdb51_test_feature.pth.tar")
    assert p["train", "vname"] == os.path.join("exp", "model", "feature", "hmdb51_train_vname.pkl")
    assert p["sim"] == os.path.join("exp", "model", "feature", "hmdb51_sim.pth.tar")
    args.dirname = "feat2"
    assert MC.retrieval_paths(args)["test", "label"] == os.path.join("exp", "model", "feat2", "hmdb51_test_label.pth.tar")


def test_vname_pickle_is_default_collation_at_batch_size_one(tmp_path):
    from torch.utils.data import default_collate
    names = ["a/b/v_1", "a/c/v_2"]
    rec = MC.vname_records(names)
    assert rec == [default_collate([n]) for n in names] == [["a/b/v_1"], ["a/c/v_2"]]
    with open(tmp_path / "v.pkl", "wb") as fp:
        pickle.dump(rec, fp)
    with open(tmp_path / "v.pkl", "rb") as fp:
        assert pickle.load(fp) == rec


def test_num_seq_and_short_videos_raise():
    with pytest.raises(ValueError):
        EV.evaluate(None, [], seq_len=8, batch_size=4, num_seq=2)
    with pytest.raises(ValueError):
        EV.clips_of(torch.zeros(3, 7, 4, 4), seq_len=8)
    assert EV.clips_of(torch.zeros(3, 23, 4, 4), seq_len=8) == 2


def test_synthetic_videos():
    args = MC.parse_args(["--synthetic", "--seq_len", "4", "--img_dim", "8", "--dataset", "hmdb51",
                          "--synthetic-videos", "12"])
    args.num_class = 51
    vids = list(MC.SyntheticVideos(args, "test", torch.device("cpu")))
    assert len(vids) == 12
    assert {EV.clips_of(v, 4) for v, _, _ in vids} == {1, 2, 3, 4}
    assert all(v.min() >= 0 and v.max() <= 1 and v.shape[0] == 3 and v.shape[2:] == (8, 8) for v, _, _ in vids)
    assert len({n for _, _, n in vids}) == 12 and {lab for _, lab, _ in vids} == {0, 1, 2, 3}
    again = list(MC.SyntheticVideos(args, "test", torch.device("cpu")))
    assert all(torch.equal(a[0], b[0]) for a, b in zip(vids, again))
    flipped = list(MC.SyntheticVideos(args, "test", torch.device("cpu"), view=(1, 1)))
    assert not torch.equal(flipped[0][0], vids[0][0])
