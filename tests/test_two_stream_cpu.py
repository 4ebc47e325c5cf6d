"""The host side of the two-stream merge (eval/merge_2stream_prob.py, coclr_b200.evaluate): the name alignment, label
parsing and class-list reading against what the unmodified reference did on tests/golden/two_stream.npz, the flags, and
every input the merge rejects with a ValueError."""
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "eval"))

import merge_2stream_prob as M  # noqa: E402
from coclr_b200 import evaluate as EV  # noqa: E402

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "two_stream.npz"))
SIM_CASES = sorted({k.split("/")[1] for k in GOLDEN.files if k.startswith("sim/")})
PROB_CASES = sorted({k.split("/")[1] for k in GOLDEN.files if k.startswith("prob/")})


def _g(case, key, kind="sim"):
    return GOLDEN["%s/%s/%s" % (kind, case, key)]


def _records(names):
    return [[str(v)] for v in names]          # what --test --retrieval pickles


@pytest.mark.parametrize("case", SIM_CASES)
def test_alignment_equals_reference_order(case):
    idx = EV.align_two_stream(_records(_g(case, "train1/vname")), _records(_g(case, "test1/vname")),
                              _records(_g(case, "train2/vname")), _records(_g(case, "test2/vname")))
    for got, key in zip(idx, ("train1", "test1", "train2", "test2")):
        assert got.dtype == torch.int64
        assert np.array_equal(got.numpy(), _g(case, "order_" + key)), key
    # flat name lists give the same indices
    flat = EV.align_two_stream(*(list(_g(case, k + "/vname")) for k in ("train1", "test1", "train2", "test2")))
    assert all(torch.equal(a, b) for a, b in zip(idx, flat))


def test_fixture_covers_both_filter_branches_and_odd_shapes():
    n = {c: (len(_g(c, "train1/vname")), len(_g(c, "train2/vname")), len(_g(c, "order_train1"))) for c in SIM_CASES}
    assert any(a > b and k < a for a, b, k in n.values())                # stream 1 filtered
    assert any(a < b for a, b, k in n.values())                          # stream 2 filtered
    assert n["both"][0] < n["both"][1] and n["both"][2] < n["both"][0]   # both branches
    assert any(k % 4 for _, _, k in n.values())
    assert any(_g(c, "train1/feature").shape[1] != _g(c, "train2/feature").shape[1] for c in SIM_CASES)
    assert any(_g(c, "train1/feature").shape[1] % 4 for c in SIM_CASES)
    assert all(float(_g(c, "gaps").min()) > 1e-4 for c in SIM_CASES)


@pytest.mark.parametrize("case", PROB_CASES)
def test_labels_and_class_index_equal_reference(case, tmp_path):
    path = tmp_path / "ClassInd.txt"
    path.write_text(str(_g(case, "class_text", "prob")))
    actions = M.read_class_index(str(path))
    assert actions == [str(a) for a in _g(case, "action_list", "prob")]
    dataset = str(_g(case, "dataset", "prob"))
    to_idx = dict(zip(actions, range(len(actions))))
    labels = [to_idx[M.action_of(str(v), dataset)] for v in _g(case, "vname", "prob")]
    assert labels == _g(case, "label", "prob").tolist()


@pytest.mark.parametrize("case", PROB_CASES)
def test_load_probabilities_reads_both_value_formats(case, tmp_path):
    for i in (1, 2):
        (tmp_path / ("p%d.json" % i)).write_text(str(_g(case, "json%d" % i, "prob")))
    (tmp_path / "c.txt").write_text(str(_g(case, "class_text", "prob")))
    args = M.parse_args(["--prob1", str(tmp_path / "p1.json"), "--prob2", str(tmp_path / "p2.json"), "--dataset",
                         str(_g(case, "dataset", "prob")), "--class-index", str(tmp_path / "c.txt")])
    p1, p2, target = M.load_probabilities(args)
    assert np.array_equal(p1, _g(case, "p1", "prob")) and np.array_equal(p2, _g(case, "p2", "prob"))
    assert np.array_equal(target, _g(case, "label", "prob"))


def test_class_index_reading(tmp_path):
    p = tmp_path / "c.txt"
    p.write_text("1,ApplyEyeMakeup\n2,Archery \n  3,Baby,Crawling\n\n")
    assert M.read_class_index(str(p)) == ["ApplyEyeMakeup", "Archery", "Crawling", ""]
    p.write_text("1 ApplyEyeMakeup\n2,Archery\n")            # no ',' in the first line: lines are kept whole
    assert M.read_class_index(str(p)) == ["1 ApplyEyeMakeup", "2,Archery"]
    p.write_text("air drumming\nabseiling")
    assert M.read_class_index(str(p)) == ["air drumming", "abseiling"]


def test_action_of():
    assert M.action_of("/d/ucf101/frame/Archery/v_Archery_g01_c02/", "ucf101") == "Archery"
    assert M.action_of("/d/hmdb51/frame/brush_hair/clip_3/", "hmdb51") == "brush_hair"
    assert M.action_of("/d/k400/val/air drumming/yt01_000010_000020", "k400") == "air drumming"
    with pytest.raises(ValueError, match="no action field"):
        M.action_of("v_Archery_g01_c02/", "ucf101")


def test_flags():
    a = M.parse_args(["--class-index", "c.txt"])
    assert (a.prob1, a.prob2, a.dataset, a.mode, a.class_index) == ("", "", "ucf101", "c", "c.txt")
    a = M.parse_args(["--mode", "s", "--prob1", "A", "--prob2", "B", "--dataset", "hmdb51"])
    assert (a.prob1, a.prob2, a.dataset, a.mode, a.class_index) == ("A", "B", "hmdb51", "s", None)
    with pytest.raises(SystemExit):
        M.parse_args(["--mode", "c"])                     # mode c needs the class list
    with pytest.raises(SystemExit):
        M.parse_args(["--mode", "x", "--class-index", "c.txt"])


def _write_probs(tmp_path, d1, d2, classes="A\nB\n"):
    (tmp_path / "p1.json").write_text(json.dumps(d1))
    (tmp_path / "p2.json").write_text(json.dumps(d2))
    (tmp_path / "c.txt").write_text(classes)
    return M.parse_args(["--prob1", str(tmp_path / "p1.json"), "--prob2", str(tmp_path / "p2.json"),
                         "--class-index", str(tmp_path / "c.txt")])


def test_load_probabilities_errors(tmp_path):
    v, w = "/f/A/v_A_g01_c01/", "/f/B/v_B_g01_c01/"
    with pytest.raises(ValueError, match="v_B_g01_c01.*is not in"):
        M.load_probabilities(_write_probs(tmp_path, {v: [0.5, 0.5], w: [0.1, 0.9]}, {v: [0.5, 0.5]}))
    with pytest.raises(ValueError, match="action 'C'"):
        M.load_probabilities(_write_probs(tmp_path, {"/f/C/v_C/": [1.0, 0.0]}, {"/f/C/v_C/": [1.0, 0.0]}))
    with pytest.raises(ValueError, match="not one row"):
        M.load_probabilities(_write_probs(tmp_path, {v: [[0.5, 0.5], [0.5, 0.5]]}, {v: [0.5, 0.5]}))
    with pytest.raises(ValueError, match="different numbers of classes"):
        M.load_probabilities(_write_probs(tmp_path, {v: [0.5, 0.5]}, {v: {"mean_prob": [[0.2, 0.3, 0.5]]}}))
    with pytest.raises(ValueError, match="holds no videos"):
        M.load_probabilities(_write_probs(tmp_path, {}, {}))


def test_align_errors():
    tr, te = ["a/", "b/", "c/"], ["x/", "y/"]
    with pytest.raises(ValueError, match=r"train video 1 differs after alignment: 'b/' in stream 1, 'bb/' in stream 2"):
        EV.align_two_stream(tr, te, ["c/", "bb/", "a/"], te)
    with pytest.raises(ValueError, match=r"test video 0 differs after alignment: 'x/' in stream 1, 'w/'"):
        EV.align_two_stream(tr, te, tr, ["y/", "w/"])
    # stream 2 has more train videos: its test list is filtered by name, and an extra stream 1 test video remains
    with pytest.raises(ValueError, match="after alignment stream 1 has 3 test videos and stream 2 has 2"):
        EV.align_two_stream(tr, ["x/", "y/", "z/"], tr + ["d/"], te + ["u/"])


def test_merge_and_retrieval_shape_errors():
    with pytest.raises(ValueError, match="same non-empty shape"):
        EV.merge_probabilities(torch.zeros(3, 4, dtype=torch.float64), torch.zeros(3, 5, dtype=torch.float64),
                               torch.zeros(3, dtype=torch.long))
    with pytest.raises(ValueError, match="same non-empty shape"):
        EV.merge_probabilities(torch.zeros(0, 4, dtype=torch.float64), torch.zeros(0, 4, dtype=torch.float64),
                               torch.zeros(0, dtype=torch.long))
    with pytest.raises(ValueError, match="align them first"):
        EV.two_stream_retrieval(torch.zeros(3, 8), torch.zeros(5, 8), torch.zeros(2, 4), torch.zeros(5, 4),
                                torch.zeros(3, dtype=torch.long), torch.zeros(5, dtype=torch.long))
