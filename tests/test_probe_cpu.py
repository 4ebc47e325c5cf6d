"""The feature linear probe without a GPU: coclr_b200.probe.plan against the unmodified reference
(tests/golden/feature_probe.npz, written by tests/golden/make_golden_probe.py), the stock-torch oracle over the plan's
batches against the reference's trajectory, and the driver's flags, lines, file names and input checks."""
import argparse
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "eval"))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))

import feature_linear_probe as FLP  # noqa: E402
import probe_oracle as O  # noqa: E402
from coclr_b200 import probe as P  # noqa: E402

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "feature_probe.npz"))
CASES = ["bn", "norm", "bn_norm"]


def case(name):
    t = lambda k: torch.from_numpy(GOLDEN[name + "/" + k])   # noqa: E731
    args = FLP.parse_args(["--test", "<DIR>/model.pth.tar"] + json.loads(str(GOLDEN[name + "/flags"])))
    state = {k.split("/", 2)[2]: torch.from_numpy(GOLDEN[k]) for k in GOLDEN.files if k.startswith(name + "/state/")}
    init = {k.split("/", 2)[2]: torch.from_numpy(GOLDEN[k]) for k in GOLDEN.files if k.startswith(name + "/init/")}
    return dict(x=(t("train_feature"), t("train_label"), t("test_feature"), t("test_label")), args=args, state=state,
                init=init, prob=t("prob"), stdout=str(GOLDEN[name + "/stdout"]), vname=list(GOLDEN[name + "/vname"]))


def oracle(c, dtype):
    a = c["args"]
    return O.fit(*c["x"], a.lr, a.wd, a.epochs, a.batch_size, a.schedule, a.eval_freq, a.final_bn, a.normalize,
                 dtype=dtype)[0]


@pytest.mark.parametrize("name", CASES)
def test_plan_init_is_the_reference_lp(name):
    c = case(name)
    N, Nq, D = c["x"][0].shape[0], c["x"][2].shape[0], c["x"][0].shape[1]
    Cn = int(c["x"][1].max()) + 1
    p = P.plan(N, Nq, D, Cn)
    assert torch.equal(p.weight, c["init"]["fc.weight"]) and torch.equal(p.bias, c["init"]["fc.bias"])
    if c["args"].final_bn:
        assert torch.equal(c["init"]["bn.weight"], torch.ones(D)) and torch.equal(c["init"]["bn.bias"], torch.zeros(D))


def test_plan_leaves_the_callers_rng_alone():
    torch.manual_seed(123)
    before = torch.random.get_rng_state()
    P.plan(50, 20, 8, 3, epochs=4, batch_size=16, eval_freq=2)
    assert torch.equal(before, torch.random.get_rng_state())


def test_plan_order_and_lr_table():
    p = P.plan(37, 11, 8, 3, lrs=[1.0, 0.3], epochs=5, batch_size=16, schedule=[2, 4], eval_freq=2)
    assert p.order.shape == (5, 37)
    for e in range(5):
        assert sorted(p.order[e].tolist()) == list(range(37))
        assert [len(b) for b in p.batches(e)] == [16, 16, 5]
    assert p.eval_epochs == [0, 2, 4]
    assert p.lr[:, 0].tolist() == [1.0, 1.0, 0.1, 0.1, 1.0 * 0.1 * 0.1]
    assert p.lr[1, 1].item() == 0.3 and p.lr[4, 1].item() == 0.3 * 0.1 * 0.1
    assert not torch.equal(p.order[0], p.order[1])


@pytest.mark.parametrize("name", CASES)
def test_float32_oracle_reproduces_the_reference(name):
    """Same batches, same modules: state dict, probabilities and every printed line of the reference."""
    c = case(name)
    res = oracle(c, torch.float32)
    sd = res.state_dict()
    assert sorted(sd) == sorted(c["state"])
    for k, v in c["state"].items():
        if k.endswith("num_batches_tracked"):
            assert int(sd[k]) == int(v)
        else:
            assert float((sd[k].double() - v.double()).abs().max()) < 1e-5, k
    assert float((res.prob.double() - c["prob"]).abs().max()) < 1e-5
    path = "<DIR>/feature/model.pth.tar-lp-ucf101-prob.json"
    assert FLP.prob_path(c["args"]) == path
    lines = FLP.preamble(c["args"]) + FLP.report_lines(res, c["args"], path)
    assert lines == c["stdout"].strip("\n").split("\n")


@pytest.mark.parametrize("name", CASES)
def test_float64_oracle_stays_close_to_the_reference(name):
    c = case(name)
    res = oracle(c, torch.float64)
    for k, v in c["state"].items():
        if not k.endswith("num_batches_tracked"):
            ref = v.double()
            assert float((res.state_dict()[k] - ref).norm() / ref.norm().clamp_min(1e-12)) < 1e-5, k
    assert float((res.prob - c["prob"]).abs().max()) < 1e-5
    printed = [float(x) for x in FLP.report_lines(res, c["args"], "")[-2].split()[-3::2]]
    golden = [float(x) for x in c["stdout"].strip().split("\n")[-2].split()[-3::2]]
    assert np.allclose(printed, golden, atol=1e-4)


def test_saved_probabilities_are_the_final_models():
    """The reference's best_model aliases the live parameters: the JSON holds the final model's probabilities, and
    the closing line prints the final model's numbers under the best epoch.  In the `bn` case the best epoch (6) is
    not the last one (7), and the final model differs from the best epoch's."""
    c = case("bn")
    res = oracle(c, torch.float32)
    assert res.best_epoch == 6 and len(res.train_loss) == 8
    closing = c["stdout"].strip().split("\n")[-2]
    assert closing == "eval[6] loss {:.4f} acc {:.4f}".format(res.final_loss, res.final_acc)
    assert res.final_acc != res.val_acc[res.eval_epochs.index(6)]
    js = FLP.prob_json(res, c["vname"])
    assert list(js) == c["vname"] and all(len(v) == 1 and len(v[0]) == 5 for v in js.values())
    assert np.allclose(np.array([js[v][0] for v in c["vname"]]), c["prob"].numpy(), atol=1e-5)


def test_flags_match_the_reference():
    a = FLP.parse_args([])
    assert (a.test, a.dataset, a.dirname, a.batch_size, a.lr, a.wd, a.epochs, a.eval_freq, a.verbose, a.schedule,
            a.normalize, a.final_bn) == ("", "ucf101", "feature", 1024, [1.0], [1e-3], 100, 5, 0, [60, 80], False,
                                         False)
    a = FLP.parse_args(["--lr", "0.1", "0.3", "1.0", "--wd", "1e-4", "1e-3", "1e-2", "1e-1", "--schedule"])
    assert a.lr == [0.1, 0.3, 1.0] and a.wd == [1e-4, 1e-3, 1e-2, 1e-1] and a.schedule == []
    assert FLP.is_sweep(a) and not FLP.is_sweep(FLP.parse_args(["--lr", "0.5"]))


def test_grid_order_and_sweep_file_names():
    a = FLP.parse_args(["--test", "/x/model/epoch3.pth.tar", "--dataset", "hmdb51", "--lr", "0.1", "1.0",
                        "--wd", "1e-4", "1e-3"])
    assert P.grid(a.lr, a.wd) == [(0.1, 1e-4), (0.1, 1e-3), (1.0, 1e-4), (1.0, 1e-3)]
    names = [os.path.basename(FLP.prob_path(a, lr, wd)) for lr, wd in P.grid(a.lr, a.wd)]
    assert names == ["epoch3.pth.tar-lp-hmdb51-lr0.1-wd0.0001-prob.json",
                     "epoch3.pth.tar-lp-hmdb51-lr0.1-wd0.001-prob.json",
                     "epoch3.pth.tar-lp-hmdb51-lr1-wd0.0001-prob.json", "epoch3.pth.tar-lp-hmdb51-lr1-wd0.001-prob.json"]
    assert FLP.sweep_path(a) == "/x/model/feature/epoch3.pth.tar-lp-hmdb51-sweep.json"
    one = FLP.parse_args(["--test", "/x/model/epoch3.pth.tar"])
    assert FLP.prob_path(one) == "/x/model/feature/epoch3.pth.tar-lp-ucf101-prob.json"
    assert FLP.input_paths(one)["test_vname"] == "/x/model/feature/ucf101_test_vname.pkl"


def test_vname_records_unwrap_as_the_reference_collates_them():
    assert FLP.unwrap_vnames([["a/v1"], ["b/v2"]]) == ["a/v1", "b/v2"]
    assert FLP.unwrap_vnames(["a/v1", "b/v2"]) == ["a/v1", "b/v2"]


def test_missing_features_exit_zero(tmp_path, capsys):
    with pytest.raises(SystemExit) as e:
        FLP.main(["--test", str(tmp_path / "model.pth.tar")])
    assert e.value.code == 0
    assert capsys.readouterr().out == "feature path does not exist\n"


def _inputs(N=40, Nq=10, D=8, C=4):
    g = torch.Generator().manual_seed(0)
    return (torch.randn(N, D, generator=g), torch.arange(N) % C, torch.randn(Nq, D, generator=g), torch.arange(Nq) % C)


def test_value_errors_before_anything_runs():
    xtr, ytr, xte, yte = _inputs()
    with pytest.raises(ValueError, match="test label 4 is outside the 4 classes"):
        P.fit(xtr, ytr, xte, torch.where(yte == 0, torch.tensor(4), yte), [1.0], [1e-3], epochs=1)
    with pytest.raises(ValueError, match="train label -1"):
        P.fit(xtr, torch.where(ytr == 0, torch.tensor(-1), ytr), xte, yte, [1.0], [1e-3], epochs=1)
    # 41 rows at batch 8: the last batch has one row
    x41, y41 = torch.cat([xtr, xtr[:1]]), torch.cat([ytr, ytr[:1]])
    with pytest.raises(ValueError, match="last training batch has one row"):
        P.fit(x41, y41, xte, yte, [1.0], [1e-3], epochs=1, batch_size=8, final_bn=True)
    with pytest.raises(ValueError, match="at least one value"):
        P.fit(xtr, ytr, xte, yte, [], [1e-3])
    # without BN a one-row batch is fine (checked on the host, no device needed)
    assert P.check_inputs(x41, y41, xte, yte, 1, 8, 1, False) == (41, 10, 8, 4)


def test_best_epoch_is_the_last_to_reach_the_best():
    """summarize's `>=`: two evaluations with equal accuracy -> the later epoch is the best."""
    sizes_q = 4
    val_hits = [[2], [3], [3], [1], [0]]   # evals at epochs 0, 2, 4, 6, then the final pass
    res = P.summarize(1.0, 0.0, [[1.0]] * 7, [[1]] * 7, [[1.0]] * 5, val_hits, [0, 2, 4, 6], 2, sizes_q, 8,
                      torch.zeros(sizes_q, 3), {})
    assert res.val_acc == [0.5, 0.75, 0.75, 0.25] and res.best_acc == 0.75 and res.best_epoch == 4
    assert res.final_acc == 0.0 and res.final_hits == 0


def test_reference_shaped_oracle_matches_the_plain_one():
    xtr, ytr, xte, yte = _inputs()
    kw = dict(epochs=3, batch_size=16, schedule=[2], eval_freq=2, final_bn=True, dtype=torch.float32)
    a = O.fit(xtr, ytr, xte, yte, [0.5], [1e-3], **kw)[0]
    b = O.fit(xtr, ytr, xte, yte, [0.5], [1e-3], reference_shaped=True, **kw)[0]
    for k, v in a.state_dict().items():
        assert torch.equal(v, b.state_dict()[k]), k
    assert a.val_acc == b.val_acc and a.train_hits == b.train_hits
