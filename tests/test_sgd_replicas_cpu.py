"""SGD and DataParallel replicas without a GPU: the float64 DataParallel oracle (tests/tools/replica_oracle.py) against
what the unmodified reference LinearClassifier computed under DataParallel's rules (tests/golden/replicas.npz), the
replica split against torch.chunk, and eval/main_classifier.py's --optim sgd / --gpu list handling."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "eval"))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import classifier_oracle as O  # noqa: E402
import main_classifier as MC  # noqa: E402
import make_golden as MG  # noqa: E402
import make_golden_classifier as MGC  # noqa: E402
import make_golden_replicas as MGR  # noqa: E402
import replica_oracle as RO  # noqa: E402
from coclr_b200 import _signatures, moco  # noqa: E402
from model.classifier import LinearClassifier, replica_chunks  # noqa: E402

GOLD = np.load(os.path.join(ROOT, "tests", "golden", "replicas.npz"))


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def test_sgd_step_is_declared():
    assert _signatures.EXPORTS["coclr_sgd_step"] == (_signatures.I, [_signatures.P, _signatures.I, _signatures.P])


@pytest.mark.parametrize("B,R", [(8, 3), (5, 4), (4, 2), (64, 2), (1, 2), (7, 7), (3, 5), (33, 2)])
def test_replica_chunks_match_torch_chunk(B, R):
    ref = [c.shape[0] for c in torch.chunk(torch.empty(B), R)]
    got = replica_chunks(B, R)
    assert [r1 - r0 for r0, r1 in got] == ref
    assert got[0][0] == 0 and got[-1][1] == B and all(a[1] == b[0] for a, b in zip(got, got[1:]))


def test_replica_chunks_examples():
    assert [r1 - r0 for r0, r1 in replica_chunks(8, 3)] == [3, 3, 2]
    assert [r1 - r0 for r0, r1 in replica_chunks(5, 4)] == [2, 2, 1]


def test_replicas_argument():
    assert LinearClassifier(num_class=11, network="s3d").replicas == 1
    assert LinearClassifier(num_class=11, network="s3d", replicas=3).replicas == 3
    with pytest.raises(ValueError):
        LinearClassifier(num_class=11, network="s3d", replicas=0)


@pytest.mark.parametrize("case", sorted(MGR.CASES))
def test_replica_oracle_matches_reference(case):
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    cfg, R, B = MGR.CASES[case]
    kw = MGC.CONFIGS[cfg]
    sd = O.classifier_state("s3d", MGR.SHAPE["num_class"], kw["use_dropout"], kw["use_final_bn"], seed=0)
    sd = {k: v.double() if v.is_floating_point() else v.clone() for k, v in sd.items()}
    trained = [k for k in sd if (k.endswith(".weight") or k.endswith(".bias"))
               and (cfg == "ft" or not k.startswith("backbone."))]
    for k in trained:
        sd[k].requires_grad_(True)
    x, y = MGR.case_inputs(B, MGR.SHAPE["num_class"])
    last = cfg == "last"
    logit, _ = RO.dataparallel_forward(sd, x.double(), R, backbone_training=not last, bn_training=last,
                                       use_l2_norm=kw["use_l2_norm"])
    loss = F.cross_entropy(logit, y)
    loss.backward()
    assert _rel(logit.detach().numpy(), GOLD[case + "/logit"]) < 1e-10
    assert abs(float(loss.detach()) - float(GOLD[case + "/loss"])) < 1e-10
    for k in MGR.grad_keys(cfg):
        assert _rel(MG.compact(sd[k].grad.numpy(), 4096)[0], GOLD["%s/grad/%s" % (case, k)]) < 1e-10, k
    for k in MGR.state_keys(cfg):
        assert _rel(sd[k].numpy(), GOLD["%s/state/%s" % (case, k)]) < 1e-10, k
    # only chunk 0 counts towards num_batches_tracked
    init = O.classifier_state("s3d", MGR.SHAPE["num_class"], kw["use_dropout"], kw["use_final_bn"], seed=0)
    k = "final_bn.num_batches_tracked" if last else "backbone.Conv_2b.bn.num_batches_tracked"
    assert int(sd[k]) == int(init[k]) + 1


def _args(*flags):
    args = MC.parse_args(list(flags))
    MC.check_supported(args)
    return args


def test_gpu_list_doubles_the_batch(capsys):
    args = _args("--synthetic", "--gpu", "0,1", "--batch_size", "32")
    MC.apply_gpu_list(args)
    assert args.replicas == 2 and args.batch_size == 64
    assert "=> Effective BatchSize = 64" in capsys.readouterr().out
    args.num_class = 101
    assert MC.build_model(args).replicas == 2


def test_single_gpu_and_no_gpu_are_unchanged(capsys):
    for flags in (["--gpu", "0"], []):
        args = _args("--synthetic", "--batch_size", "32", *flags)
        MC.apply_gpu_list(args)
        assert args.replicas == 1 and args.batch_size == 32
    assert "Effective" not in capsys.readouterr().out


def _spans(model):
    """flat_spans without a device: the module's parameters concatenated (stand-ins with the right sizes)."""
    def flat(ps):
        n = sum(p.numel() for p in ps)
        return torch.zeros(n), torch.zeros(n)
    head = [p for n, p in model.named_parameters() if not n.startswith("backbone.")]
    return {"backbone": flat(list(model.backbone.parameters())), "head": flat(head)}


@pytest.mark.parametrize("train_what,groups", [("last", {"head": 0.1}), ("ft", {"backbone": 0.01, "head": 0.1}),
                                               ("all", {"backbone": 0.1, "head": 0.1})])
def test_sgd_groups(train_what, groups, monkeypatch):
    args = _args("--synthetic", "--optim", "sgd", "--lr", "0.1", "--wd", "1e-3", "--train_what", train_what)
    args.num_class = 11
    model = MC.build_model(args)
    monkeypatch.setattr(model, "flat_spans", lambda: _spans(model))
    opt = MC.build_optimizer(model, args)
    assert isinstance(opt, moco.SpanSGD)
    assert {g["name"]: g["lr"] for g in opt.param_groups} == pytest.approx(groups)
    assert [g["name"] for g in opt.param_groups][-1] == "head"
    assert all(g["momentum"] == 0.9 and g["weight_decay"] == 1e-3 for g in opt.param_groups)
    assert all(b is None for b in opt.state_dict()["momentum_buffer"])


def test_adam_state_into_sgd_raises():
    p, g = torch.zeros(8), torch.zeros(8)
    adam = moco.SpanAdam([dict(name="head", params=p, grad=g, lr=1e-3)])
    sgd = moco.SpanSGD([dict(name="head", params=p, grad=g, lr=1e-3)])
    with pytest.raises(ValueError, match="SpanAdam.*SpanSGD"):
        sgd.load_state_dict(adam.state_dict())


def test_sgd_state_without_buffers_round_trips():
    p, g = torch.zeros(8), torch.zeros(8)
    a = moco.SpanSGD([dict(name="head", params=p, grad=g, lr=0.1)], weight_decay=1e-3)
    a.param_groups[0]["lr"] = 0.01
    b = moco.SpanSGD([dict(name="head", params=p, grad=g, lr=0.1)], weight_decay=1e-3)
    b.load_state_dict(a.state_dict())
    assert b.param_groups[0]["lr"] == 0.01 and b.momentum_buffer == [None]
    with pytest.raises(ValueError):
        moco.SpanSGD([dict(name="other", params=p, grad=g, lr=0.1)]).load_state_dict(a.state_dict())


def test_sgd_path_name(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    args = _args("--synthetic", "--optim", "sgd", "--gpu", "0,1", "--batch_size", "32", "--train_what", "last")
    MC.apply_gpu_list(args)
    path = MC.set_path(args)
    assert "_s3d_SGD_bs64_" in path and "_Adam" not in path
    args = _args("--synthetic", "--batch_size", "32")
    MC.apply_gpu_list(args)
    assert "_s3d_Adam_bs32_" in MC.set_path(args)


@pytest.mark.parametrize("flags", [["--optim", "rmsprop"], ["--synthetic", "--optim", "rmsprop"],
                                   ["--synthetic", "--optim", "adamw"]])
def test_other_optimizers_still_raise(flags):
    with pytest.raises(NotImplementedError):
        MC.check_supported(MC.parse_args(flags))


@pytest.mark.parametrize("flags", [["--optim", "sgd"], ["--gpu", "0,1"]])
def test_sgd_and_gpu_list_need_synthetic_training(flags):
    MC.check_supported(MC.parse_args(["--synthetic"] + flags))
    for extra in ([], ["--synthetic", "--test", "x", "--center_crop"]):
        with pytest.raises(NotImplementedError):
            MC.check_supported(MC.parse_args(extra + flags))
