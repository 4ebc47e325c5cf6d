"""LinearClassifier surface without a GPU: state_dict keys / shapes against the reference's (tests/golden/classifier.npz,
written by make_golden_classifier.py from the unmodified reference), the float64 oracle classifier against the
reference module's outputs and gradients, the --pretrain key mapping, and eval/main_classifier.py's options."""
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.join(ROOT, "eval"))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
import classifier_oracle as O  # noqa: E402
import make_golden as MG  # noqa: E402
import make_golden_classifier as MGC  # noqa: E402
import main_classifier as MC  # noqa: E402
from model.classifier import LinearClassifier  # noqa: E402
from model.pretrain import InfoNCE  # noqa: E402

GOLD = np.load(os.path.join(ROOT, "tests", "golden", "classifier.npz"))


@pytest.mark.parametrize("net", ["s3d", "s3dg", "r50"])
@pytest.mark.parametrize("cfg", ["last", "ft"])
def test_state_dict_keys_match_reference(net, cfg):
    ref = json.loads(str(GOLD["keys_json"]))["%s/%s" % (net, cfg)]
    m = LinearClassifier(num_class=101, network=net, dropout=0.9, **MGC.CONFIGS[cfg])
    ours = {k: list(v.shape) for k, v in m.state_dict().items()}
    assert ours == ref


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


@pytest.mark.parametrize("case,cfg", [("eval", "ft"), ("train", "last")])
def test_oracle_classifier_matches_reference(case, cfg):
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    kw = MGC.CONFIGS[cfg]
    x, w = MGC.inputs(**MGC.SHAPE)
    sd = O.classifier_state("s3d", MGC.SHAPE["num_class"], kw["use_dropout"], kw["use_final_bn"], seed=0)
    sd = {k: v.double() if v.is_floating_point() else v.clone() for k, v in sd.items()}
    params = [k for k in sd if k.endswith(".weight") or k.endswith(".bias")]
    for k in params:
        sd[k].requires_grad_(True)
    train = case == "train"
    logit, feat = O.classifier_forward(sd, x.double(), train, bn_training=train, use_l2_norm=kw["use_l2_norm"])
    (logit * w.double()).sum().backward()
    assert _rel(logit.detach().numpy(), GOLD[case + "/logit"]) < 1e-10
    assert _rel(feat.detach().numpy(), GOLD[case + "/feat3d"]) < 1e-10
    for key in GOLD.files:
        if key.startswith(case + "/grad/"):
            k = key[len(case + "/grad/"):]
            assert _rel(MG.compact(sd[k].grad.numpy(), 4096)[0], GOLD[key]) < 1e-10, k
        elif key.startswith(case + "/state/"):
            k = key[len(case + "/state/"):]
            assert _rel(sd[k].numpy(), GOLD[key]) < 1e-10, k


def test_pretrain_mapping_is_bit_exact():
    torch.manual_seed(0)
    pre = InfoNCE("s3d", 128, 256)
    with torch.no_grad():
        for v in pre.state_dict().values():
            if v.is_floating_point():
                v.copy_(torch.randn(v.shape))
    sd = pre.state_dict()
    cls = LinearClassifier(num_class=101, network="s3d", use_dropout=True)
    missing = MC.load_pretrained(cls, {"module." + k: v for k, v in sd.items()})
    assert sorted(missing) == ["final_fc.1.bias", "final_fc.1.weight"]
    csd = cls.state_dict()
    n = 0
    for k, v in sd.items():
        if k.startswith("encoder_q.0."):
            assert torch.equal(csd["backbone." + k[len("encoder_q.0."):]], v), k
            n += 1
    assert n == sum(1 for k in csd if k.startswith("backbone."))


def test_reference_flags_parse():
    flags = json.loads(str(GOLD["flags_json"]))
    argv = []
    for name, (takes_value, _) in flags.items():
        if name in ("-h", "--help"):
            continue
        argv += [name, "1"] if takes_value else [name]
    args = MC.parse_args(argv)
    assert args.train_what == "1" and args.dropout == 1.0 and args.ten_crop


@pytest.mark.parametrize("flag", [["--test", "x"], ["--retrieval"], ["--center_crop"], ["--five_crop"], ["--ten_crop"],
                                  ["--optim", "sgd"], ["--gpu", "0,1"]])
def test_unsupported_options_raise(flag):
    with pytest.raises(NotImplementedError):
        MC.check_supported(MC.parse_args(flag))


def test_adjust_learning_rate_multiplies_at_listed_epochs():
    args = MC.parse_args(["--schedule", "2", "4", "--lr", "1e-2"])

    class Opt:
        param_groups = [{"lr": 1e-3}, {"lr": 1e-2}]
    opt = Opt()
    for ep in range(6):
        MC.adjust_learning_rate(opt, ep, args)
    assert opt.param_groups[0]["lr"] == pytest.approx(1e-5) and opt.param_groups[1]["lr"] == pytest.approx(1e-4)
