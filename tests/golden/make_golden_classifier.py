"""Writes tests/golden/classifier.npz from the UNMODIFIED reference ($COCLR_REFERENCE):

  * the state_dict keys and shapes of its LinearClassifier (model/classifier.py) for s3d, s3dg and r50, in the linear-
    probe configuration (`--train_what last`: l2norm + final BN, no dropout) and the fine-tune one (dropout 0.9);
  * float64 forward and gradients of the S3D LinearClassifier from tests/tools/classifier_oracle.py (classifier_state) on seeded clips:
    eval mode with the dropout head, and train mode with l2norm + final BN (no dropout);
  * the option names of eval/main_classifier.py.

Run in the build container only:  COCLR_REFERENCE=<checkout> python tests/golden/make_golden_classifier.py
"""
import importlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
from make_golden import REF, compact  # noqa: E402
from make_golden_cli import ref_flags  # noqa: E402

OUT = os.path.join(HERE, "classifier.npz")
CONFIGS = {"last": dict(use_dropout=False, use_l2_norm=True, use_final_bn=True),
           "ft": dict(use_dropout=True, use_l2_norm=False, use_final_bn=False)}
GRAD_KEYS = ["backbone.Conv_1a.conv1.weight", "backbone.Conv_2c.bn1.weight", "backbone.Mixed_4c.branch2.0.conv.weight",
             "backbone.Mixed_5c.branch1.1.conv2.weight", "backbone.Mixed_5c.branch3.1.bn.bias"]
SHAPE = dict(B=4, T=8, HW=64, num_class=51)


def inputs(B, T, HW, num_class, seed=4321):
    """Seeded clips (noise + per-clip offset so that the pooled features differ) and the weights of the scalar loss
    sum(logits * w) whose gradients are recorded."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 3, T, HW, HW, generator=g) + 1.5 * torch.randn(B, 3, 1, 1, 1, generator=g)
    w = torch.randn(B, num_class, generator=g)
    return x, w


def import_reference_classifier():
    clash = lambda k: k in ("model", "backbone") or k.startswith("model.") or k.startswith("backbone.")
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if clash(k)}
    sys.path.insert(0, REF)
    try:
        mod = importlib.import_module("model.classifier")
        assert mod.__file__.startswith(REF), mod.__file__
    finally:
        sys.path.remove(REF)
        for k in list(sys.modules):
            if clash(k):
                sys.modules.pop(k)
        sys.modules.update(saved)
    return mod


def main():
    import classifier_oracle as O
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    LC = import_reference_classifier().LinearClassifier
    out = {"flags_json": np.array(json.dumps(ref_flags(os.path.join(REF, "eval", "main_classifier.py")), sort_keys=True))}
    keys = {}
    for net in ("s3d", "s3dg", "r50"):
        for cfg, kw in CONFIGS.items():
            m = LC(num_class=101, network=net, dropout=0.9, **kw)
            keys["%s/%s" % (net, cfg)] = {k: list(v.shape) for k, v in m.state_dict().items()}
    out["keys_json"] = np.array(json.dumps(keys, sort_keys=True))
    x, w = inputs(**SHAPE)
    for case, cfg in (("eval", "ft"), ("train", "last")):
        kw = CONFIGS[cfg]
        m = LC(num_class=SHAPE["num_class"], network="s3d", dropout=0.9, **kw).double()
        sd = O.classifier_state("s3d", SHAPE["num_class"], kw["use_dropout"], kw["use_final_bn"], seed=0)
        res = m.load_state_dict({k: v.double() if v.is_floating_point() else v for k, v in sd.items()}, strict=False)
        assert not res.unexpected_keys and all(".block" in k for k in res.missing_keys), res
        m.train() if case == "train" else m.eval()
        logit, feat = m(x.double())
        (logit * w.double()).sum().backward()
        named = dict(m.named_parameters())
        out[case + "/logit"] = logit.detach().numpy()
        out[case + "/feat3d"] = feat.detach().numpy()
        fc = "final_fc.1." if kw["use_dropout"] else "final_fc.0."
        for k in GRAD_KEYS + [fc + "weight", fc + "bias"] + (["final_bn.weight", "final_bn.bias"] if kw["use_final_bn"] else []):
            out["%s/grad/%s" % (case, k)] = compact(named[k].grad.numpy(), 4096)[0]
        if case == "train":
            msd = m.state_dict()
            for k in ("final_bn.running_mean", "final_bn.running_var", "backbone.Conv_2c.bn1.running_var"):
                out["train/state/" + k] = msd[k].numpy()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, sorted(out))


if __name__ == "__main__":
    main()
