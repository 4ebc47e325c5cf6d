"""Writes tests/golden/replicas.npz from the UNMODIFIED reference ($COCLR_REFERENCE): its S3D LinearClassifier
(model/classifier.py) in float64 under nn.DataParallel's rules, on the states of tests/tools/classifier_oracle.py
(classifier_state) and seeded clips:

  * scatter by torch.chunk(x, R); replica 0 is the module itself; replicas r > 0 run the module too, and the buffer
    updates they make are undone after the step (their running-statistics updates are lost);
  * gather by concatenation, nn.CrossEntropyLoss on the gathered logits, one backward (gradients sum over replicas).

Cases: `ft` with the backbone in train mode (dropout off: its mask is random) at R = 2 (B = 4) and R = 3 (B = 5: chunks
2, 2, 1), and `last` (eval backbone, train-mode final BN) at R = 2 (B = 5: chunks 3, 2).  Recorded: logits, loss, the
gradients of make_golden_classifier.GRAD_KEYS and of the head, and running statistics after the step.

Run in the build container only:  COCLR_REFERENCE=<checkout> python tests/golden/make_golden_replicas.py
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
from make_golden import compact  # noqa: E402
from make_golden_classifier import CONFIGS, GRAD_KEYS, import_reference_classifier, inputs  # noqa: E402

OUT = os.path.join(HERE, "replicas.npz")
CASES = {"ft_r2": ("ft", 2, 4), "ft_r3": ("ft", 3, 5), "last_r2": ("last", 2, 5)}
SHAPE = dict(T=8, HW=64, num_class=51)
STATE_KEYS = ["backbone.Conv_1a.bn1.running_mean", "backbone.Conv_2c.bn1.running_var",
              "backbone.Mixed_5c.branch0.0.bn.running_mean", "backbone.Conv_2b.bn.num_batches_tracked"]
HEAD_STATE_KEYS = ["final_bn.running_mean", "final_bn.running_var", "final_bn.num_batches_tracked"]


def case_inputs(B, num_class, seed=4321):
    x, _ = inputs(B, SHAPE["T"], SHAPE["HW"], num_class, seed=seed)
    y = torch.randint(0, num_class, (B,), generator=torch.Generator().manual_seed(seed + 1))
    return x, y


def grad_keys(cfg):
    kw = CONFIGS[cfg]
    fc = "final_fc.1." if kw["use_dropout"] else "final_fc.0."
    keys = [fc + "weight", fc + "bias"] + (["final_bn.weight", "final_bn.bias"] if kw["use_final_bn"] else [])
    return (GRAD_KEYS if cfg == "ft" else []) + keys


def state_keys(cfg):
    return STATE_KEYS + (HEAD_STATE_KEYS if cfg == "last" else [])


def main():
    import classifier_oracle as O
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    LC = import_reference_classifier().LinearClassifier
    out = {}
    for name, (cfg, R, B) in CASES.items():
        kw = CONFIGS[cfg]
        m = LC(num_class=SHAPE["num_class"], network="s3d", dropout=0.9, **kw).double()
        sd = O.classifier_state("s3d", SHAPE["num_class"], kw["use_dropout"], kw["use_final_bn"], seed=0)
        res = m.load_state_dict({k: v.double() if v.is_floating_point() else v for k, v in sd.items()}, strict=False)
        assert not res.unexpected_keys and all(".block" in k for k in res.missing_keys), res
        if cfg == "last":
            m.eval()
            m.final_bn.train()
            for p in m.backbone.parameters():
                p.requires_grad = False
        else:
            m.train()
            m.final_fc[0].eval()
        x, y = case_inputs(B, SHAPE["num_class"])
        params = dict(m.named_parameters())
        logits = []
        for r, xr in enumerate(torch.chunk(x.double(), R, dim=0)):
            lg, _ = m(xr)
            if r == 0:
                kept = {k: v.clone() for k, v in m.named_buffers()}
            logits.append(lg)
        logit = torch.cat(logits)
        loss = F.cross_entropy(logit, y)
        loss.backward()
        # the buffer updates of replicas r > 0 are lost: the buffers end as chunk 0 left them (train-mode running
        # statistics are only written, never read, so restoring them after the step equals private copies; it waits
        # for backward, which checks that the tensors it saved were not modified in place)
        with torch.no_grad():
            for k, v in m.named_buffers():
                v.copy_(kept[k])
        out[name + "/logit"] = logit.detach().numpy()
        out[name + "/loss"] = np.array(float(loss.detach()))
        for k in grad_keys(cfg):
            out["%s/grad/%s" % (name, k)] = compact(params[k].grad.numpy(), 4096)[0]
        msd = m.state_dict()
        for k in state_keys(cfg):
            out["%s/state/%s" % (name, k)] = msd[k].numpy()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, sorted(out))


if __name__ == "__main__":
    main()
