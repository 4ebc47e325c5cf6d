"""Float64 restatement of the reference's LinearClassifier (model/classifier.py) in stock PyTorch ops -- TEST
INFRASTRUCTURE ONLY, like oracle/coclr_oracle.py, whose backbone restatements (s3d, r2d3d50) and BatchNorm it reuses.
Only tests/ and tests/tools/bench_classifier.py import it; tests/test_classifier_cpu.py pins it against what the
unmodified reference module computed (tests/golden/classifier.npz, written by tests/golden/make_golden_classifier.py).

State is a flat dict {state_dict key: tensor} with the reference's key names: 'backbone.*', 'final_bn.*',
'final_fc.0.*' / 'final_fc.1.*'.
"""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle.coclr_oracle import _bn, r2d3d50, r50_shapes, s3d, s3d_shapes, synth_state  # noqa: E402
# ---------------------------------------------------------------------------------------------
# LinearClassifier (fine-tuning / linear probe); model/classifier.py
# ---------------------------------------------------------------------------------------------
def classifier_forward(sd, x, backbone_training, bn_training=False, use_l2_norm=False, dropout_mask=None, p=0.5):
    """LinearClassifier.forward; model/classifier.py:47-61.  Returns (logit [B, ncls], feat3d [B, fs]).
    sd keys: 'backbone.*', optional 'final_bn.*' (use_final_bn), 'final_fc.1.*' (use_dropout) or 'final_fc.0.*'.
    Dropout is applied only when `dropout_mask` ([B, fs], 1 = kept) is given: x * mask / (1 - p), i.e. nn.Dropout in
    train mode with that mask."""
    backbone = r2d3d50 if "backbone.layer1.0.conv1.weight" in sd else s3d          # select_backbone.py:4-16
    B = x.shape[0]
    f = backbone(sd, "backbone.", x, backbone_training)                            # :49
    f = F.adaptive_avg_pool3d(f, (1, 1, 1)).view(B, -1)                            # :50-51
    if use_l2_norm:
        f = F.normalize(f, p=2, dim=1)                                             # :53-54
    h = _bn(sd, "final_bn", f, bn_training) if "final_bn.weight" in sd else f      # :56-57
    fc = "final_fc.1." if "final_fc.1.weight" in sd else "final_fc.0."
    if dropout_mask is not None:
        h = h * dropout_mask.to(h.dtype) / (1.0 - p)
    return F.linear(h, sd[fc + "weight"], sd[fc + "bias"]), f                     # :57-61


def classifier_state(network="s3d", num_class=101, use_dropout=True, use_final_bn=False, seed=0):
    """Deterministic classifier state: synth_state's backbone under 'backbone.', fc weights N(0, 1/fs) (larger than the
    reference's N(0, 0.01) init so that the logits are not dominated by the bias), non-trivial final BN."""
    shapes = r50_shapes("backbone.") if network == "r50" else s3d_shapes("backbone.", gating=network == "s3dg")
    sd = synth_state(shapes, seed=seed)
    fs = 2048 if network == "r50" else 1024
    g = torch.Generator().manual_seed(seed + 101)
    if use_final_bn:
        sd["final_bn.weight"] = torch.rand(fs, generator=g) + 0.5
        sd["final_bn.bias"] = torch.randn(fs, generator=g) * 0.1
        sd["final_bn.running_mean"] = torch.randn(fs, generator=g) * 0.01
        sd["final_bn.running_var"] = torch.rand(fs, generator=g) * 0.01 + 0.005
        sd["final_bn.num_batches_tracked"] = torch.tensor(3, dtype=torch.long)
    fc = "final_fc.1." if use_dropout else "final_fc.0."
    sd[fc + "weight"] = torch.randn(num_class, fs, generator=g) / fs ** 0.5
    sd[fc + "bias"] = torch.randn(num_class, generator=g) * 0.05
    return sd
