"""Float64 restatement of nn.DataParallel(LinearClassifier) -- TEST INFRASTRUCTURE ONLY, built on
tests/tools/classifier_oracle.py.  tests/test_sgd_replicas_cpu.py pins it against the unmodified reference module run
under the same rules (tests/golden/replicas.npz, written by tests/golden/make_golden_replicas.py).

DataParallel scatters the batch as torch.chunk(x, R) (fewer chunks than R when the batch is short), runs one replica
per chunk and concatenates the outputs.  Replica 0 shares the module's parameters and buffers; every other replica
shares the parameters (its gradients add up in theirs) but updates private copies of the buffers, which are lost.
"""
import torch

from classifier_oracle import classifier_forward
from oracle.coclr_oracle import _bn_scratch


def dataparallel_forward(sd, x, replicas, backbone_training, bn_training=False, use_l2_norm=False, dropout_mask=None,
                         p=0.5):
    """(logit, feat3d) of nn.DataParallel(LinearClassifier) with `replicas` devices; sd's buffers end as chunk 0 left
    them.  dropout_mask [B, fs] is split like the batch."""
    xs = torch.chunk(x, replicas, dim=0)
    masks = torch.chunk(dropout_mask, replicas, dim=0) if dropout_mask is not None else [None] * len(xs)
    logits, feats = [], []
    for r, (xr, mr) in enumerate(zip(xs, masks)):
        sdr = sd if r == 0 else _bn_scratch(sd, "")
        lg, f = classifier_forward(sdr, xr, backbone_training, bn_training, use_l2_norm, mr, p)
        logits.append(lg)
        feats.append(f)
    return torch.cat(logits), torch.cat(feats)
