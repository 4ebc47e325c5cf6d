"""The q encoder of oracle/coclr_oracle.py with its ReLU and max-pool decisions passed in -- TEST INFRASTRUCTURE ONLY.

A ReLU decides per element which side of zero a value falls on, a max-pool which element of a window wins.  Where two
evaluations of the network disagree on such a decision (a pre-ReLU value within rounding of zero, two elements of a
window that tie), they compute different functions, and their gradients differ by far more than arithmetic error.  With
the decisions fixed, the encoder is one smooth function of its parameters, and autograd gives its exact gradient; the
engine's gradients can then be compared against float64 tensor by tensor at the level of its arithmetic.

Every ReLU is `torch.where(mask, z, 0)` and every max-pool gathers its window at a given tap.  Decisions are keyed by
the engine's names (coclr_b200.engine.Graph, relative to its backbone prefix):
  masks: BatchNorm member name -> bool [B, C, T, H, W] (a residual unit is keyed by its bn3: relu(bn3(y) + r)),
         HEAD_RELU -> bool [B, fs, 1, 1, 1] (the projection head's bias + ReLU);
  taps:  PoolSpec.name -> integer [B, C, To, Ho, Wo], tap (t * kh + h) * kw + w within the window.
A `Decisions()` built without masks takes every decision from the value it is evaluated at (z > 0, the arg-max
F.max_pool3d picks) and records it: evaluated that way the restatement is the oracle, bit for bit
(tests/test_grad_pinned_cpu.py).

Built from the oracle's pieces: F.conv3d, F.batch_norm in train mode with no running statistics (the state dict is
not changed), coclr_oracle.self_gating.  Only the training-mode forward is restated: that is the one with a backward.
"""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle.coclr_oracle import BN_EPS, BN_MOMENTUM, INCEPTION, R50_LAYERS, self_gating  # noqa: E402

HEAD_RELU = "2"   # the ReLU after the projection head's first conv (encoder child "2"), model/pretrain.py:49-54


def taps_from_indices(ind, in_dims, k, s, p):
    """F.max_pool3d(..., return_indices=True) indices (flat over the unpadded T*H*W) -> taps within each window."""
    T, H, W = in_dims
    To, Ho, Wo = ind.shape[2:]
    dev = ind.device
    t0 = (torch.arange(To, device=dev) * s[0] - p[0]).view(-1, 1, 1)
    h0 = (torch.arange(Ho, device=dev) * s[1] - p[1]).view(1, -1, 1)
    w0 = (torch.arange(Wo, device=dev) * s[2] - p[2]).view(1, 1, -1)
    dt, dh, dw = ind // (H * W) - t0, (ind // W) % H - h0, ind % W - w0
    return (dt * k[1] + dh) * k[2] + dw


def pool_at(x, taps, k, s, p):
    """Max-pool output with the winners given: out[b, c, o] = x_padded[b, c, window(o) at taps[b, c, o]].
    The padding is -inf, as in nn.MaxPool3d, so a tap that points into it shows up as -inf."""
    B, C = x.shape[:2]
    xp = F.pad(x, (p[2], p[2], p[1], p[1], p[0], p[0]), value=float("-inf"))
    Hp, Wp = xp.shape[3], xp.shape[4]
    To, Ho, Wo = taps.shape[2:]
    dev = x.device
    tp = taps.long()
    t = torch.arange(To, device=dev).view(-1, 1, 1) * s[0] + tp // (k[1] * k[2])
    h = torch.arange(Ho, device=dev).view(1, -1, 1) * s[1] + (tp // k[2]) % k[1]
    w = torch.arange(Wo, device=dev).view(1, 1, -1) * s[2] + tp % k[2]
    flat = ((t * Hp + h) * Wp + w).view(B, C, -1)
    return xp.reshape(B, C, -1).gather(2, flat).view(B, C, To, Ho, Wo)


class Decisions:
    """ReLU masks and max-pool taps by site name (module docstring).  Without `masks` / `taps` every decision is taken
    from the value at hand and recorded.  Subclasses may override `act` to see every BatchNorm member's conv output
    ('y'), its activation after the ReLU and before any gating ('a') and its gated output ('gated')."""

    def __init__(self, masks=None, taps=None):
        self.record = masks is None
        assert (taps is None) == self.record
        self.masks = {} if masks is None else masks
        self.taps = {} if taps is None else taps
        self.residual = set()   # mask sites of the form relu(bn(y) + r)
        self.used = set()

    def relu(self, name, z, residual=False):
        if residual:
            self.residual.add(name)
        if self.record:
            assert name not in self.masks, name
            self.masks[name] = (z > 0).detach()
        self.used.add(name)
        return torch.where(self.masks[name], z, 0.0)

    def pool(self, name, x, k, s, p):
        if self.record:
            assert name not in self.taps, name
            _, ind = F.max_pool3d(x.detach(), k, s, p, return_indices=True)
            self.taps[name] = taps_from_indices(ind, x.shape[2:], k, s, p)
        self.used.add(name)
        return pool_at(x, self.taps[name], k, s, p)

    def act(self, kind, name, t):
        pass


def _bn(sd, key, y):
    return F.batch_norm(y, None, None, sd[key + ".weight"], sd[key + ".bias"], True, BN_MOMENTUM, BN_EPS)


def _bn_relu(sd, bb, name, y, dec):
    dec.act("y", name, y)
    a = dec.relu(name, _bn(sd, bb + name, y))
    dec.act("a", name, a)
    return a


# ---------------------------------------------------------------------------------------------
# S3D / S3D-G; coclr_oracle.s3d
# ---------------------------------------------------------------------------------------------
def basic_conv(sd, bb, name, x, dec):
    return _bn_relu(sd, bb, name + ".bn", F.conv3d(x, sd[bb + name + ".conv.weight"]), dec)


def st_conv(sd, bb, name, x, k, stride, t_stride, pad, dec):
    x = F.conv3d(x, sd[bb + name + ".conv1.weight"], stride=(1, stride, stride), padding=(0, pad, pad))
    x = _bn_relu(sd, bb, name + ".bn1", x, dec)
    x = F.conv3d(x, sd[bb + name + ".conv2.weight"], stride=(t_stride, 1, 1), padding=(pad, 0, 0))
    return _bn_relu(sd, bb, name + ".bn2", x, dec)


def sep_inception(sd, bb, name, x, dec):
    x0 = basic_conv(sd, bb, name + ".branch0.0", x, dec)
    x1 = basic_conv(sd, bb, name + ".branch1.0", x, dec)
    x1 = st_conv(sd, bb, name + ".branch1.1", x1, 3, 1, 1, 1, dec)
    x2 = basic_conv(sd, bb, name + ".branch2.0", x, dec)
    x2 = st_conv(sd, bb, name + ".branch2.1", x2, 3, 1, 1, 1, dec)
    x3 = dec.pool(name + ".branch3.0", x, (3, 3, 3), (1, 1, 1), (1, 1, 1))
    x3 = basic_conv(sd, bb, name + ".branch3.1", x3, dec)
    xs = [x0, x1, x2, x3]
    if (bb + name + ".gating_b0.fc.weight") in sd:
        members = [".branch0.0.bn", ".branch1.1.bn2", ".branch2.1.bn2", ".branch3.1.bn"]
        for i in range(4):
            xs[i] = self_gating(sd, "%s%s.gating_b%d" % (bb, name, i), xs[i])
            dec.act("gated", name + members[i], xs[i])
    return torch.cat(xs, 1)


def s3d(sd, bb, x, dec):
    x = st_conv(sd, bb, "Conv_1a", x, 7, 2, 2, 3, dec)
    x = dec.pool("MaxPool_2a", x, (1, 3, 3), (1, 2, 2), (0, 1, 1))
    x = basic_conv(sd, bb, "Conv_2b", x, dec)
    x = st_conv(sd, bb, "Conv_2c", x, 3, 1, 1, 1, dec)
    x = dec.pool("MaxPool_3a", x, (1, 3, 3), (1, 2, 2), (0, 1, 1))
    for name, _, _ in INCEPTION[:2]:
        x = sep_inception(sd, bb, name, x, dec)
    x = dec.pool("MaxPool_4a", x, (3, 3, 3), (2, 2, 2), (1, 1, 1))
    for name, _, _ in INCEPTION[2:7]:
        x = sep_inception(sd, bb, name, x, dec)
    x = dec.pool("MaxPool_5a", x, (2, 2, 2), (2, 2, 2), (0, 0, 0))
    for name, _, _ in INCEPTION[7:]:
        x = sep_inception(sd, bb, name, x, dec)
    return x


# ---------------------------------------------------------------------------------------------
# ResNet2d3d-50; coclr_oracle.r2d3d50
# ---------------------------------------------------------------------------------------------
def bottleneck(sd, bb, name, x, stride, is3d, dec):
    p = bb + name
    out = F.conv3d(x, sd[p + ".conv1.weight"], padding=(1, 0, 0) if is3d else 0)
    out = _bn_relu(sd, bb, name + ".bn1", out, dec)
    out = F.conv3d(out, sd[p + ".conv2.weight"], stride=(1, stride, stride), padding=(0, 1, 1))
    out = _bn_relu(sd, bb, name + ".bn2", out, dec)
    y3 = F.conv3d(out, sd[p + ".conv3.weight"])
    dec.act("y", name + ".bn3", y3)
    out = _bn(sd, p + ".bn3", y3)
    if (p + ".downsample.0.weight") in sd:
        yd = F.conv3d(x, sd[p + ".downsample.0.weight"], stride=(1, stride, stride))
        dec.act("y", name + ".downsample.1", yd)
        x = _bn(sd, p + ".downsample.1", yd)
        dec.act("a", name + ".downsample.1", x)
    a = dec.relu(name + ".bn3", out + x, residual=True)
    dec.act("a", name + ".bn3", a)
    return a


def r2d3d50(sd, bb, x, dec):
    x = F.conv3d(x, sd[bb + "conv1.weight"], stride=(2, 2, 2), padding=(2, 3, 3))
    x = _bn_relu(sd, bb, "bn1", x, dec)
    x = dec.pool("maxpool", x, (1, 3, 3), (1, 2, 2), (0, 1, 1))
    for name, _, blocks, stride, is3d in R50_LAYERS:
        for i in range(blocks):
            x = bottleneck(sd, bb, "%s.%d" % (name, i), x, stride if i == 0 else 1, is3d, dec)
    return x


# ---------------------------------------------------------------------------------------------
# the encoder forms the engine runs
# ---------------------------------------------------------------------------------------------
def backbone(sd, bb, x, dec):
    """The backbone under state prefix `bb` (e.g. 'encoder_q.0.', 'backbone.'), recognised from the state keys."""
    return (r2d3d50 if (bb + "layer1.0.conv1.weight") in sd else s3d)(sd, bb, x, dec)


def encoder(sd, pre, x, dec):
    """coclr_oracle.encoder: backbone -> average pool -> conv + bias -> ReLU -> conv + bias; [B, dim, 1, 1, 1]."""
    f = F.adaptive_avg_pool3d(backbone(sd, pre + "0.", x, dec), (1, 1, 1))
    dec.act("feat", "", f)
    h = dec.relu(HEAD_RELU, F.conv3d(f, sd[pre + "2.weight"], sd[pre + "2.bias"]))
    return F.conv3d(h, sd[pre + "4.weight"], sd[pre + "4.bias"])


def query(sd, pre, x, dec):
    """The normalised query q [B, dim] of InfoNCE (model/pretrain.py:153-155): what the engine's plan.q holds."""
    return F.normalize(encoder(sd, pre, x, dec), dim=1).view(x.shape[0], -1)


def pooled(sd, bb, x, dec):
    """The average-pooled backbone feature [B, fs] of a `pooled` engine graph (LinearClassifier's backbone)."""
    return F.adaptive_avg_pool3d(backbone(sd, bb, x, dec), (1, 1, 1)).view(x.shape[0], -1)
