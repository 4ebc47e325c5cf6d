"""S3D backbone -- drop-in module surface for the reference's backbone/s3dg.py (S3D, :135-217).

Same constructor, same parameter / buffer names (incl. the `blockN.i` aliases the reference's
state_dict carries) and the same initialisation (conv N(0, 0.01), BN weight 1 / bias 0; s3dg.py:20-22,
51-56).  The modules below only *hold* parameters: the arithmetic of `forward` runs on the sm_90a
kernels of coclr_b200 (implicit-GEMM convs with BatchNorm/ReLU folded around them); there is no
PyTorch/cuDNN execution path and no CPU path.
"""
import torch
import torch.nn as nn

from coclr_b200.s3d_spec import s3d_stages, S3D_BLOCKS
from coclr_b200.backbone_base import EngineBackbone, holder_forward as _holder_forward


class BasicConv3d(nn.Module):
    """1x1x1 (or general) conv + BatchNorm3d + ReLU parameter group (reference s3dg.py:8-28)."""

    def __init__(self, in_planes, out_planes, kernel_size, stride, padding=0):
        super().__init__()
        self.conv = nn.Conv3d(in_planes, out_planes, kernel_size=kernel_size, stride=stride, padding=padding,
                              bias=False)
        self.bn = nn.BatchNorm3d(out_planes)
        self.relu = nn.ReLU(inplace=True)
        nn.init.normal_(self.conv.weight, mean=0, std=0.01)
        nn.init.ones_(self.bn.weight)
        nn.init.zeros_(self.bn.bias)

    forward = _holder_forward


class STConv3d(nn.Module):
    """Separable (1,k,k) then (k,1,1) conv, each with BN + ReLU (reference s3dg.py:30-65)."""

    def __init__(self, in_planes, out_planes, kernel_size, stride, padding=0):
        super().__init__()
        if isinstance(stride, tuple):
            t_stride, stride = stride[0], stride[-1]
        else:
            t_stride = stride
        self.conv1 = nn.Conv3d(in_planes, out_planes, (1, kernel_size, kernel_size), (1, stride, stride),
                               (0, padding, padding), bias=False)
        self.conv2 = nn.Conv3d(out_planes, out_planes, (kernel_size, 1, 1), (t_stride, 1, 1), (padding, 0, 0),
                               bias=False)
        self.bn1 = nn.BatchNorm3d(out_planes)
        self.bn2 = nn.BatchNorm3d(out_planes)
        self.relu = nn.ReLU(inplace=True)
        for conv in (self.conv1, self.conv2):
            nn.init.normal_(conv.weight, mean=0, std=0.01)
        for bn in (self.bn1, self.bn2):
            nn.init.ones_(bn.weight)
            nn.init.zeros_(bn.bias)

    forward = _holder_forward


class SelfGating(nn.Module):
    """S3D-G feature gating: x * sigmoid(fc(mean_thw(x))) (reference s3dg.py:68-78); nn.Linear's default init."""

    def __init__(self, input_dim):
        super().__init__()
        self.fc = nn.Linear(input_dim, input_dim)

    forward = _holder_forward


class SepInception(nn.Module):
    """Four-branch separable Inception block (reference s3dg.py:81-132); gating=True adds one SelfGating per branch
    output (:107-112,125-129)."""

    def __init__(self, in_planes, out_planes, gating=False):
        super().__init__()
        assert isinstance(out_planes, list) and len(out_planes) == 6
        o0, o1a, o1b, o2a, o2b, o3b = out_planes
        self.branch0 = nn.Sequential(BasicConv3d(in_planes, o0, 1, 1))
        self.branch1 = nn.Sequential(BasicConv3d(in_planes, o1a, 1, 1), STConv3d(o1a, o1b, 3, 1, 1))
        self.branch2 = nn.Sequential(BasicConv3d(in_planes, o2a, 1, 1), STConv3d(o2a, o2b, 3, 1, 1))
        self.branch3 = nn.Sequential(nn.MaxPool3d((3, 3, 3), 1, 1), BasicConv3d(in_planes, o3b, 1, 1))
        self.out_channels = o0 + o1b + o2b + o3b
        self.gating = gating
        if gating:
            self.gating_b0 = SelfGating(o0)
            self.gating_b1 = SelfGating(o1b)
            self.gating_b2 = SelfGating(o2b)
            self.gating_b3 = SelfGating(o3b)

    forward = _holder_forward


class S3D(EngineBackbone):
    """x: [B, C, T, H, W] -> [B, 1024, T/8, H/32, W/32] (reference s3dg.py:135-217)."""

    _probe = "Conv_1a.conv1.weight"

    def __init__(self, input_channel=3, gating=False, slow=False, precision="parity"):
        super().__init__()
        if slow:
            raise NotImplementedError("the `slow` variant (no temporal stride in the stem) is outside the accelerated path")
        self.gating, self.slow = gating, slow
        self.input_channel = input_channel
        self.precision = precision
        self._stages = s3d_stages(input_channel, gating=gating)
        for stg in self._stages:
            kind, name = stg[0], stg[1]
            if kind == "st":
                _, _, cin, cout, k, ss, ts, pad = stg
                mod = STConv3d(cin, cout, k, (ts, ss, ss) if ts != ss else ss, pad)
            elif kind == "basic":
                mod = BasicConv3d(stg[2], stg[3], 1, 1)
            elif kind == "pool":
                mod = nn.MaxPool3d(kernel_size=stg[2], stride=stg[3], padding=stg[4])
            else:
                mod = SepInception(stg[2], list(stg[3]), gating=gating)
            setattr(self, name, mod)
            if kind == "st" and name == "Conv_1a":
                self.block1 = nn.Sequential(mod)
        for blk, members in S3D_BLOCKS.items():
            if blk != "block1":
                setattr(self, blk, nn.Sequential(*[getattr(self, m) for m in members]))
        self._init_engine_state()
