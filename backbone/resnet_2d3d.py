"""ResNet2d3d-50 -- drop-in module surface for the reference's backbone/resnet_2d3d.py (r2d3d50, :204-208).

Same constructors, parameter / buffer names (conv1, bn1, layerN.i.{conv1..3, bn1..3, downsample.0/1}) and the same
initialisation (kaiming_normal_(fan_out) convs, BN weight 1 / bias 0; :147-153).  The modules only *hold* parameters:
`forward` runs on the sm_90a kernels of coclr_b200 (implicit-GEMM convs, BatchNorm + residual add + ReLU fused into
one pass); there is no PyTorch/cuDNN execution path and no CPU path.
"""
import torch.nn as nn

from coclr_b200.r50_spec import r50_stages, R50_LAYERS
from coclr_b200.backbone_base import EngineBackbone, holder_forward

__all__ = ['ResNet2d3d', 'r2d3d50']


class _Bottleneck(nn.Module):
    expansion = 4
    _conv1_kernel, _conv1_pad = (1, 1, 1), (0, 0, 0)

    def __init__(self, inplanes, planes, stride=1, downsample=None, use_final_relu=True):
        super().__init__()
        self.use_final_relu = use_final_relu
        self.conv1 = nn.Conv3d(inplanes, planes, kernel_size=self._conv1_kernel, padding=self._conv1_pad, bias=False)
        self.bn1 = nn.BatchNorm3d(planes)
        self.conv2 = nn.Conv3d(planes, planes, kernel_size=(1, 3, 3), stride=(1, stride, stride), padding=(0, 1, 1),
                               bias=False)
        self.bn2 = nn.BatchNorm3d(planes)
        self.conv3 = nn.Conv3d(planes, planes * 4, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm3d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride

    forward = holder_forward


class Bottleneck2d(_Bottleneck):
    """1x1x1 -> (1,3,3) -> 1x1x1 residual block (reference resnet_2d3d.py:89-131)."""


class Bottleneck3d(_Bottleneck):
    """(3,1,1) -> (1,3,3) -> 1x1x1 residual block (reference resnet_2d3d.py:46-86)."""
    _conv1_kernel, _conv1_pad = (3, 1, 1), (1, 0, 0)


class ResNet2d3d(EngineBackbone):
    """r2d3d50 layout only (the table in coclr_b200/r50_spec.py); `block` / `layers` are accepted for signature
    compatibility with the reference (resnet_2d3d.py:134) and must describe that layout."""

    _probe = "conv1.weight"

    def __init__(self, block=None, layers=(3, 4, 6, 3), input_channel=3, precision="parity"):
        super().__init__()
        if list(layers) != [3, 4, 6, 3]:
            raise NotImplementedError("only the r2d3d50 layout [3, 4, 6, 3] is on the accelerated path")
        want = [Bottleneck2d, Bottleneck2d, Bottleneck3d, Bottleneck3d]
        if block is not None and list(block if isinstance(block, list) else [block] * 4) != want:
            raise NotImplementedError("only [Bottleneck2d, Bottleneck2d, Bottleneck3d, Bottleneck3d] is on the accelerated path")
        self.input_channel, self.precision = input_channel, precision
        self._stages = r50_stages(input_channel)
        self.inplanes = 64
        self.conv1 = nn.Conv3d(input_channel, 64, kernel_size=(5, 7, 7), stride=(2, 2, 2), padding=(2, 3, 3), bias=False)
        self.bn1 = nn.BatchNorm3d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool3d(kernel_size=(1, 3, 3), stride=(1, 2, 2), padding=(0, 1, 1))
        for name, planes, blocks, stride, is3d in R50_LAYERS:
            cls = Bottleneck3d if is3d else Bottleneck2d
            mods = []
            for i in range(blocks):
                ds = None
                if i == 0:
                    ds = nn.Sequential(nn.Conv3d(self.inplanes, planes * 4, kernel_size=1, stride=(1, stride, stride), bias=False),
                                       nn.BatchNorm3d(planes * 4))
                last = name == "layer4" and i == blocks - 1          # reference :181-185 (the final F.relu follows anyway)
                mods.append(cls(self.inplanes, planes, stride if i == 0 else 1, ds, use_final_relu=not last))
                self.inplanes = planes * 4
            setattr(self, name, nn.Sequential(*mods))
        for m in self.modules():                                       # reference :147-153
            if isinstance(m, nn.Conv3d):
                m.weight = nn.init.kaiming_normal_(m.weight, mode='fan_out')
            elif isinstance(m, nn.BatchNorm3d):
                m.weight.data.fill_(1)
                m.bias.data.zero_()
        self._init_engine_state()


def r2d3d50(**kwargs):
    """ResNet-50 with 2D bottlenecks in layer1-2 and 3D bottlenecks in layer3-4 (reference resnet_2d3d.py:204-208)."""
    return ResNet2d3d([Bottleneck2d, Bottleneck2d, Bottleneck3d, Bottleneck3d], [3, 4, 6, 3], **kwargs)
