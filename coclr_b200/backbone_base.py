"""Shared plumbing of the backbone modules (backbone/s3dg.py, backbone/resnet_2d3d.py): they hold parameters with the
reference's names; the arithmetic of a bare-backbone forward runs on the engine."""
import torch
import torch.nn as nn

from .engine import Graph, bind_engine


def holder_forward(self, *a, **k):
    raise RuntimeError("%s is a parameter holder; run the enclosing backbone / encoder module (CUDA only)"
                       % type(self).__name__)


class EngineBackbone(nn.Module):
    """Subclasses set `_stages` (engine stage table), `input_channel`, `precision` and `_probe` (name of one conv weight,
    used to notice that the parameters were moved / re-bound)."""

    _probe = None

    def _init_engine_state(self):
        self._engine = None

    def _get_engine(self):
        self._engine = bind_engine(self._engine, self.get_parameter(self._probe), self,
                                   lambda: Graph(self._stages, self.input_channel), self.precision)
        return self._engine

    def forward(self, x):
        """x: [B, C, T, H, W] -> backbone feature map [B, C', T', H', W'] (inference-style use of the bare backbone;
        training goes through the MoCo encoder, which owns forward + backward)."""
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise RuntimeError("the bare backbone module is forward-only; wrap it in coclr_b200's MoCo encoder "
                               "(model.pretrain) for training, or call under torch.no_grad()")
        eng = self._get_engine()
        plan = eng.forward(x.contiguous(), training=self.training, with_backward=False)
        return eng.backbone_output_ncdhw(plan)
