"""``SceneContraction`` (nerfstudio/field_components/spatial_distortions.py:31-73), mip-NeRF-360 eq. 10.

A plain autograd-friendly module: SDFField reads only ``.order`` from it on the kernel path (the contraction is fused into
the field kernels, csrc/field_simt.cu / field_tc.cu) and calls it on the differentiable training path.
"""
from typing import Optional, Union

import torch
from torch import nn

from . import _lib


class SpatialDistortion(nn.Module):
    def forward(self, positions):  # pragma: no cover - interface
        raise NotImplementedError


class SceneContraction(SpatialDistortion):
    def __init__(self, order: Optional[Union[float, int]] = None) -> None:
        super().__init__()
        self.order = order

    def forward(self, positions):
        mag = torch.linalg.norm(positions, ord=self.order, dim=-1, keepdim=True)
        outside = mag >= 1
        safe = torch.where(outside, mag, torch.ones_like(mag))  # keeps the unused branch finite for autograd
        return torch.where(outside, (2 - 1 / safe) * (positions / safe), positions)


def contraction_code(sd) -> int:
    """The kernels' contraction code of a spatial distortion (None = no contraction): CONTRACT_NONE / _LINF / _L2."""
    if sd is None:
        return _lib.CONTRACT_NONE
    order = getattr(sd, "order", None)
    if order is None:
        return _lib.CONTRACT_L2
    if order == float("inf"):
        return _lib.CONTRACT_LINF
    raise NotImplementedError(f"SceneContraction order {order!r} is not supported")
