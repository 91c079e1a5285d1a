"""Drop-ins for the nerfacc 0.3.5 functions neus-acc composites its packed samples with (models/neus_acc.py:102-120):
``render_weight_from_alpha`` and ``accumulate_along_rays``, same signatures, differentiable (autograd_ops.PackedWeightsFn /
PackedAccumulateFn).  The kernels (csrc/render.cu, render_backward.cu) walk each ray's samples as one contiguous segment, so
``ray_indices`` must be non-decreasing, which is also what nerfacc's ``pack_info`` assumes.  ``NeuSAccSampler`` hands out ray indices
that carry their segment offsets; for any other tensor the offsets are derived here after one sortedness check.
"""
from typing import Optional

import torch

from . import autograd_ops as _ag

OFFSETS_ATTR = "_packed_offsets"   # [n_rays + 1] int64 segment offsets carried by the sampler's ray_indices


def segment_offsets(ray_indices: torch.Tensor, n_rays: int) -> torch.Tensor:
    """[n_rays + 1] int64 offsets of the segments of `ray_indices` (sorted, values in [0, n_rays)).  Raises ValueError otherwise."""
    off = getattr(ray_indices, OFFSETS_ATTR, None)
    if off is not None and off.numel() == n_rays + 1:
        return off
    ri = ray_indices.reshape(-1).long().contiguous()
    if ri.numel() > 0:
        bad = (ri[1:] < ri[:-1]).any() | (ri[0] < 0) | (ri[-1] >= n_rays)
        if bool(bad):
            raise ValueError("ray_indices must be non-decreasing and lie in [0, n_rays): the packed kernels take each ray's samples as one "
                             "contiguous segment")
    return torch.searchsorted(ri, torch.arange(n_rays + 1, device=ri.device, dtype=torch.int64))


def _n_rays(ray_indices: torch.Tensor, n_rays: Optional[int]) -> int:
    if n_rays is not None:
        return int(n_rays)
    if ray_indices.numel() == 0:
        raise ValueError("n_rays is required when there are no samples")
    return int(ray_indices.max()) + 1


def render_weight_from_alpha(alphas: torch.Tensor, packed_info: Optional[torch.Tensor] = None, ray_indices: Optional[torch.Tensor] = None,
                             n_rays: Optional[int] = None) -> torch.Tensor:
    """weights = alpha * T with T the exclusive product of (1 - alpha) over the samples of each ray.  alphas [N, 1] (or [N]);
    packed_info [n_rays, 2] (start, count) of contiguous segments, or ray_indices [N] (+ n_rays).  Returns alphas' shape."""
    if packed_info is not None:
        pi = packed_info.long()
        starts, counts = pi[:, 0], pi[:, 1]
        if pi.shape[0] > 0 and bool((starts[0] != 0) | (starts[1:] != starts[:-1] + counts[:-1]).any()):
            raise ValueError("packed_info must describe contiguous segments in ray order")
        offsets = torch.cat([starts, (starts[-1:] + counts[-1:]) if pi.shape[0] > 0 else starts.new_zeros(1)]).contiguous()
    elif ray_indices is not None:
        offsets = segment_offsets(ray_indices, _n_rays(ray_indices, n_rays))
    else:
        raise ValueError("one of packed_info or ray_indices is required")
    w = _ag.PackedWeightsFn.apply(alphas.reshape(-1), offsets)
    return w.view(alphas.shape)


def accumulate_along_rays(weights: torch.Tensor, ray_indices: torch.Tensor, values: Optional[torch.Tensor] = None,
                          n_rays: Optional[int] = None) -> torch.Tensor:
    """[n_rays, C] per-ray sums of weights * values (values [N, C]), or of the weights alone ([n_rays, 1]).  weights [N, 1] (or [N])."""
    n = _n_rays(ray_indices, n_rays)
    offsets = segment_offsets(ray_indices, n)
    if values is not None and (values.dim() != 2 or values.shape[0] != weights.shape[0]):
        raise ValueError(f"values must be [N, C] with N = {weights.shape[0]}, got {tuple(values.shape)}")
    ri = ray_indices.reshape(-1).long().contiguous()
    return _ag.PackedAccumulateFn.apply(weights.reshape(-1), values, offsets, ri)
