"""TEST INFRASTRUCTURE -- CPU restatement of the renderers (SURVEY.md section 8a rows a18-a20).

Follows nerfstudio/model_components/renderers.py: RGBRenderer :53-118, AccumulationRenderer :171-197,
DepthRenderer :215-261, SemanticRenderer :284-295.  Dense branch: rgb [R,S,3], weights [R,S,1], starts/ends [R,S,1].  Packed branch
(``ray_indices`` + ``num_rays``, :74-79, :192-194, :249-257): rgb [N,3], weights / starts / ends [N,1], nerfacc.accumulate_along_rays
restated as a per-ray ``index_add`` (differentiable like nerfacc's).
"""
from typing import Optional, Union

import torch


def render_rgb(rgb, weights, background: Union[str, torch.Tensor], training: bool = False, rand_bg: Optional[torch.Tensor] = None):
    """renderers.py:53-118.  background: tensor[3] | 'last_sample' | 'random' (then ``rand_bg`` [R,3] supplies the draw)."""
    comp = torch.sum(weights * rgb, dim=-2)
    acc = torch.sum(weights, dim=-2)
    if isinstance(background, str):
        if background == "last_sample":
            bg = rgb[..., -1, :]
        elif background == "random":
            bg = rand_bg
        else:
            raise ValueError(background)
    else:
        bg = background
    comp = comp + bg * (1.0 - acc)
    if not training:
        comp = torch.clamp(comp, min=0.0, max=1.0)
    return comp


def render_accumulation(weights):
    """renderers.py:171-197."""
    return torch.sum(weights, dim=-2)


def render_depth(weights, starts, ends, method: str = "expected"):
    """renderers.py:215-261.  NOTE the *batch-global* clip to [steps.min(), steps.max()] in 'expected' (:257)."""
    steps = (starts + ends) / 2
    if method == "median":
        cum = torch.cumsum(weights[..., 0], dim=-1)
        split = torch.ones((*weights.shape[:-2], 1), dtype=weights.dtype) * 0.5
        idx = torch.searchsorted(cum, split, side="left")
        idx = torch.clamp(idx, 0, steps.shape[-2] - 1)
        return torch.gather(steps[..., 0], dim=-1, index=idx)
    if method == "expected":
        eps = 1e-10
        depth = torch.sum(weights * steps, dim=-2) / (torch.sum(weights, -2) + eps)
        return torch.clip(depth, steps.min(), steps.max())
    raise NotImplementedError(method)


def render_semantics(semantics, weights):
    """renderers.py:284-295 (used as the normal renderer, base_surface_model.py:216)."""
    return torch.sum(weights * semantics, dim=-2)


def accumulate_along_rays(weights, ray_indices, values, num_rays):
    """nerfacc.accumulate_along_rays as the packed branch calls it: [num_rays, C] per-ray sums of weights [N,1] * values [N,C]
    (values None: of the weights).  Rays without a sample get 0."""
    src = weights if values is None else weights * values
    return torch.zeros(num_rays, src.shape[-1], dtype=src.dtype).index_add(0, ray_indices, src)


def render_rgb_packed(rgb, weights, ray_indices, num_rays, background: torch.Tensor, training: bool = False):
    """renderers.py:74-79 + :84-90 (background tensor [3] or [R,3]; 'last_sample' raises NotImplementedError there)."""
    comp = accumulate_along_rays(weights, ray_indices, rgb, num_rays)
    acc = accumulate_along_rays(weights, ray_indices, None, num_rays)
    comp = comp + background * (1.0 - acc)
    return comp if training else torch.clamp(comp, min=0.0, max=1.0)


def render_depth_packed(weights, starts, ends, ray_indices, num_rays):
    """renderers.py:246-257: expected depth of packed samples, clipped to the batch's [steps.min(), steps.max()]."""
    steps = (starts + ends) / 2
    depth = accumulate_along_rays(weights, ray_indices, steps, num_rays) / (accumulate_along_rays(weights, ray_indices, None, num_rays) + 1e-10)
    return torch.clip(depth, steps.min(), steps.max())
