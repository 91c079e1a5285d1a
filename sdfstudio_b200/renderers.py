"""H100-native drop-ins for ``nerfstudio.model_components.renderers`` (dense branch): RGBRenderer :42-118,
AccumulationRenderer :171-197, DepthRenderer :200-261, SemanticRenderer :284-295.  The per-ray reductions run in
libsdfb200.so (csrc/render.cu, sdfb200_render).  ``render_all`` composites every per-ray output SurfaceModel.get_outputs
asks for (models/base_surface_model.py:300-310) in ONE kernel launch.
"""
from typing import Optional, Union

import torch
from torch import nn

from . import _lib
from . import autograd_ops as _ag
from .rays import bins_of


def _background(background, R, dev):
    """-> (bg_mode, bg tensor | None)"""
    if isinstance(background, str):
        if background == "last_sample":
            return _lib.BG_LAST_SAMPLE, None
        if background == "random":
            return _lib.BG_PER_RAY, torch.rand(R, 3, device=dev)
        raise ValueError(f"unknown background {background!r}")
    bg_t = _lib.f32c(torch.as_tensor(background, dtype=torch.float32).to(dev))
    return (_lib.BG_PER_RAY if bg_t.dim() == 2 else _lib.BG_COLOR), bg_t


def _render_grad(weights, rgb, normals, bins, background, clamp01, depth_method, want_acc, want_normal, clip_depth):
    """training path of _render: same outputs through RenderFn (explicit backward kernels)."""
    if depth_method == "median":
        bins_k, med = None, True
    else:
        bins_k, med = (bins if depth_method is not None else None), False
    R = weights.shape[0]
    bg_mode, bg_t = _background(background, R, weights.device) if rgb is not None else (_lib.BG_COLOR, None)
    o_rgb, o_depth, o_nrm, o_acc, mm = _ag.RenderFn.apply(weights[..., 0], rgb, normals if want_normal else None, bins_k, bg_t, bg_mode)
    res = {}
    if rgb is not None:
        res["rgb"] = torch.clamp(o_rgb, 0.0, 1.0) if clamp01 else o_rgb
    if want_normal:
        res["normal"] = o_nrm
    if want_acc:
        res["accumulation"] = o_acc[:, None]
    if med:
        with torch.no_grad():  # median depth is an index pick: no gradient (torch.searchsorted in the reference)
            res["depth"] = _render(weights.detach(), bins=bins, depth_method="median")["depth"]
    elif depth_method is not None:
        d = torch.clamp(o_depth, min=mm[0], max=mm[1]) if clip_depth else o_depth
        res["depth"] = d[:, None]
    return res


def _render(weights, rgb=None, normals=None, bins=None, background=None, clamp01=False, depth_method: Optional[str] = None,
            want_acc=False, want_normal=False, clip_depth=True):
    if _ag.needs_grad(weights, rgb, normals if want_normal else None):
        return _render_grad(weights, rgb, normals, bins, background, clamp01, depth_method, want_acc, want_normal, clip_depth)
    w = _lib.f32c(weights[..., 0])
    R = w.shape[0]
    bg_mode, bg_t = _background(background, R, w.device) if rgb is not None else (_lib.BG_COLOR, None)
    nrm_c = _lib.f32c(normals) if want_normal else None
    if nrm_c is not None and nrm_c.shape[-1] != 3:
        raise NotImplementedError("SemanticRenderer: only 3 channels (normals) are composited by the kernel")
    o_rgb, o_depth, o_nrm, o_acc, mm = _ag.launch_render(w, _lib.f32c(rgb) if rgb is not None else None, nrm_c,
                                                         bins if depth_method is not None else None, bg_t, bg_mode, clamp01,
                                                         depth_method == "median", want_acc)
    if depth_method == "expected" and clip_depth:
        _lib.check(_lib.load().sdfb200_depth_clip(_lib.ptr(o_depth), _lib.ptr(mm), R, _lib.stream_ptr()), "sdfb200_depth_clip")
    res = {}
    if o_rgb is not None:
        res["rgb"] = o_rgb
    if o_nrm is not None:
        res["normal"] = o_nrm
    if o_acc is not None:
        res["accumulation"] = o_acc[:, None]
    if o_depth is not None:
        res["depth"] = o_depth[:, None]
    return res


def _render_packed_grad(weights, idx, R, rgb, normals, starts, ends, background, clamp01, want_acc):
    """training path of _render_packed: same outputs through PackedRenderFn, the depth clip as a torch.clamp like the dense path."""
    bg_mode, bg_t = _lib.BG_COLOR, None
    if rgb is not None:
        if isinstance(background, str) and background == "last_sample":
            raise NotImplementedError("Background color 'last_sample' not implemented for packed samples.")
        bg_mode, bg_t = _background(background, R, weights.device)
    rs = lambda t, *shape: t.reshape(*shape) if t is not None else None  # noqa: E731
    o_rgb, o_depth, o_nrm, o_acc, mm = _ag.PackedRenderFn.apply(weights.reshape(-1), rs(rgb, -1, 3), rs(normals, -1, 3), rs(starts, -1), rs(ends, -1),
                                                                idx, R, bg_t, bg_mode)
    res = {}
    if rgb is not None:
        res["rgb"] = torch.clamp(o_rgb, 0.0, 1.0) if clamp01 else o_rgb
    if normals is not None:
        res["normal"] = o_nrm
    if want_acc:
        res["accumulation"] = o_acc[:, None]
    if starts is not None:
        lo, hi = mm[0], mm[1]
        if _ag.needs_grad(starts, ends):   # the clip bounds steps.min() / steps.max() (renderers.py:257) pass gradient to their samples
            steps = (starts + ends) / 2
            lo, hi = steps.min(), steps.max()
        res["depth"] = torch.clamp(o_depth, min=lo, max=hi)[:, None]
    return res


def _render_packed(weights, ray_indices, num_rays, rgb=None, normals=None, ray_samples=None, background=None, clamp01=False, want_acc=False,
                   want_normal=False, want_depth=False):
    """packed-sample branch (samples of all rays in one flat list + ``ray_indices``; what nerfacc.accumulate_along_rays does in the
    reference, renderers.py:74-79,192-194,249-253): one scatter-add launch + one per-ray finishing launch (sdfb200_render_packed).
    nerfacc.accumulate_along_rays is differentiable, so under autograd this goes through PackedRenderFn."""
    idx = ray_indices.reshape(-1).to(torch.int64).contiguous()
    starts = ray_samples.frustums.starts if want_depth else None
    ends = ray_samples.frustums.ends if want_depth else None
    if _ag.needs_grad(weights, rgb, normals if want_normal else None, starts, ends):
        return _render_packed_grad(weights, idx, int(num_rays), rgb, normals if want_normal else None, starts, ends, background, clamp01,
                                   want_acc)
    w = _lib.f32c(weights.reshape(-1))
    R = int(num_rays)
    bg_mode, bg_t = _lib.BG_COLOR, None
    if rgb is not None:
        if isinstance(background, str) and background == "last_sample":
            raise NotImplementedError("Background color 'last_sample' not implemented for packed samples.")
        bg_mode, bg_t = _background(background, R, w.device)
    rs = lambda t, *shape: _lib.f32c(t.reshape(*shape)) if t is not None else None  # noqa: E731
    o_rgb, o_depth, o_nrm, o_acc, mm = _ag.launch_render_packed(w, rs(rgb, -1, 3), rs(normals if want_normal else None, -1, 3), rs(starts, -1),
                                                                rs(ends, -1), idx, R, bg_t, bg_mode, clamp01, want_acc)
    res = {}
    if o_rgb is not None:
        res["rgb"] = o_rgb
    if o_nrm is not None:
        res["normal"] = o_nrm
    if o_acc is not None:
        res["accumulation"] = o_acc[:, None]
    if o_depth is not None:
        _lib.check(_lib.load().sdfb200_depth_clip(_lib.ptr(o_depth), _lib.ptr(mm), R, _lib.stream_ptr()), "sdfb200_depth_clip")
        res["depth"] = o_depth[:, None]
    return res


class RGBRenderer(nn.Module):
    """renderers.py:42-118, dense and packed (``ray_indices`` + ``num_rays``) branches."""

    def __init__(self, background_color: Union[str, torch.Tensor] = "random") -> None:
        super().__init__()
        self.background_color = background_color

    @classmethod
    def combine_rgb(cls, rgb, weights, background_color="random", ray_indices=None, num_rays=None):
        if ray_indices is not None and num_rays is not None:
            return _render_packed(weights, ray_indices, num_rays, rgb=rgb, background=background_color, clamp01=False)["rgb"]
        return _render(weights, rgb=rgb, background=background_color, clamp01=False)["rgb"]

    def forward(self, rgb, weights, ray_indices=None, num_rays=None):
        if ray_indices is not None and num_rays is not None:
            return _render_packed(weights, ray_indices, num_rays, rgb=rgb, background=self.background_color, clamp01=not self.training)["rgb"]
        return _render(weights, rgb=rgb, background=self.background_color, clamp01=not self.training)["rgb"]


class AccumulationRenderer(nn.Module):
    """renderers.py:171-197."""

    @classmethod
    def forward(cls, weights, ray_indices=None, num_rays=None):
        if ray_indices is not None and num_rays is not None:
            return _render_packed(weights, ray_indices, num_rays, want_acc=True)["accumulation"]
        return _render(weights, want_acc=True)["accumulation"]


class DepthRenderer(nn.Module):
    """renderers.py:200-261."""

    def __init__(self, method: str = "median") -> None:
        super().__init__()
        if method not in ("median", "expected"):
            raise NotImplementedError(f"Method {method} not implemented")
        self.method = method

    def forward(self, weights, ray_samples, ray_indices=None, num_rays=None):
        if ray_indices is not None and num_rays is not None:
            if self.method == "median":
                raise NotImplementedError("Median depth calculation is not implemented for packed samples.")
            return _render_packed(weights, ray_indices, num_rays, ray_samples=ray_samples, want_depth=True)["depth"]
        return _render(weights, bins=bins_of(ray_samples), depth_method=self.method)["depth"]


class SemanticRenderer(nn.Module):
    """renderers.py:284-295 (used as the normal renderer, base_surface_model.py:216)."""

    @classmethod
    def forward(cls, semantics, weights):
        return _render(weights, normals=semantics, want_normal=True)["normal"]


def render_all(weights, rgb, normals, ray_samples, background, training: bool = False, depth_method: str = "expected"):
    """rgb + depth + normal + accumulation in one launch (what SurfaceModel.get_outputs computes with four renderers)."""
    return _render(weights, rgb=rgb, normals=normals, bins=bins_of(ray_samples), background=background, clamp01=not training,
                   depth_method=depth_method, want_acc=True, want_normal=True)


def render_from_alphas(alphas, rgb, normals, ray_samples, background, training: bool = False, want_weights: bool = True):
    """alphas [R,S,1] -> weights + rgb + expected depth + normal + accumulation + bg_transmittance in ONE launch
    (sdfb200_render_alphas): the fused form of get_weights_and_transmittance_from_alphas + the four renderers."""
    if _ag.needs_grad(alphas, rgb, normals):
        R = alphas.shape[0]
        bg_mode, bg_t = _background(background, R, alphas.device)
        w, o_rgb, o_depth, o_nrm, o_acc, o_bgT, mm = _ag.RenderAlphasFn.apply(alphas[..., 0], rgb, normals, bins_of(ray_samples), bg_t, bg_mode)
        res = {"rgb": o_rgb if training else torch.clamp(o_rgb, 0.0, 1.0), "depth": torch.clamp(o_depth, min=mm[0], max=mm[1])[:, None],
               "normal": o_nrm, "accumulation": o_acc[:, None], "bg_transmittance": o_bgT[:, None]}
        if want_weights:
            res["weights"] = w[..., None]
        return res
    a = _lib.f32c(alphas[..., 0])
    R = a.shape[0]
    bg_mode, bg_t = _background(background, R, a.device)
    w, o_rgb, o_depth, o_nrm, o_acc, o_bgT, mm = _ag.launch_render_alphas(a, _lib.f32c(rgb), _lib.f32c(normals), bins_of(ray_samples), bg_t, bg_mode,
                                                                           not training, want_weights)
    _lib.check(_lib.load().sdfb200_depth_clip(_lib.ptr(o_depth), _lib.ptr(mm), R, _lib.stream_ptr()), "sdfb200_depth_clip")
    res = {"rgb": o_rgb, "depth": o_depth[:, None], "normal": o_nrm, "accumulation": o_acc[:, None], "bg_transmittance": o_bgT[:, None]}
    if want_weights:
        res["weights"] = w[..., None]
    return res
