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


_MM_INIT = {}


def _minmax_init(dev):
    """device-resident {+inf, -inf} (cloned on the device: no host->device copy / sync per call)."""
    t = _MM_INIT.get(str(dev))
    if t is None:
        t = torch.tensor([float("inf"), float("-inf")], device=dev, dtype=torch.float32)
        _MM_INIT[str(dev)] = t
    return t.clone()


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
    lib = _lib.load()
    w = _lib.f32c(weights[..., 0])
    R, S = w.shape
    dev = w.device
    out = _lib.RenderOut()
    res = {}
    bg_mode, bg_t = _lib.BG_COLOR, None
    rgb_c = None
    if rgb is not None:
        rgb_c = _lib.f32c(rgb)
        res["rgb"] = torch.empty(R, 3, device=dev, dtype=torch.float32)
        out.rgb = res["rgb"].data_ptr()
        if isinstance(background, str):
            if background == "last_sample":
                bg_mode = _lib.BG_LAST_SAMPLE
            elif background == "random":
                bg_mode, bg_t = _lib.BG_PER_RAY, torch.rand(R, 3, device=dev)
            else:
                raise ValueError(f"unknown background {background!r}")
        else:
            bg_t = _lib.f32c(torch.as_tensor(background, dtype=torch.float32).to(dev))
            if bg_t.dim() == 2:
                bg_mode = _lib.BG_PER_RAY
    nrm_c = None
    if want_normal:
        nrm_c = _lib.f32c(normals)
        res["normal"] = torch.empty(R, nrm_c.shape[-1], device=dev, dtype=torch.float32)
        if nrm_c.shape[-1] != 3:
            raise NotImplementedError("SemanticRenderer: only 3 channels (normals) are composited by the kernel")
        out.normal = res["normal"].data_ptr()
    if want_acc:
        res["accumulation"] = torch.empty(R, device=dev, dtype=torch.float32)
        out.accumulation = res["accumulation"].data_ptr()
    mm = None
    if depth_method is not None:
        res["depth"] = torch.empty(R, device=dev, dtype=torch.float32)
        out.depth = res["depth"].data_ptr()
        mm = _minmax_init(dev)
        out.steps_minmax = mm.data_ptr()
    _lib.check(lib.sdfb200_render(_lib.ptr(w), _lib.ptr(rgb_c), _lib.ptr(nrm_c), _lib.ptr(bins), _lib.ptr(bg_t), bg_mode, int(clamp01),
                                  int(depth_method == "median"), R, S, out, _lib.stream_ptr()), "sdfb200_render")
    if depth_method == "expected" and clip_depth:
        _lib.check(lib.sdfb200_depth_clip(out.depth, out.steps_minmax, R, _lib.stream_ptr()), "sdfb200_depth_clip")
    if "depth" in res:
        res["depth"] = res["depth"][:, None]
    if "accumulation" in res:
        res["accumulation"] = res["accumulation"][:, None]
    return res


def _render_packed(weights, ray_indices, num_rays, rgb=None, normals=None, ray_samples=None, background=None, clamp01=False, want_acc=False,
                   want_normal=False, want_depth=False):
    """packed-sample branch (samples of all rays in one flat list + ``ray_indices``; what nerfacc.accumulate_along_rays does in the
    reference, renderers.py:74-79,192-194,249-253): one scatter-add launch + one per-ray finishing launch (sdfb200_render_packed)."""
    lib = _lib.load()
    w = _lib.f32c(weights.reshape(-1))
    N, R = w.shape[0], int(num_rays)
    dev = w.device
    idx = ray_indices.reshape(-1).to(torch.int64).contiguous()
    out = _lib.RenderOut()
    res = {}
    rgb_c = nrm_c = st = en = bg_t = None
    bg_mode = _lib.BG_COLOR
    if rgb is not None:
        if isinstance(background, str) and background == "last_sample":
            raise NotImplementedError("Background color 'last_sample' not implemented for packed samples.")
        bg_mode, bg_t = _background(background, R, dev)
        rgb_c = _lib.f32c(rgb.reshape(-1, 3))
        res["rgb"] = torch.empty(R, 3, device=dev, dtype=torch.float32)
        out.rgb = res["rgb"].data_ptr()
    if want_normal:
        nrm_c = _lib.f32c(normals.reshape(-1, 3))
        res["normal"] = torch.empty(R, 3, device=dev, dtype=torch.float32)
        out.normal = res["normal"].data_ptr()
    if want_acc:
        res["accumulation"] = torch.empty(R, device=dev, dtype=torch.float32)
        out.accumulation = res["accumulation"].data_ptr()
    if want_depth:
        st, en = _lib.f32c(ray_samples.frustums.starts.reshape(-1)), _lib.f32c(ray_samples.frustums.ends.reshape(-1))
        res["depth"] = torch.empty(R, device=dev, dtype=torch.float32)
        mm = _minmax_init(dev)
        out.depth, out.steps_minmax = res["depth"].data_ptr(), mm.data_ptr()
    ws = torch.empty(max(R, 1) * 8, device=dev, dtype=torch.float32)
    _lib.check(lib.sdfb200_render_packed(_lib.ptr(w), _lib.ptr(rgb_c), _lib.ptr(nrm_c), _lib.ptr(st), _lib.ptr(en), _lib.ptr(idx), N, R, _lib.ptr(bg_t), bg_mode,
                                         int(clamp01), out, _lib.ptr(ws), ws.numel() * 4, _lib.stream_ptr()), "sdfb200_render_packed")
    if want_depth:
        _lib.check(lib.sdfb200_depth_clip(out.depth, out.steps_minmax, R, _lib.stream_ptr()), "sdfb200_depth_clip")
        res["depth"] = res["depth"][:, None]
    if want_acc:
        res["accumulation"] = res["accumulation"][:, None]
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
    lib = _lib.load()
    a = _lib.f32c(alphas[..., 0])
    R, S = a.shape
    dev = a.device
    rgb_c, nrm_c, bins = _lib.f32c(rgb), _lib.f32c(normals), bins_of(ray_samples)
    bg_mode, bg_t = _lib.BG_COLOR, None
    if isinstance(background, str):
        if background == "last_sample":
            bg_mode = _lib.BG_LAST_SAMPLE
        elif background == "random":
            bg_mode, bg_t = _lib.BG_PER_RAY, torch.rand(R, 3, device=dev)
        else:
            raise ValueError(f"unknown background {background!r}")
    else:
        bg_t = _lib.f32c(torch.as_tensor(background, dtype=torch.float32).to(dev))
        if bg_t.dim() == 2:
            bg_mode = _lib.BG_PER_RAY
    res = {"rgb": torch.empty(R, 3, device=dev), "depth": torch.empty(R, device=dev), "normal": torch.empty(R, 3, device=dev),
           "accumulation": torch.empty(R, device=dev), "bg_transmittance": torch.empty(R, device=dev)}
    w = torch.empty(R, S, device=dev) if want_weights else None
    mm = _minmax_init(dev)
    out = _lib.RenderOut()
    out.rgb, out.depth, out.normal, out.accumulation, out.steps_minmax = (res["rgb"].data_ptr(), res["depth"].data_ptr(), res["normal"].data_ptr(),
                                                                           res["accumulation"].data_ptr(), mm.data_ptr())
    _lib.check(lib.sdfb200_render_alphas(_lib.ptr(a), _lib.ptr(rgb_c), _lib.ptr(nrm_c), _lib.ptr(bins), _lib.ptr(bg_t), bg_mode, int(not training), R, S,
                                         _lib.ptr(w), res["bg_transmittance"].data_ptr(), out, _lib.stream_ptr()), "sdfb200_render_alphas")
    _lib.check(lib.sdfb200_depth_clip(out.depth, out.steps_minmax, R, _lib.stream_ptr()), "sdfb200_depth_clip")
    res["depth"], res["accumulation"], res["bg_transmittance"] = res["depth"][:, None], res["accumulation"][:, None], res["bg_transmittance"][:, None]
    if want_weights:
        res["weights"] = w[..., None]
    return res
