"""Render-path composition above the kernels: collider -> sampler -> SDFField -> weights -> renderers, i.e. what
``SurfaceModel.get_outputs`` (nerfstudio/models/base_surface_model.py:292-365) does with ``NeuSModel.sample_and_forward_field``
(models/neus.py:85-116) or ``VolSDFModel.sample_and_forward_field`` (models/volsdf.py:62-87), plus the replacement of the
1024-ray Python chunk loop ``Model.get_outputs_for_camera_ray_bundle`` (models/base_model.py:165-189) by large chunks
(default 65 536 rays per launch sequence) and per-rank contiguous ray slices (parallel.py).

With ``field_background`` (NeRFField, TCNNNerfactoField or any field with the ``Field.forward`` contract) the renderer also runs the
background branch of base_surface_model.py:313-328.  This is host orchestration only; the losses and the training loop stay with sdfstudio.
"""
import copy
from typing import Dict, Optional

import torch
from torch import nn

from . import parallel
from .field_heads import FieldHeadNames
from .ray_samplers import ErrorBoundedSampler, LinearDisparitySampler, NeuSSampler
from .renderers import RGBRenderer, render_all, render_from_alphas


class SurfaceRenderer(nn.Module):
    """``kind="neus"``: NeuSSampler + alpha compositing; ``kind="volsdf"``: ErrorBoundedSampler + Laplace-density weights.
    ``field_background``: the background model, evaluated on ``num_samples_outside`` samples per ray between the far plane and
    ``far_plane_bg`` (SurfaceModelConfig.num_samples_outside / far_plane_bg) and merged as ``rgb += bg_transmittance * rgb_bg``."""

    def __init__(self, field, sampler, collider=None, kind: str = "neus", background_color="white", eval_num_rays_per_chunk: int = 65536,
                 field_background=None, num_samples_outside: int = 32, far_plane_bg: float = 1000.0):
        super().__init__()
        if kind not in ("neus", "volsdf"):
            raise ValueError("kind must be 'neus' or 'volsdf'")
        if kind == "neus" and not isinstance(sampler, NeuSSampler) or kind == "volsdf" and not isinstance(sampler, ErrorBoundedSampler):
            raise TypeError(f"sampler {type(sampler).__name__} does not match kind={kind!r}")
        self.field, self.sampler, self.collider, self.kind = field, sampler, collider, kind
        self.background_color = background_color
        self.eval_num_rays_per_chunk = eval_num_rays_per_chunk
        self.field_background = field_background
        self.far_plane_bg = far_plane_bg
        self.sampler_bg = LinearDisparitySampler(num_samples=num_samples_outside) if field_background is not None else None

    def _background(self, device):
        if isinstance(self.background_color, str) and self.background_color in ("white", "black"):
            return torch.full((3,), 1.0 if self.background_color == "white" else 0.0, device=device)
        return self.background_color

    def sample_and_forward_field(self, ray_bundle) -> Dict:
        if self.kind == "neus":                                                      # models/neus.py:85-116
            ray_samples = self.sampler(ray_bundle, sdf_fn=self.field.get_sdf)
            field_outputs = self.field(ray_samples, return_alphas=True)
            return {"ray_samples": ray_samples, "field_outputs": field_outputs}
        ray_samples, eik_points = self.sampler(ray_bundle, density_fn=self.field.laplace_density, sdf_fn=self.field.get_sdf)   # volsdf.py:62-87
        field_outputs = self.field(ray_samples)
        return {"ray_samples": ray_samples, "field_outputs": field_outputs, "eik_points": eik_points}

    def background_rgb(self, ray_bundle, background) -> torch.Tensor:
        """base_surface_model.py:317-326: the background field's colour of each ray, sampled from the far plane to far_plane_bg.  The
        caller's bundle is left as it is."""
        bundle = copy.copy(ray_bundle)
        bundle.nears = ray_bundle.fars
        bundle.fars = torch.ones_like(ray_bundle.fars) * self.far_plane_bg
        ray_samples_bg = self.sampler_bg(bundle)
        field_outputs_bg = self.field_background(ray_samples_bg)
        weights_bg = ray_samples_bg.get_weights(field_outputs_bg[FieldHeadNames.DENSITY])
        return RGBRenderer(background_color=background).train(self.training)(field_outputs_bg[FieldHeadNames.RGB], weights_bg)

    def get_outputs(self, ray_bundle) -> Dict[str, torch.Tensor]:
        """base_surface_model.py:292-365 without the patch warping branch."""
        if self.collider is not None:
            ray_bundle = self.collider(ray_bundle)
        s = self.sample_and_forward_field(ray_bundle)
        rs, fo = s["ray_samples"], s["field_outputs"]
        bg = self._background(ray_bundle.origins.device)
        if self.kind == "neus":
            out = render_from_alphas(fo[FieldHeadNames.ALPHA], fo[FieldHeadNames.RGB], fo[FieldHeadNames.NORMAL], rs, bg, training=self.training)
        elif self.field_background is None:
            weights = rs.get_weights(fo[FieldHeadNames.DENSITY])
            out = render_all(weights, fo[FieldHeadNames.RGB], fo[FieldHeadNames.NORMAL], rs, bg, training=self.training)
            out["weights"] = weights
        else:                                                                        # volsdf.py:67-68
            weights, transmittance = rs.get_weights_and_transmittance(fo[FieldHeadNames.DENSITY])
            out = render_all(weights, fo[FieldHeadNames.RGB], fo[FieldHeadNames.NORMAL], rs, bg, training=self.training)
            out["weights"] = weights
            out["bg_transmittance"] = transmittance[:, -1, :]
        if self.field_background is not None:
            out["rgb"] = out["rgb"] + out["bg_transmittance"] * self.background_rgb(ray_bundle, bg)
        dn = getattr(ray_bundle, "directions_norm", None)
        if dn is not None:
            out["depth"] = out["depth"] / dn                                        # base_surface_model.py:303-304
        if self.training:
            out["eik_grad"] = fo[FieldHeadNames.GRADIENT]
            out["points_norm"] = fo["points_norm"]
        out["field_outputs"] = fo
        return out

    def forward(self, ray_bundle):
        return self.get_outputs(ray_bundle)

    @torch.no_grad()
    def get_outputs_for_camera_ray_bundle(self, camera_ray_bundle, keys=("rgb", "depth", "normal", "accumulation"),
                                          image_shape: Optional[tuple] = None, distributed: bool = False) -> Optional[Dict[str, torch.Tensor]]:
        """base_model.py:165-189 with big chunks.  ``camera_ray_bundle``: the reference's [H, W] camera ray bundle (outputs come back
        as [H, W, k] like ``outputs[name].view(image_height, image_width, -1)`` there) or flat [N] rays in row-major image order (then
        ``image_shape`` optionally reshapes).  With ``distributed=True`` every rank renders its contiguous slice and rank 0 gets the
        gathered image (others: None)."""
        camera_ray_bundle, hw = parallel.flatten_ray_bundle(camera_ray_bundle)
        if hw is not None and image_shape is None:
            image_shape = hw
        n = camera_ray_bundle.origins.shape[0]
        bundle = camera_ray_bundle
        if distributed and parallel.dist.is_initialized() and parallel.dist.get_world_size() > 1:
            bundle = parallel.shard_ray_bundle(camera_ray_bundle, parallel.dist.get_rank(), parallel.dist.get_world_size())
        m = bundle.origins.shape[0]
        lists = {k: [] for k in keys}
        for i in range(0, m, self.eval_num_rays_per_chunk):
            o = self.get_outputs(parallel.slice_ray_bundle(bundle, i, min(m, i + self.eval_num_rays_per_chunk)))
            for k in keys:
                lists[k].append(o[k])
        outputs = {k: torch.cat(v) if v else torch.empty(0) for k, v in lists.items()}
        if bundle is not camera_ray_bundle:
            outputs = parallel.gather_outputs(outputs, n)
            if outputs is None:
                return None
        if image_shape is not None:
            outputs = {k: v.view(*image_shape, -1) for k, v in outputs.items()}
        return outputs
