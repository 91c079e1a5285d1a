"""Minimal stand-ins for the reference containers crossing the hot path's boundary
(nerfstudio/cameras/rays.py: Frustums :29-106, RaySamples :109-230, RayBundle :233-339).

When the modules of this package run *inside* sdfstudio they receive (and hand back, via
``ray_bundle.get_ray_samples``) the reference's own TensorDataclass objects -- they only rely on attribute names.
These classes exist so the package is usable stand-alone (tests, bench) and keep the same field names, shapes
(``[R, S, k]``) and methods.  The alpha/density -> weights math runs in libsdfb200.so (render.cu).
"""
from dataclasses import dataclass
from typing import Callable, Dict, Optional

import torch

from . import _lib
from . import autograd_ops as _ag


@dataclass
class Frustums:
    origins: torch.Tensor  # [R, S, 3] (expanded views are fine)
    directions: torch.Tensor  # [R, S, 3]
    starts: torch.Tensor  # [R, S, 1]
    ends: torch.Tensor  # [R, S, 1]
    pixel_area: torch.Tensor  # [R, S, 1]
    offsets: Optional[torch.Tensor] = None

    @property
    def shape(self):
        return self.starts.shape[:-1]

    def get_positions(self):
        pos = self.origins + self.directions * (self.starts + self.ends) / 2
        if self.offsets is not None:
            pos = pos + self.offsets
        return pos

    def get_start_positions(self):
        return self.origins + self.directions * self.starts


def bins_of(ray_samples) -> torch.Tensor:
    """[R, S+1] euclidean bin edges of a (reference or local) RaySamples.  The reference's starts/ends are overlapping
    slices of one [R, S+1] buffer (ray_samplers.py:119-125); rebuilding it costs one small copy."""
    b = getattr(ray_samples, "_euclid_bins", None)
    if b is not None:
        return b
    st, en = ray_samples.frustums.starts, ray_samples.frustums.ends
    return torch.cat([st[..., 0], en[..., -1:, 0]], dim=-1).float().contiguous()


def spacing_bins_of(ray_samples) -> torch.Tensor:
    b = getattr(ray_samples, "_spacing_bins", None)
    if b is not None:
        return b
    return torch.cat([ray_samples.spacing_starts[..., 0], ray_samples.spacing_ends[..., -1:, 0]], dim=-1).float().contiguous()


def rays_of(ray_samples):
    """(origins [R,3], directions [R,3]) from the per-sample expanded fields."""
    fr = ray_samples.frustums
    return _lib.f32c(fr.origins[:, 0, :]), _lib.f32c(fr.directions[:, 0, :])


def sample_geometry(ray_samples):
    """What the field kernels take for a RaySamples: (origins, directions, bins, shape).  Dense samples [R,S]: per-ray origins /
    directions [R,3] and euclidean bins [R,S+1].  Packed samples (flat frustums [N], NeuSAccSampler): per-sample origins / directions
    [N,3] and bins [N,2] = (start, end), i.e. N rays of one sample each.  `shape` is the frustums' shape ((R,S) or (N,))."""
    fr = ray_samples.frustums
    if fr.starts.dim() == 2:
        bins = torch.cat([fr.starts, fr.ends], dim=-1).float().contiguous()
        return _lib.f32c(fr.origins), _lib.f32c(fr.directions), bins, tuple(fr.starts.shape[:1])
    origins, directions = rays_of(ray_samples)
    return origins, directions, bins_of(ray_samples), tuple(fr.starts.shape[:2])


def point_or_ray_inputs(ray_samples):
    """What the background field kernels take for a RaySamples: (origins, directions, bins | None, n_rows, S, shape).  Ray mode when
    the samples carry this package's contiguous [R, S+1] bin buffer (make_ray_samples): per-ray origins / directions [R,3] and the
    bins, S samples per row.  Point mode for any other RaySamples: positions and directions [N,3] per sample, bins None and S = 0.
    `shape` is the frustums' shape."""
    fr = ray_samples.frustums
    shape = tuple(fr.starts.shape[:-1])
    bins = getattr(ray_samples, "_euclid_bins", None)
    if bins is not None and len(shape) == 2 and getattr(fr, "offsets", None) is None:
        origins, directions = rays_of(ray_samples)
        return origins, directions, bins, origins.shape[0], bins.shape[1] - 1, shape
    origins = _lib.f32c(fr.get_positions().reshape(-1, 3))
    directions = _lib.f32c(fr.directions.expand(*shape, 3).reshape(-1, 3))
    return origins, directions, None, origins.shape[0], 0, shape


def weights_from_alphas(alphas: torch.Tensor, with_transmittance: bool = False):
    """rays.py:194-230.  alphas [R,S,1] -> weights [R,S,1] (, transmittance [R,S+1,1])."""
    if _ag.needs_grad(alphas):
        w, T = _ag.WeightsFromAlphasFn.apply(alphas[..., 0])
    else:
        w, T = _ag.launch_weights_from_alphas(_lib.f32c(alphas[..., 0]), with_transmittance)
    return (w[..., None], T[..., None]) if with_transmittance else w[..., None]


def weights_from_density(bins: torch.Tensor, densities: torch.Tensor, with_transmittance: bool = False):
    """rays.py:146-192.  bins [R,S+1] euclidean, densities [R,S,1]."""
    if _ag.needs_grad(densities):
        w, T = _ag.WeightsFromDensityFn.apply(densities[..., 0], bins)
    else:
        w, T = _ag.launch_weights_from_density(_lib.f32c(densities[..., 0]), bins, with_transmittance)
    return (w[..., None], T[..., None]) if with_transmittance else w[..., None]


@dataclass
class RaySamples:
    frustums: Frustums
    camera_indices: Optional[torch.Tensor] = None
    deltas: Optional[torch.Tensor] = None
    spacing_starts: Optional[torch.Tensor] = None
    spacing_ends: Optional[torch.Tensor] = None
    spacing_to_euclidean_fn: Optional[Callable] = None
    metadata: Optional[Dict[str, torch.Tensor]] = None
    times: Optional[torch.Tensor] = None
    _euclid_bins: Optional[torch.Tensor] = None  # [R,S+1] backing buffers (kept to avoid re-concatenation)
    _spacing_bins: Optional[torch.Tensor] = None

    @property
    def shape(self):
        return self.frustums.shape

    def get_alphas(self, densities):
        return 1 - torch.exp(-(self.deltas * densities))

    def get_weights(self, densities):
        return weights_from_density(bins_of(self), densities)

    def get_weights_and_transmittance(self, densities):
        return weights_from_density(bins_of(self), densities, True)

    def get_weights_from_alphas(self, alphas):
        return weights_from_alphas(alphas)

    def get_weights_and_transmittance_from_alphas(self, alphas):
        return weights_from_alphas(alphas, True)


@dataclass
class RayBundle:
    origins: torch.Tensor  # [R, 3]
    directions: torch.Tensor  # [R, 3]
    pixel_area: torch.Tensor  # [R, 1]
    directions_norm: Optional[torch.Tensor] = None
    camera_indices: Optional[torch.Tensor] = None
    nears: Optional[torch.Tensor] = None
    fars: Optional[torch.Tensor] = None
    metadata: Optional[Dict[str, torch.Tensor]] = None
    times: Optional[torch.Tensor] = None

    def __len__(self):
        return self.origins.shape[0]

    def get_ray_samples(self, bin_starts, bin_ends, spacing_starts=None, spacing_ends=None, spacing_to_euclidean_fn=None) -> RaySamples:
        """rays.py:295-339."""
        R, S = bin_starts.shape[:2]
        fr = Frustums(
            origins=self.origins[:, None, :].expand(R, S, 3),
            directions=self.directions[:, None, :].expand(R, S, 3),
            starts=bin_starts,
            ends=bin_ends,
            pixel_area=self.pixel_area[:, None, :].expand(R, S, 1),
        )
        cam = None if self.camera_indices is None else self.camera_indices[:, None, :].expand(R, S, 1)
        return RaySamples(frustums=fr, camera_indices=cam, deltas=bin_ends - bin_starts, spacing_starts=spacing_starts, spacing_ends=spacing_ends,
                          spacing_to_euclidean_fn=spacing_to_euclidean_fn, metadata=self.metadata)


def make_ray_samples(ray_bundle, spacing_bins: torch.Tensor, euclid_bins: torch.Tensor, spacing_fn) -> RaySamples:
    """Wrap two [R,S+1] bin buffers as a RaySamples through the *bundle's own* get_ray_samples (so a reference RayBundle
    yields a reference RaySamples), and remember the backing buffers."""
    rs = ray_bundle.get_ray_samples(
        bin_starts=euclid_bins[..., :-1, None],
        bin_ends=euclid_bins[..., 1:, None],
        spacing_starts=spacing_bins[..., :-1, None],
        spacing_ends=spacing_bins[..., 1:, None],
        spacing_to_euclidean_fn=spacing_fn,
    )
    try:
        object.__setattr__(rs, "_euclid_bins", euclid_bins)
        object.__setattr__(rs, "_spacing_bins", spacing_bins)
    except Exception:  # a frozen / slotted foreign container: bins_of() falls back to concatenation
        pass
    return rs
