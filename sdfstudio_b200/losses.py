"""The interlevel losses that train the proposal networks (nerfstudio/model_components/losses.py:38-172), drop-ins with the
reference's names and signatures:

  interlevel_loss      <- losses.interlevel_loss      (mip-NeRF 360: bakedsdf, bakedangelo, neuralangelo)
  interlevel_loss_zip  <- losses.interlevel_loss_zip  (Zip-NeRF: neus-facto)
  ray_samples_to_sdist <- losses.ray_samples_to_sdist

``weights_list`` / ``ray_samples_list`` are what ProposalNetworkSampler returns with the final level appended, as the models build
them (models/neus_facto.py:307-310).  The RaySamples may be this package's or the reference's.  Each proposal level is one kernel
launch plus a fixed-order reduction (sdfb200_interlevel_loss); nothing synchronises with the host: the reference's
``assert (y_r >= 0).all()`` is not reproduced, the values are clipped at 0 the line before it.

Gradients flow to the proposal weights only.  The final level is detached, as in the reference, and a bin-edge tensor that requires
grad is treated as a constant: PDFSampler detaches the edges it draws, so the reference's edges never carry a gradient either.
"""
import torch

from . import _lib
from .autograd_ops import InterlevelLossFn
from .rays import spacing_bins_of

ZIP_BLUR_RADII = (0.03, 0.003)     # losses.py:140, zipped against the proposal levels: a third level is not visited


def ray_samples_to_sdist(ray_samples) -> torch.Tensor:
    """The spacing-domain bin edges [R, S+1] of a sample set (losses.py:90-95)."""
    return spacing_bins_of(ray_samples)


def _levels(weights_list, ray_samples_list, what):
    """[(bins [R,S+1], weights [R,S])] per level after the shape and device checks (no launch before they pass)."""
    if len(weights_list) != len(ray_samples_list) or len(weights_list) == 0:
        raise ValueError(f"{what}: weights_list and ray_samples_list must have the same, non-zero length "
                         f"({len(weights_list)} and {len(ray_samples_list)})")
    levels = []
    for i, (weights, ray_samples) in enumerate(zip(weights_list, ray_samples_list)):
        bins = ray_samples_to_sdist(ray_samples)
        w = weights[..., 0]
        if w.dim() != 2 or bins.dim() != 2:
            raise ValueError(f"{what}: level {i} needs weights [R, S, 1] and bin edges [R, S+1], got {tuple(weights.shape)} and {tuple(bins.shape)}")
        if bins.shape != (w.shape[0], w.shape[1] + 1):
            raise ValueError(f"{what}: level {i} has weights {tuple(weights.shape)} but bin edges {tuple(bins.shape)}")
        if levels and w.shape[0] != levels[0][1].shape[0]:
            raise ValueError(f"{what}: level {i} has {w.shape[0]} rays, level 0 has {levels[0][1].shape[0]}")
        levels.append((bins, w))
    for bins, w in levels:
        _lib.require_cuda(w.device, f"losses.{what}")
        _lib.require_cuda(bins.device, f"losses.{what}")
    return levels


def _interlevel(weights_list, ray_samples_list, form, radii, what):
    levels = _levels(weights_list, ray_samples_list, what)
    c, w = levels[-1]
    c, w = _lib.f32c(c.detach()), _lib.f32c(w.detach())
    total = torch.zeros((), device=w.device, dtype=torch.float32)
    proposals = levels[:-1] if radii is None else levels[:-1][: len(radii)]
    for k, (cp, wp) in enumerate(proposals):
        if wp.shape[0] == 0:
            total = total + wp.sum() * float("nan")          # torch.mean over no elements
            continue
        total = total + InterlevelLossFn.apply(wp, _lib.f32c(cp.detach()), c, w, form, 0.0 if radii is None else radii[k])
    return total


def interlevel_loss(weights_list, ray_samples_list) -> torch.Tensor:
    """The proposal loss of mip-NeRF 360 (losses.py:98-112): per proposal level, the mean over the fine samples of
    max(w - w_outer, 0)^2 / (w + 1e-7), w_outer the proposal weight of the proposal bins a fine bin touches.  0-dim CUDA tensor."""
    return _interlevel(weights_list, ray_samples_list, _lib.INTERLEVEL_OUTER, None, "interlevel_loss")


def interlevel_loss_zip(weights_list, ray_samples_list) -> torch.Tensor:
    """The proposal loss of Zip-NeRF (losses.py:131-172): the fine histogram blurred with radius 0.03 for the first proposal level and
    0.003 for the second, resampled on that level's bins; the mean over the proposal samples of max(w_gt - wp, 0)^2 / (wp + 1e-5).
    0-dim CUDA tensor.  A fine bin of zero width makes its ray's loss inf or NaN, as the reference's division by the width does."""
    return _interlevel(weights_list, ray_samples_list, _lib.INTERLEVEL_ZIP, ZIP_BLUR_RADII, "interlevel_loss_zip")
