"""TEST INFRASTRUCTURE -- CPU restatement of the interlevel (proposal) losses of nerfstudio/model_components/losses.py: the
mip-NeRF 360 outer-measure form (:38-112) and the Zip-NeRF blurred-histogram form (:116-172).  Plain torch, dtype-generic: fed fp64
tensors it is the 'exact' answer the GPU tests calibrate fp32 noise against, and autograd through it gives the reference gradient
with respect to the proposal weights.  Pinned against the unmodified reference by tests/golden/losses.npz
(oracle/make_golden_losses.py) and, where the reference tree is present, directly (tests/test_oracle_losses.py).

Histograms are (edges [R, S+1], weights [R, S]) in the spacing domain; `c, w` is the final level, `cp, wp` a proposal level."""
import torch

OUTER_EPS = 1.0e-7
ZIP_EPS = 1.0e-5
ZIP_BLUR_RADII = (0.03, 0.003)


def _with_leading_zero(t):
    return torch.cat([torch.zeros_like(t[..., :1]), t], dim=-1)


def outer_measure(c, cp, wp):
    """Upper bound of a fine bin's weight from the proposal histogram: the summed weight of every proposal bin it touches (:38-67)."""
    n = wp.shape[-1]
    cy = _with_leading_zero(torch.cumsum(wp, dim=-1))
    first = (torch.searchsorted(cp[..., :-1].contiguous(), c[..., :-1].contiguous(), right=True) - 1).clamp(0, n - 1)
    last = torch.searchsorted(cp[..., 1:].contiguous(), c[..., 1:].contiguous(), right=True).clamp(0, n - 1)
    return torch.gather(cy, -1, last + 1) - torch.gather(cy, -1, first)


def interlevel_outer_elements(c, w, cp, wp):
    excess = (w - outer_measure(c, cp, wp)).clamp(min=0)
    return excess**2 / (w + OUTER_EPS)


def interlevel_outer(c, w, cp, wp):
    """One proposal level of interlevel_loss (:98-112): mean over the fine samples."""
    return interlevel_outer_elements(c, w, cp, wp).mean()


def blurred_histogram(c, w, radius):
    """The fine histogram as a density (w / width), convolved with a box of half-width `radius` (:116-128, :137, :143): piecewise linear
    with knots at c -+ radius.  Returns the sorted knots x [R, 2(S+1)] and the function's values there, clipped at 0."""
    density = w / (c[..., 1:] - c[..., :-1])
    zero = torch.zeros_like(density[..., :1])
    step = (torch.cat([density, zero], -1) - torch.cat([zero, density], -1)) / (2 * radius)      # jump of the density at each edge / 2r
    x, order = torch.sort(torch.cat([c - radius, c + radius], -1), dim=-1)
    slope_change = torch.gather(torch.cat([step, -step], -1), -1, order[..., :-1])
    dx = x[..., 1:] - x[..., :-1]
    y = _with_leading_zero(torch.cumsum(dx * torch.cumsum(slope_change, -1), -1))
    return x, y.clamp(min=0)


def resample_cdf(x, cdf, at):
    """Linear interpolation of (x, cdf) at `at` the way PDFSampler-style resampling does it (:156-165): side="right" search, indices
    clamped into the table, 0/0 -> 0, t clipped to [0, 1]."""
    n = x.shape[-1]
    idx = torch.searchsorted(x.contiguous(), at.contiguous(), right=True)
    lo, hi = (idx - 1).clamp(0, n - 1), idx.clamp(0, n - 1)
    x0, x1 = torch.gather(x, -1, lo), torch.gather(x, -1, hi)
    f0, f1 = torch.gather(cdf, -1, lo), torch.gather(cdf, -1, hi)
    t = torch.nan_to_num((at - x0) / (x1 - x0), 0).clamp(0, 1)
    return f0 + t * (f1 - f0)


def zip_target_weights(c, w, cp, radius):
    """What the proposal histogram should hold: the blurred fine histogram integrated over each proposal bin."""
    x, y = blurred_histogram(c, w, radius)
    dx = x[..., 1:] - x[..., :-1]
    cdf = _with_leading_zero(torch.cumsum((y[..., 1:] + y[..., :-1]) * 0.5 * dx, -1))
    at_edges = resample_cdf(x, cdf, cp)
    return at_edges[..., 1:] - at_edges[..., :-1]


def interlevel_zip_elements(c, w, cp, wp, radius):
    excess = (zip_target_weights(c, w, cp, radius) - wp).clamp(min=0)
    return excess**2 / (wp + ZIP_EPS)


def interlevel_zip(c, w, cp, wp, radius):
    """One proposal level of interlevel_loss_zip (:131-172): mean over the proposal samples."""
    return interlevel_zip_elements(c, w, cp, wp, radius).mean()


def interlevel_loss(bins_list, weights_list):
    """Sum over the proposal levels; the last entry of the lists is the final level and is treated as a constant."""
    c, w = bins_list[-1].detach(), weights_list[-1].detach()
    return sum(interlevel_outer(c, w, cp, wp) for cp, wp in zip(bins_list[:-1], weights_list[:-1]))


def interlevel_loss_zip(bins_list, weights_list):
    c, w = bins_list[-1].detach(), weights_list[-1].detach()
    return sum(interlevel_zip(c, w, cp, wp, r) for cp, wp, r in zip(bins_list[:-1], weights_list[:-1], ZIP_BLUR_RADII))
