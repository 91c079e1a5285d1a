"""TEST INFRASTRUCTURE -- CPU restatement of the ray samplers (SURVEY.md section 8a rows a2-a7) on plain tensors.

Follows nerfstudio/model_components/ray_samplers.py: SpacedSampler :80-127, PDFSampler :275-370,
ProposalNetworkSampler :537-578, ErrorBoundedSampler :613-788, NeuSSampler :847-944, UniSurfSampler :993-1130.

A sample set along R rays is a ``Bins``: spacing-domain bin edges ``[R, S+1]`` + euclidean bin edges ``[R, S+1]`` + the
spacing->euclidean map.  ``starts = euclid[:, :-1]``, ``ends = euclid[:, 1:]``, ``deltas = ends - starts``
(cameras/rays.py:295-339: the reference's starts/ends are overlapping slices of exactly this buffer).

Op order follows the reference so that ``searchsorted`` / ``sort`` indices are bit-identical on identical inputs
(torch-CPU semantics: ``cumsum`` accumulates in double and rounds each prefix to float).
"""
import math
from dataclasses import dataclass
from typing import Callable, List, Optional, Tuple

import torch

SPACING = {
    # name: (spacing_fn, spacing_fn_inv)   ray_samplers.py:130-247
    "uniform": (lambda x: x, lambda x: x),
    "lindisp": (lambda x: 1 / x, lambda x: 1 / x),
    "sqrt": (torch.sqrt, lambda x: x**2),
    "log": (torch.log, torch.exp),
    "piecewise": (lambda x: torch.where(x < 1, x / 2, 1 - 1 / (2 * x)), lambda x: torch.where(x < 0.5, 2 * x, 1 / (2 - 2 * x))),
}


@dataclass
class Bins:
    spacing: torch.Tensor  # [R, S+1]
    euclid: torch.Tensor  # [R, S+1]
    to_euclid: Callable

    @property
    def starts(self):
        return self.euclid[:, :-1]

    @property
    def ends(self):
        return self.euclid[:, 1:]

    @property
    def deltas(self):
        return self.euclid[:, 1:] - self.euclid[:, :-1]

    @property
    def num_samples(self):
        return self.euclid.shape[1] - 1


def make_to_euclid(kind: str, nears, fars):
    fn, inv = SPACING[kind]
    s_near, s_far = fn(nears.clone()), fn(fars.clone())
    return lambda x: inv(x * s_far + (1 - x) * s_near)


def spaced_sampler(nears, fars, num_samples: int, kind: str = "uniform", t_rand: Optional[torch.Tensor] = None) -> Bins:
    """ray_samplers.py:80-127.  nears/fars [R,1].  ``t_rand`` ([R,1] or [R,S+1]) = the stratified jitter the reference
    draws with torch.rand when ``training``; None = eval mode (no jitter)."""
    bins = torch.linspace(0.0, 1.0, num_samples + 1, dtype=nears.dtype)[None, :]
    if t_rand is not None:
        centers = (bins[..., 1:] + bins[..., :-1]) / 2.0
        upper = torch.cat([centers, bins[..., -1:]], -1)
        lower = torch.cat([bins[..., :1], centers], -1)
        bins = lower + (upper - lower) * t_rand
    to_euclid = make_to_euclid(kind, nears, fars)
    eu = to_euclid(bins)
    R = nears.shape[0]
    return Bins(bins.expand(R, -1) if bins.shape[0] == 1 else bins, eu, to_euclid)


def pdf_sampler(existing: Bins, weights, num_samples: int, histogram_padding: float = 0.01, include_original: bool = False,
                u_rand: Optional[torch.Tensor] = None, eps: float = 1e-5, return_indices: bool = False):
    """ray_samplers.py:275-370.  weights [R, S_in] (the reference's [..., 0] slice).  u_rand: jitter for training mode
    ([R,1] or [R,S_out+1]), None = eval mode."""
    num_bins = num_samples + 1
    w = weights + histogram_padding
    w_sum = torch.sum(w, dim=-1, keepdim=True)
    padding = torch.relu(eps - w_sum)
    w = w + padding / w.shape[-1]
    w_sum = w_sum + padding
    pdf = w / w_sum
    cdf = torch.min(torch.ones_like(pdf), torch.cumsum(pdf, dim=-1))
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], dim=-1)
    u = torch.linspace(0.0, 1.0 - (1.0 / num_bins), steps=num_bins, dtype=cdf.dtype)
    if u_rand is not None:
        u = u.expand(cdf.shape[0], num_bins) + u_rand / num_bins
    else:
        u = (u + 1.0 / (2 * num_bins)).expand(cdf.shape[0], num_bins)
    u = u.contiguous()
    eb = existing.spacing
    inds = torch.searchsorted(cdf, u, side="right")
    below = torch.clamp(inds - 1, 0, eb.shape[-1] - 1)
    above = torch.clamp(inds, 0, eb.shape[-1] - 1)
    cdf_g0 = torch.gather(cdf, -1, below)
    bins_g0 = torch.gather(eb, -1, below)
    cdf_g1 = torch.gather(cdf, -1, above)
    bins_g1 = torch.gather(eb, -1, above)
    t = torch.clip(torch.nan_to_num((u - cdf_g0) / (cdf_g1 - cdf_g0), 0), 0, 1)
    bins = bins_g0 + t * (bins_g1 - bins_g0)
    if include_original:
        bins, _ = torch.sort(torch.cat([eb, bins], -1), -1)
    out = Bins(bins, existing.to_euclid(bins), existing.to_euclid)
    if return_indices:
        return out, inds
    return out


def merge_bins(a: Bins, b: Bins) -> Tuple[Bins, torch.Tensor]:
    """ErrorBoundedSampler.merge_ray_samples, ray_samplers.py:758-788 (spacing-domain sort; returns sorted_index)."""
    ends = torch.maximum(a.spacing[:, -1:], b.spacing[:, -1:])
    bins, sorted_index = torch.sort(torch.cat([a.spacing[:, :-1], b.spacing[:, :-1]], -1), -1)
    bins = torch.cat([bins, ends], dim=-1)
    return Bins(bins, a.to_euclid(bins), a.to_euclid), sorted_index


def merge_bins_euclidean(a: Bins, b: Bins) -> Bins:
    """UniSurfSampler.merge_ray_samples_in_eculidean, ray_samplers.py:1095-1130 (spacing bins := euclidean bins)."""
    s1, s2 = a.to_euclid(a.spacing[:, :-1]), b.to_euclid(b.spacing[:, :-1])
    end = torch.maximum(a.to_euclid(a.spacing[:, -1:]), b.to_euclid(b.spacing[:, -1:]))
    eu, _ = torch.sort(torch.cat([s1, s2], -1), -1)
    eu = torch.cat([eu, end], dim=-1)
    return Bins(eu, eu, a.to_euclid)


# ---- density-form / alpha-form weights (cameras/rays.py:146-230) ------------------------------------------------
def weights_from_density(deltas, density):
    """rays.py:146-192: w = (1-exp(-sigma*delta)) * exp(-cumsum_excl(sigma*delta)); returns (weights, transmittance)."""
    dd = deltas * density
    alphas = 1 - torch.exp(-dd)
    T = torch.cumsum(dd[..., :-1], dim=-1)
    T = torch.cat([torch.zeros_like(T[..., :1]), T], dim=-1)
    T = torch.exp(-T)
    return alphas * T, T


def weights_from_alphas(alphas):
    """rays.py:194-230: T = cumprod([1, 1-alpha+1e-7]); w = alpha*T[:-1]; returns (weights [R,S], T [R,S+1])."""
    T = torch.cumprod(torch.cat([torch.ones_like(alphas[..., :1]), 1.0 - alphas + 1e-7], -1), -1)
    return alphas * T[..., :-1], T


# ---- NeuS ---------------------------------------------------------------------------------------------------------
def neus_fixed_inv_s_alpha(deltas, sdf, inv_s: float):
    """ray_samplers.py:909-944.  deltas, sdf [R,S] -> alpha [R,S-1]."""
    prev_sdf, next_sdf = sdf[:, :-1], sdf[:, 1:]
    d = deltas[:, :-1]
    mid = (prev_sdf + next_sdf) * 0.5
    cos_val = (next_sdf - prev_sdf) / (d + 1e-5)
    prev_cos = torch.cat([torch.zeros_like(cos_val[:, :1]), cos_val[:, :-1]], dim=-1)
    cos_val = torch.minimum(prev_cos, cos_val).clip(-1e3, 0.0)
    prev_esti = mid - cos_val * d * 0.5
    next_esti = mid + cos_val * d * 0.5
    prev_cdf = torch.sigmoid(prev_esti * inv_s)
    next_cdf = torch.sigmoid(next_esti * inv_s)
    return (prev_cdf - next_cdf + 1e-5) / (prev_cdf + 1e-5)


def neus_sampler(nears, fars, sdf_fn: Callable, num_samples=64, num_samples_importance=64, num_upsample_steps=4,
                 base_variance=64.0, t_rand=None, u_rands: Optional[List] = None, trace: Optional[list] = None) -> Bins:
    """ray_samplers.py:847-907.  ``sdf_fn(starts [R,k]) -> [R,k]``."""
    cur = spaced_sampler(nears, fars, num_samples, "uniform", t_rand)
    new = cur
    sdf = None
    sorted_index = None
    for it in range(num_upsample_steps):
        new_sdf = sdf_fn(new.starts)
        if sorted_index is not None:
            sdf = torch.gather(torch.cat([sdf, new_sdf], -1), 1, sorted_index)
        else:
            sdf = new_sdf
        alphas = neus_fixed_inv_s_alpha(cur.deltas, sdf, base_variance * 2**it)
        w, _ = weights_from_alphas(alphas)
        w = torch.cat((w, torch.zeros_like(w[:, :1])), dim=1)
        new, inds = pdf_sampler(cur, w, num_samples_importance // num_upsample_steps, histogram_padding=1e-5,
                                u_rand=None if u_rands is None else u_rands[it], return_indices=True)
        cur, sorted_index = merge_bins(cur, new)
        if trace is not None:
            trace.append({"sdf": sdf, "alphas": alphas, "weights": w, "inds": inds, "new_spacing": new.spacing, "sorted_index": sorted_index, "merged_spacing": cur.spacing})
    return cur


# ---- VolSDF error-bounded sampler ---------------------------------------------------------------------------------
def laplace_density(sdf, beta):
    """sdf_field.py:57-66."""
    alpha = 1.0 / beta
    return alpha * (0.5 + 0.5 * sdf.sign() * torch.expm1(-sdf.abs() / beta))


def volsdf_dstar(sdf, deltas):
    """ray_samplers.py:704-726."""
    d = sdf
    a, b, c = deltas[:, :-1], d[:, :-1].abs(), d[:, 1:].abs()
    first = a.pow(2) + b.pow(2) <= c.pow(2)
    second = a.pow(2) + c.pow(2) <= b.pow(2)
    d_star = torch.zeros(d.shape[0], d.shape[1] - 1, dtype=d.dtype)
    d_star[first] = b[first]
    d_star[second] = c[second]
    s = (a + b + c) / 2.0
    area = s * (s - a) * (s - b) * (s - c)
    mask = ~first & ~second & (b + c - a > 0)
    d_star[mask] = (2.0 * torch.sqrt(area[mask])) / (a[mask])
    d_star = (d[:, 1:].sign() * d[:, :-1].sign() == 1) * d_star
    return torch.cat((d_star, d_star[:, -1:]), dim=-1)


def volsdf_error_bound(beta, sdf, d_star, deltas):
    """ray_samplers.py:740-756.  beta broadcastable to [R,S]."""
    dens = laplace_density(sdf, beta)
    dd = deltas * dens
    integ = torch.cumsum(dd[..., :-1], dim=-1)
    integ = torch.cat([torch.zeros_like(integ[..., :1]), integ], dim=-1)
    err_sec = torch.exp(-d_star / beta) * (deltas**2.0) / (4 * beta**2)
    err_int = torch.cumsum(err_sec, dim=-1)
    bound = (torch.clamp(torch.exp(err_int), max=1.0e6) - 1.0) * torch.exp(-integ)
    return bound.max(-1)[0]


def volsdf_updated_beta(beta0, beta, sdf, d_star, deltas, eps: float, beta_iters: int):
    """ray_samplers.py:728-738.  beta0 [1]; beta [R] (modified in place like the reference)."""
    R = sdf.shape[0]
    curr = volsdf_error_bound(beta0, sdf, d_star, deltas)
    beta[curr <= eps] = beta0
    beta_min, beta_max = beta0.repeat(R), beta
    for _ in range(beta_iters):
        mid = (beta_min + beta_max) / 2.0
        curr = volsdf_error_bound(mid.unsqueeze(-1), sdf, d_star, deltas)
        beta_max[curr <= eps] = mid[curr <= eps]
        beta_min[curr > eps] = mid[curr > eps]
    return beta_max


def frustum_centres(origins, directions, bins: Bins):
    """Frustums.get_positions (rays.py:47-57): [R, S, 3] sample positions at the bin centres."""
    return origins[:, None, :] + directions[:, None, :] * ((bins.starts + bins.ends) / 2)[..., None]


def _next(rands: Optional[List], i: int):
    return None if rands is None else rands[i]


def error_bounded_sampler(nears, fars, sdf_fn: Callable, beta0, num_samples=64, num_samples_eval=128, num_samples_extra=32,
                          eps=0.1, beta_iters=10, max_total_iters=5, trace: Optional[list] = None, t_rand=None,
                          u_rands: Optional[List] = None, t_rand_extra=None, eikonal_idx=None, origins=None, directions=None):
    """ray_samplers.py:613-702.  Training mode takes the reference's draws in its order: ``t_rand`` of the first uniform
    draw, ``u_rands[k]`` of the k-th PDF draw (one per loop iteration) and ``t_rand_extra`` of the extra uniform draw.
    With ``eikonal_idx`` (the reference's torch.randint draw, :688-692) the frustum centres of the final pre-extra samples at
    those flat indices are returned as well: ``(bins, points)``."""
    cur = spaced_sampler(nears, fars, num_samples_eval, "uniform", t_rand)
    n_pdf = 0
    deltas = cur.deltas
    bound = (1.0 / (4.0 * torch.log(torch.tensor(eps + 1.0)))) * (deltas**2.0).sum(-1)
    beta = torch.sqrt(bound)
    total_iters, not_converge = 0, True
    sorted_index = None
    new = cur
    sdf = None
    while not_converge and total_iters < max_total_iters:
        new_sdf = sdf_fn(new.starts)
        if sorted_index is not None:
            sdf = torch.gather(torch.cat([sdf, new_sdf], -1), 1, sorted_index)
        else:
            sdf = new_sdf
        d_star = volsdf_dstar(sdf, cur.deltas)
        beta = volsdf_updated_beta(beta0, beta, sdf, d_star, cur.deltas, eps, beta_iters)
        density = laplace_density(sdf, beta.unsqueeze(-1))
        weights, transmittance = weights_from_density(cur.deltas, density)
        total_iters += 1
        not_converge = bool(beta.max() > beta0)
        if trace is not None:
            trace.append({"sdf": sdf.clone(), "d_star": d_star, "beta": beta.clone(), "S": cur.num_samples})
        if not_converge and total_iters < max_total_iters:
            deltas = cur.deltas
            err_sec = torch.exp(-d_star / beta.unsqueeze(-1)) * (deltas**2.0) / (4 * beta.unsqueeze(-1) ** 2)
            err_int = torch.cumsum(err_sec, dim=-1)
            w = (torch.clamp(torch.exp(err_int), max=1.0e6) - 1.0) * transmittance
            new = pdf_sampler(cur, w, num_samples_eval, histogram_padding=1e-5, u_rand=_next(u_rands, n_pdf))
            cur, sorted_index = merge_bins(cur, new)
        else:
            cur = pdf_sampler(cur, weights, num_samples, histogram_padding=1e-5, u_rand=_next(u_rands, n_pdf))
        n_pdf += 1
    points = None
    if eikonal_idx is not None:
        points = frustum_centres(origins, directions, cur).reshape(-1, 3)[eikonal_idx]
    if num_samples_extra > 0:
        uni = spaced_sampler(nears, fars, num_samples_extra, "uniform", t_rand_extra)
        cur, _ = merge_bins(cur, uni)
    return cur if eikonal_idx is None else (cur, points)


# ---- UniSurf ------------------------------------------------------------------------------------------------------
def unisurf_sampler(origins, directions, nears, fars, sdf_fn: Callable, delta: float = 0.25, num_samples_interval=64,
                    num_samples_outside=32, num_samples_importance=32, num_marching_steps=256, t_rand_march=None, u_rand_importance=None,
                    t_rand_outside=None, t_rand_interval=None):
    """ray_samplers.py:993-1093.  Returns (Bins, surface_points, mask).  Training mode takes the reference's draws: the
    marching, importance (PDF), outside and interval draws, in that order.  (The reference also draws 1024 random surface
    points, between the outside and the interval draws, when no ray has a surface crossing; those are not sample positions.)"""
    march = spaced_sampler(nears, fars, num_marching_steps, "uniform", t_rand_march)
    sdf = sdf_fn(march.starts)  # [R, M]
    occ = torch.sigmoid(-10.0 * sdf)
    w, _ = weights_from_alphas(occ)
    imp = pdf_sampler(march, w, num_samples_importance, histogram_padding=1e-5, u_rand=u_rand_importance)
    outside = spaced_sampler(nears, fars, num_samples_outside, "uniform", t_rand_outside)
    uni_imp, _ = merge_bins(imp, outside)
    z, mask, n2, f2 = unisurf_interval(march.starts, sdf, nears, fars, delta)
    surface_points = origins[mask] + directions[mask] * z[..., None]
    interval = spaced_sampler(n2, f2, num_samples_interval, "uniform", t_rand_interval)
    merged = merge_bins_euclidean(interval, uni_imp)
    return merged, surface_points, mask


def unisurf_interval(starts, sdf, nears, fars, delta: float):
    """ray_samplers.py:1031-1076: the first positive-to-negative sign change of the marching sdf [R, M] at the euclidean
    ``starts`` [R, M] -> (z of the hit rays [H], hit mask [R], new nears [R,1], new fars [R,1])."""
    R, M = sdf.shape
    sign_matrix = torch.cat([torch.sign(sdf[:, :-1] * sdf[:, 1:]), torch.ones(R, 1, dtype=sdf.dtype)], dim=-1)
    cost = sign_matrix * torch.arange(M, 0, -1).to(sdf.dtype)
    values, indices = torch.min(cost, -1)
    ar = torch.arange(R)
    mask = (values < 0) & (sdf[ar, indices] > 0)
    d_low, v_low = starts[ar, indices][mask], sdf[ar, indices][mask]
    ind2 = torch.clamp(indices + 1, max=M - 1)
    d_high, v_high = starts[ar, ind2][mask], sdf[ar, ind2][mask]
    z = (v_low * d_high - v_high * d_low) / (v_low - v_high)
    dists = fars - nears
    n2, f2 = nears.clone(), fars.clone()
    n2[mask] = z[:, None] - dists[mask] * delta
    f2[mask] = z[:, None] + dists[mask] * delta
    return z, mask, torch.maximum(n2, nears), torch.minimum(f2, fars)


# ---- proposal-network sampler (neus-facto / bakedsdf) ---------------------------------------------------------------
def proposal_sampler(origins, directions, nears, fars, density_fns: List[Callable], num_proposal_samples=(256, 96),
                     num_nerf_samples=48, anneal: float = 1.0, use_uniform: bool = False, t_rand=None, u_rands: Optional[List] = None):
    """ray_samplers.py:537-578.  density_fns[i](positions [R,S,3]) -> [R,S] (positions = frustum *centres*,
    rays.py:47-57).  Training mode takes the reference's draws: ``t_rand`` of the initial spaced draw and ``u_rands[i-1]`` of
    the PDF draw of level i.  Returns (final Bins, weights_list, bins_list)."""
    weights_list, bins_list = [], []
    n = len(num_proposal_samples)
    cur, weights = None, None
    for i in range(n + 1):
        is_prop = i < n
        ns = num_proposal_samples[i] if is_prop else num_nerf_samples
        if i == 0:
            cur = spaced_sampler(nears, fars, ns, "uniform" if use_uniform else "piecewise", t_rand)
        else:
            cur = pdf_sampler(cur, torch.pow(weights, anneal), ns, histogram_padding=0.01, u_rand=_next(u_rands, i - 1))
        if is_prop:
            dens = density_fns[i](frustum_centres(origins, directions, cur))
            weights, _ = weights_from_density(cur.deltas, dens)
            weights_list.append(weights)
            bins_list.append(cur)
    return cur, weights_list, bins_list
