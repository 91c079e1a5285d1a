"""H100-native drop-ins for ``nerfstudio.model_components.ray_samplers`` (same class names, constructor arguments,
``forward`` signatures and train/eval behaviour).  Every per-ray scan runs in libsdfb200.so (csrc/samplers.cu); the
Python here only sequences kernels and draws the training-mode jitter with ``torch.rand`` in the reference's order.
"""
import math
from typing import Callable, List, Optional, Tuple, Union

import torch
from torch import nn

from . import _lib
from .rays import bins_of, make_ray_samples, spacing_bins_of, weights_from_alphas

_SPACING_TORCH = {
    "uniform": (lambda x: x, lambda x: x),
    "lindisp": (lambda x: 1 / x, lambda x: 1 / x),
    "sqrt": (torch.sqrt, lambda x: x**2),
    "log": (torch.log, torch.exp),
    "piecewise": (lambda x: torch.where(x < 1, x / 2, 1 - 1 / (2 * x)), lambda x: torch.where(x < 0.5, 2 * x, 1 / (2 - 2 * x))),
}


class SpacingFn:
    """``spacing_to_euclidean_fn`` (ray_samplers.py:115-116) as an object: callable on tensors like the reference's
    lambda, and carrying (kind, nears, fars) so the kernels can apply the same map in-register."""

    def __init__(self, kind: str, nears: torch.Tensor, fars: torch.Tensor):
        self.kind = kind
        self.nears = _lib.f32c(nears.reshape(-1))
        self.fars = _lib.f32c(fars.reshape(-1))

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        if self.kind == "identity":
            return x
        fn, inv = _SPACING_TORCH[self.kind]
        shape = [-1] + [1] * (x.dim() - 1)
        s_near, s_far = fn(self.nears.view(shape)), fn(self.fars.view(shape))
        return inv(x * s_far + (1 - x) * s_near)

    def to_euclid(self, spacing_bins: torch.Tensor) -> torch.Tensor:
        """[R, nb] spacing bins -> euclidean bins through sdfb200_bins_to_euclid."""
        lib = _lib.load()
        sb = _lib.f32c(spacing_bins)
        out = torch.empty_like(sb)
        _lib.check(lib.sdfb200_bins_to_euclid(_lib.ptr(sb), _lib.ptr(self.nears), _lib.ptr(self.fars), sb.shape[0], sb.shape[1],
                                              _lib.SPACING[self.kind], _lib.ptr(out), _lib.stream_ptr()), "sdfb200_bins_to_euclid")
        return out


def _to_euclid(fn, spacing_bins):
    if isinstance(fn, SpacingFn):
        return fn.to_euclid(spacing_bins)
    return _lib.f32c(fn(spacing_bins))  # a foreign (reference) closure: elementwise torch ops on the GPU


_host_cache = {}


def _linspace_dev(start: float, end: float, steps: int, device, add: float = 0.0) -> torch.Tensor:
    """torch.linspace evaluated on the CPU (bit-identical to the reference's CPU values), cached per device."""
    key = (start, end, steps, add, str(device))
    t = _host_cache.get(key)
    if t is None:
        t = torch.linspace(start, end, steps)
        if add != 0.0:
            t = t + add
        t = t.to(device)
        _host_cache[key] = t
    return t


class Sampler(nn.Module):
    """ray_samplers.py:32-52."""

    def __init__(self, num_samples: Optional[int] = None) -> None:
        super().__init__()
        self.num_samples = num_samples

    def generate_ray_samples(self, *args, **kwargs):
        raise NotImplementedError

    def forward(self, *args, **kwargs):
        return self.generate_ray_samples(*args, **kwargs)


def identify_spacing(spacing_fn, spacing_fn_inv=None) -> str:
    """Name of the (spacing_fn, spacing_fn_inv) pair: the kernels implement the reference's five spacings (ray_samplers.py:130-247)
    in-register, so a callable is recognised by evaluating it on a few probe values.  Anything else is refused (there is no
    PyTorch fallback path in this package)."""
    if isinstance(spacing_fn, str):
        if spacing_fn not in _SPACING_TORCH:
            raise ValueError(f"unknown spacing {spacing_fn!r}; one of {sorted(_SPACING_TORCH)}")
        return spacing_fn
    probe = torch.tensor([0.25, 0.5, 0.75, 1.0, 1.5, 2.0, 4.0, 9.0], dtype=torch.float64)
    try:
        got = torch.as_tensor(spacing_fn(probe), dtype=torch.float64)
    except Exception as e:  # noqa: BLE001
        raise NotImplementedError(f"spacing_fn could not be evaluated on a probe tensor: {e}") from e
    for name, (fn, inv) in _SPACING_TORCH.items():
        if torch.allclose(got, fn(probe), rtol=1e-12, atol=0):
            if spacing_fn_inv is not None:
                back = torch.as_tensor(spacing_fn_inv(fn(probe)), dtype=torch.float64)
                if not torch.allclose(back, probe, rtol=1e-9, atol=0):
                    raise ValueError(f"spacing_fn_inv is not the inverse of the {name!r} spacing_fn")
            return name
    raise NotImplementedError("SpacedSampler: only the reference's spacings (uniform, 1/x, sqrt, log, uniform+lindisp piecewise) run in the "
                              "kernels; this spacing_fn is none of them")


class SpacedSampler(Sampler):
    """ray_samplers.py:55-127, same constructor: ``spacing_fn`` / ``spacing_fn_inv`` callables (recognised by probing, see
    ``identify_spacing``); a spacing NAME ("uniform", "lindisp", "sqrt", "log", "piecewise") is accepted in place of ``spacing_fn``."""

    def __init__(self, spacing_fn, spacing_fn_inv=None, num_samples: Optional[int] = None, train_stratified=True, single_jitter=False) -> None:
        super().__init__(num_samples=num_samples)
        self.spacing = identify_spacing(spacing_fn, spacing_fn_inv)
        self.spacing_fn, self.spacing_fn_inv = _SPACING_TORCH[self.spacing]
        self.train_stratified = train_stratified
        self.single_jitter = single_jitter

    def generate_ray_samples(self, ray_bundle=None, num_samples: Optional[int] = None):
        assert ray_bundle is not None and ray_bundle.nears is not None and ray_bundle.fars is not None
        num_samples = num_samples or self.num_samples
        assert num_samples is not None
        lib = _lib.load()
        dev = ray_bundle.origins.device
        R = ray_bundle.origins.shape[0]
        base = _linspace_dev(0.0, 1.0, num_samples + 1, dev)
        jitter, per_bin = None, 0
        if self.train_stratified and self.training:
            per_bin = 0 if self.single_jitter else 1
            jitter = torch.rand((R, 1) if self.single_jitter else (R, num_samples + 1), dtype=torch.float32, device=dev)
        fn = SpacingFn(self.spacing, ray_bundle.nears, ray_bundle.fars)
        sp = torch.empty(R, num_samples + 1, device=dev, dtype=torch.float32)
        eu = torch.empty_like(sp)
        _lib.check(lib.sdfb200_spaced_bins(_lib.ptr(fn.nears), _lib.ptr(fn.fars), _lib.ptr(base), _lib.ptr(jitter), per_bin, R, num_samples,
                                           _lib.SPACING[self.spacing], _lib.ptr(sp), _lib.ptr(eu), _lib.stream_ptr()), "sdfb200_spaced_bins")
        return make_ray_samples(ray_bundle, sp, eu, fn)


class UniformSampler(SpacedSampler):
    def __init__(self, num_samples=None, train_stratified=True, single_jitter=False) -> None:
        super().__init__("uniform", None, num_samples, train_stratified, single_jitter)


class LinearDisparitySampler(SpacedSampler):
    def __init__(self, num_samples=None, train_stratified=True, single_jitter=False) -> None:
        super().__init__("lindisp", None, num_samples, train_stratified, single_jitter)


class SqrtSampler(SpacedSampler):
    def __init__(self, num_samples=None, train_stratified=True, single_jitter=False) -> None:
        super().__init__("sqrt", None, num_samples, train_stratified, single_jitter)


class LogSampler(SpacedSampler):
    def __init__(self, num_samples=None, train_stratified=True, single_jitter=False) -> None:
        super().__init__("log", None, num_samples, train_stratified, single_jitter)


class UniformLinDispPiecewiseSampler(SpacedSampler):
    def __init__(self, num_samples=None, train_stratified=True, single_jitter=False) -> None:
        super().__init__("piecewise", None, num_samples, train_stratified, single_jitter)


def _pdf_sample(spacing_bins, weights2d, num_samples, histogram_padding, include_original, training_jitter, single_jitter, eps=1e-5,
                return_inds=False):
    """sdfb200_pdf_sample on [R,S_in+1] spacing bins and [R,S_in] weights."""
    lib = _lib.load()
    dev = spacing_bins.device
    R, s_in = weights2d.shape
    nb = num_samples + 1
    if training_jitter:
        u = _linspace_dev(0.0, 1.0 - (1.0 / nb), nb, dev)
        jitter = torch.rand((R, 1) if single_jitter else (R, nb), device=dev)
        per_bin = 0 if single_jitter else 1
    else:
        u = _linspace_dev(0.0, 1.0 - (1.0 / nb), nb, dev, add=1.0 / (2 * nb))
        jitter, per_bin = None, 0
    out = torch.empty(R, (s_in + 1 + nb) if include_original else nb, device=dev, dtype=torch.float32)
    inds = torch.empty(R, nb, device=dev, dtype=torch.int64) if return_inds else None
    _lib.check(lib.sdfb200_pdf_sample(_lib.ptr(weights2d), _lib.ptr(spacing_bins), _lib.ptr(u), _lib.ptr(jitter), per_bin, R, s_in, num_samples,
                                      float(histogram_padding), float(eps), int(include_original), _lib.ptr(out), _lib.ptr(inds),
                                      _lib.stream_ptr()), "sdfb200_pdf_sample")
    return (out, inds) if return_inds else out


class PDFSampler(Sampler):
    """ray_samplers.py:250-370."""

    def __init__(self, num_samples=None, train_stratified=True, single_jitter=False, include_original=True, histogram_padding=0.01) -> None:
        super().__init__(num_samples=num_samples)
        self.train_stratified = train_stratified
        self.include_original = include_original
        self.histogram_padding = histogram_padding
        self.single_jitter = single_jitter

    def generate_ray_samples(self, ray_bundle=None, ray_samples=None, weights=None, num_samples: Optional[int] = None, eps: float = 1e-5,
                             return_indices: bool = False):
        if ray_samples is None or ray_bundle is None:
            raise ValueError("ray_samples and ray_bundle must be provided")
        num_samples = num_samples or self.num_samples
        assert num_samples is not None
        assert ray_samples.spacing_starts is not None and ray_samples.spacing_ends is not None
        assert ray_samples.spacing_to_euclidean_fn is not None
        sb = spacing_bins_of(ray_samples)
        w = _lib.f32c(weights[..., 0].detach())
        res = _pdf_sample(sb, w, num_samples, self.histogram_padding, self.include_original, self.train_stratified and self.training,
                          self.single_jitter, eps, return_indices)
        bins, inds = res if return_indices else (res, None)
        fn = ray_samples.spacing_to_euclidean_fn
        out = make_ray_samples(ray_bundle, bins, _to_euclid(fn, bins), fn)
        return (out, inds) if return_indices else out


def merge_ray_samples(ray_bundle, ray_samples_1, ray_samples_2):
    """ErrorBoundedSampler.merge_ray_samples, ray_samplers.py:758-788 -> (RaySamples, sorted_index)."""
    lib = _lib.load()
    a, b = spacing_bins_of(ray_samples_1), spacing_bins_of(ray_samples_2)
    R, sa, sb = a.shape[0], a.shape[1] - 1, b.shape[1] - 1
    merged = torch.empty(R, sa + sb + 1, device=a.device, dtype=torch.float32)
    sidx = torch.empty(R, sa + sb, device=a.device, dtype=torch.int64)
    _lib.check(lib.sdfb200_merge_bins(_lib.ptr(a), _lib.ptr(b), R, sa, sb, _lib.ptr(merged), _lib.ptr(sidx), _lib.stream_ptr()), "sdfb200_merge_bins")
    fn = ray_samples_1.spacing_to_euclidean_fn
    return make_ray_samples(ray_bundle, merged, _to_euclid(fn, merged), fn), sidx


def _merge_gather(sdf_a, sdf_b, sorted_index):
    """torch.gather(cat([a, b], -1), 1, sorted_index) on [R,Sa,1] / [R,Sb,1] -> [R,Sa+Sb,1]."""
    lib = _lib.load()
    a, b = _lib.f32c(sdf_a[..., 0]), _lib.f32c(sdf_b[..., 0])
    R, sa, sb = a.shape[0], a.shape[1], b.shape[1]
    out = torch.empty(R, sa + sb, device=a.device, dtype=torch.float32)
    _lib.check(lib.sdfb200_merge_gather(_lib.ptr(a), _lib.ptr(b), _lib.ptr(sorted_index), R, sa, sb, _lib.ptr(out), _lib.stream_ptr()),
               "sdfb200_merge_gather")
    return out[..., None]


class ProposalNetworkSampler(Sampler):
    """ray_samplers.py:497-578."""

    def __init__(self, num_proposal_samples_per_ray: Tuple[int, ...] = (64,), num_nerf_samples_per_ray: int = 32,
                 num_proposal_network_iterations: int = 2, use_uniform_sampler: bool = False, single_jitter: bool = False,
                 update_sched: Callable = lambda x: 1) -> None:
        super().__init__()
        self.num_proposal_samples_per_ray = num_proposal_samples_per_ray
        self.num_nerf_samples_per_ray = num_nerf_samples_per_ray
        self.num_proposal_network_iterations = num_proposal_network_iterations
        self.update_sched = update_sched
        if self.num_proposal_network_iterations < 1:
            raise ValueError("num_proposal_network_iterations must be >= 1")
        self.initial_sampler = UniformSampler(single_jitter=single_jitter) if use_uniform_sampler else UniformLinDispPiecewiseSampler(single_jitter=single_jitter)
        self.pdf_sampler = PDFSampler(include_original=False, single_jitter=single_jitter)
        self._anneal = 1.0
        self._steps_since_update = 0
        self._step = 0

    def set_anneal(self, anneal: float) -> None:
        self._anneal = anneal

    def step_cb(self, step):
        self._step = step
        self._steps_since_update += 1

    def generate_ray_samples(self, ray_bundle=None, density_fns: Optional[List[Callable]] = None):
        assert ray_bundle is not None and density_fns is not None
        weights_list, ray_samples_list = [], []
        n = self.num_proposal_network_iterations
        weights, ray_samples = None, None
        updated = self._steps_since_update > self.update_sched(self._step) or self._step < 10
        for i_level in range(n + 1):
            is_prop = i_level < n
            num_samples = self.num_proposal_samples_per_ray[i_level] if is_prop else self.num_nerf_samples_per_ray
            if i_level == 0:
                ray_samples = self.initial_sampler(ray_bundle, num_samples=num_samples)
            else:
                annealed = weights if self._anneal == 1.0 else torch.pow(weights, self._anneal)
                ray_samples = self.pdf_sampler(ray_bundle, ray_samples, annealed, num_samples=num_samples)
            if is_prop:
                if updated:
                    density = density_fns[i_level](ray_samples.frustums.get_positions())
                else:
                    with torch.no_grad():
                        density = density_fns[i_level](ray_samples.frustums.get_positions())
                weights = ray_samples.get_weights(density)
                weights_list.append(weights)
                ray_samples_list.append(ray_samples)
        if updated:
            self._steps_since_update = 0
        return ray_samples, weights_list, ray_samples_list


class ErrorBoundedSampler(Sampler):
    """VolSDF's error-bounded sampler, ray_samplers.py:581-788."""

    def __init__(self, num_samples: int = 64, num_samples_eval: int = 128, num_samples_extra: int = 32, eps: float = 0.1, beta_iters: int = 10,
                 max_total_iters: int = 5, add_tiny: float = 1e-6, single_jitter: bool = False) -> None:
        super().__init__()
        self.num_samples, self.num_samples_eval, self.num_samples_extra = num_samples, num_samples_eval, num_samples_extra
        self.eps, self.beta_iters, self.max_total_iters, self.add_tiny, self.single_jitter = eps, beta_iters, max_total_iters, add_tiny, single_jitter
        self.uniform_sampler = UniformSampler(single_jitter=single_jitter)
        self.pdf_sampler = PDFSampler(include_original=False, single_jitter=single_jitter, histogram_padding=1e-5)

    def merge_ray_samples(self, ray_bundle, ray_samples_1, ray_samples_2):
        return merge_ray_samples(ray_bundle, ray_samples_1, ray_samples_2)

    def generate_ray_samples(self, ray_bundle=None, density_fn=None, sdf_fn=None, return_eikonal_points: bool = True):
        assert ray_bundle is not None and density_fn is not None and sdf_fn is not None
        lib = _lib.load()
        beta0 = _lib.f32c(density_fn.get_beta().detach())
        ray_samples = self.uniform_sampler(ray_bundle, num_samples=self.num_samples_eval)
        R = ray_bundle.origins.shape[0]
        dev = beta0.device
        beta = torch.empty(R, device=dev, dtype=torch.float32)
        eu = bins_of(ray_samples)
        _lib.check(lib.sdfb200_volsdf_init_beta(_lib.ptr(eu), R, eu.shape[1] - 1, float(self.eps), _lib.ptr(beta), _lib.stream_ptr()),
                   "sdfb200_volsdf_init_beta")
        total_iters, not_converge = 0, True
        sorted_index, sdf = None, None
        new_samples = ray_samples
        while not_converge and total_iters < self.max_total_iters:
            with torch.no_grad():
                new_sdf = sdf_fn(new_samples)
            sdf = _merge_gather(sdf, new_sdf, sorted_index) if sorted_index is not None else new_sdf
            eu = bins_of(ray_samples)
            S = eu.shape[1] - 1
            sdf2 = _lib.f32c(sdf[..., 0])
            weights = torch.empty(R, S, device=dev, dtype=torch.float32)
            err_w = torch.empty(R, S, device=dev, dtype=torch.float32)
            _lib.check(lib.sdfb200_volsdf_step(_lib.ptr(eu), _lib.ptr(sdf2), _lib.ptr(beta0), _lib.ptr(beta), R, S, float(self.eps),
                                               int(self.beta_iters), _lib.ptr(weights), _lib.ptr(err_w), _lib.stream_ptr()), "sdfb200_volsdf_step")
            total_iters += 1
            not_converge = bool(beta.max() > beta0)  # the reference's own host-side convergence test (:659)
            if not_converge and total_iters < self.max_total_iters:
                new_samples = self.pdf_sampler(ray_bundle, ray_samples, err_w[..., None], num_samples=self.num_samples_eval)
                ray_samples, sorted_index = merge_ray_samples(ray_bundle, ray_samples, new_samples)
            else:
                ray_samples = self.pdf_sampler(ray_bundle, ray_samples, weights[..., None], num_samples=self.num_samples)
        points = None
        if return_eikonal_points:
            sampled_points = ray_samples.frustums.get_positions().reshape(-1, 3)
            idx = torch.randint(sampled_points.shape[0], (ray_samples.shape[0] * 10,)).to(sampled_points.device)
            points = sampled_points[idx]
        if self.num_samples_extra > 0:
            ray_samples_uniform = self.uniform_sampler(ray_bundle, num_samples=self.num_samples_extra)
            ray_samples, _ = merge_ray_samples(ray_bundle, ray_samples, ray_samples_uniform)
        if return_eikonal_points:
            return ray_samples, points
        return ray_samples


class NeuSSampler(Sampler):
    """ray_samplers.py:815-944."""

    def __init__(self, num_samples: int = 64, num_samples_importance: int = 64, num_samples_outside: int = 32, num_upsample_steps: int = 4,
                 base_variance: float = 64, single_jitter: bool = True) -> None:
        super().__init__()
        self.num_samples, self.num_samples_importance, self.num_samples_outside = num_samples, num_samples_importance, num_samples_outside
        self.num_upsample_steps, self.base_variance, self.single_jitter = num_upsample_steps, base_variance, single_jitter
        self.uniform_sampler = UniformSampler(single_jitter=single_jitter)
        self.pdf_sampler = PDFSampler(include_original=False, single_jitter=single_jitter, histogram_padding=1e-5)
        self.outside_sampler = LinearDisparitySampler()
        self.error_bounded_sampler = ErrorBoundedSampler()

    def generate_ray_samples(self, ray_bundle=None, sdf_fn=None, ray_samples=None):
        assert ray_bundle is not None and sdf_fn is not None
        lib = _lib.load()
        if ray_samples is None:
            ray_samples = self.uniform_sampler(ray_bundle, num_samples=self.num_samples)
        R = ray_bundle.origins.shape[0]
        sorted_index, sdf = None, None
        new_samples = ray_samples
        for it in range(self.num_upsample_steps):
            with torch.no_grad():
                new_sdf = sdf_fn(new_samples)
            sdf = _merge_gather(sdf, new_sdf, sorted_index) if sorted_index is not None else new_sdf
            eu = bins_of(ray_samples)
            S = eu.shape[1] - 1
            sdf2 = _lib.f32c(sdf[..., 0])
            weights = torch.empty(R, S, device=eu.device, dtype=torch.float32)
            _lib.check(lib.sdfb200_neus_upsample_weights(_lib.ptr(eu), _lib.ptr(sdf2), R, S, float(self.base_variance * 2**it), _lib.ptr(weights),
                                                         _lib.stream_ptr()), "sdfb200_neus_upsample_weights")
            new_samples = self.pdf_sampler(ray_bundle, ray_samples, weights[..., None], num_samples=self.num_samples_importance // self.num_upsample_steps)
            ray_samples, sorted_index = merge_ray_samples(ray_bundle, ray_samples, new_samples)
        return ray_samples

    def rendering_sdf_with_fixed_inv_s(self, ray_samples, sdf: torch.Tensor, inv_s):
        """ray_samplers.py:909-944 (kept for API parity; the sampler itself uses the fused weight kernel)."""
        prev_sdf, next_sdf = sdf[:, :-1], sdf[:, 1:]
        deltas = ray_samples.deltas[:, :-1, 0]
        mid_sdf = (prev_sdf + next_sdf) * 0.5
        cos_val = (next_sdf - prev_sdf) / (deltas + 1e-5)
        prev_cos_val = torch.cat([torch.zeros_like(cos_val[:, :1]), cos_val[:, :-1]], dim=-1)
        cos_val = torch.minimum(prev_cos_val, cos_val).clip(-1e3, 0.0)
        prev_cdf = torch.sigmoid((mid_sdf - cos_val * deltas * 0.5) * inv_s)
        next_cdf = torch.sigmoid((mid_sdf + cos_val * deltas * 0.5) * inv_s)
        return (prev_cdf - next_cdf + 1e-5) / (prev_cdf + 1e-5)


class UniSurfSampler(Sampler):
    """ray_samplers.py:947-1138."""

    def __init__(self, num_samples_interval: int = 64, num_samples_outside: int = 32, num_samples_importance: int = 32, num_marching_steps: int = 256,
                 num_secant_steps: int = 8, interval_start: float = 0.25, interval_end: float = 0.0125, interval_decay: float = 0.00005,
                 single_jitter: bool = False) -> None:
        super().__init__()
        self.num_samples_interval, self.num_samples_outside, self.num_samples_importance = num_samples_interval, num_samples_outside, num_samples_importance
        self.num_marching_steps, self.num_secant_steps = num_marching_steps, num_secant_steps
        self.interval_start, self.interval_end, self.interval_decay, self.single_jitter = interval_start, interval_end, interval_decay, single_jitter
        self.uniform_sampler = UniformSampler(single_jitter=single_jitter)
        self.outside_sampler = UniformSampler(single_jitter=single_jitter)
        self.pdf_sampler = PDFSampler(include_original=False, single_jitter=single_jitter, histogram_padding=1e-5)
        self.error_bounded_sampler = ErrorBoundedSampler()
        self._step = 0
        self.delta = self.interval_start

    def step_cb(self, step):
        self._step = step
        self.delta = max(self.interval_start * math.exp(-1 * self.interval_decay * self._step), self.interval_end)

    def generate_ray_samples(self, ray_bundle=None, occupancy_fn=None, sdf_fn=None, return_surface_points: bool = False):
        assert ray_bundle is not None and sdf_fn is not None
        lib = _lib.load()
        ray_samples = self.uniform_sampler(ray_bundle, num_samples=self.num_marching_steps)
        with torch.no_grad():
            sdf = sdf_fn(ray_samples)
        occupancy = occupancy_fn(sdf)
        weights = weights_from_alphas(occupancy)
        importance_samples = self.pdf_sampler(ray_bundle, ray_samples, weights, num_samples=self.num_samples_importance)
        ray_samples_uniform_outside = self.outside_sampler(ray_bundle, num_samples=self.num_samples_outside)
        ray_samples_uniform_importance, _ = merge_ray_samples(ray_bundle, importance_samples, ray_samples_uniform_outside)

        eu = bins_of(ray_samples)
        R, S = eu.shape[0], eu.shape[1] - 1
        dev = eu.device
        nears, fars = _lib.f32c(ray_bundle.nears.reshape(-1)), _lib.f32c(ray_bundle.fars.reshape(-1))
        z = torch.empty(R, device=dev, dtype=torch.float32)
        hit = torch.empty(R, device=dev, dtype=torch.uint8)
        n2, f2 = torch.empty_like(z), torch.empty_like(z)
        sdf2 = _lib.f32c(sdf[..., 0])
        _lib.check(lib.sdfb200_unisurf_interval(_lib.ptr(eu), _lib.ptr(sdf2), _lib.ptr(nears), _lib.ptr(fars), R, S, float(self.delta), _lib.ptr(z),
                                                _lib.ptr(hit), _lib.ptr(n2), _lib.ptr(f2), _lib.stream_ptr()), "sdfb200_unisurf_interval")
        surface_points = None
        if return_surface_points:
            mask = hit.bool()
            surface_points = ray_bundle.origins[mask] + ray_bundle.directions[mask] * z[mask][..., None]
            if surface_points.shape[0] <= 0:
                surface_points = torch.rand((1024, 3), device=dev) - 0.5
        old_n, old_f = ray_bundle.nears, ray_bundle.fars
        ray_bundle.nears, ray_bundle.fars = n2[:, None], f2[:, None]
        ray_samples_interval = self.uniform_sampler(ray_bundle, num_samples=self.num_samples_interval)
        ray_bundle.nears, ray_bundle.fars = old_n, old_f
        ray_samples = self.merge_ray_samples_in_eculidean(ray_bundle, ray_samples_interval, ray_samples_uniform_importance)
        if return_surface_points:
            return ray_samples, surface_points
        return ray_samples

    def merge_ray_samples_in_eculidean(self, ray_bundle, ray_samples_1, ray_samples_2):
        """ray_samplers.py:1095-1130: merge on euclidean starts; the merged spacing bins ARE the euclidean bins."""
        lib = _lib.load()
        a, b = bins_of(ray_samples_1), bins_of(ray_samples_2)
        R, sa, sb = a.shape[0], a.shape[1] - 1, b.shape[1] - 1
        merged = torch.empty(R, sa + sb + 1, device=a.device, dtype=torch.float32)
        _lib.check(lib.sdfb200_merge_bins(_lib.ptr(a), _lib.ptr(b), R, sa, sb, _lib.ptr(merged), None, _lib.stream_ptr()), "sdfb200_merge_bins")
        return make_ray_samples(ray_bundle, merged, merged, ray_samples_1.spacing_to_euclidean_fn)
