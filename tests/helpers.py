"""Shared helpers for the parity tests: build the *product* SDFField for a seeded oracle case."""
import functools
import os

import numpy as np
import torch

from oracle import cases, render, samplers
from oracle.field import FieldSpec, OracleField, folded_weight, init_params

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_golden(name, device="cpu"):
    return {k: torch.from_numpy(v).to(device) for k, v in np.load(os.path.join(GOLDEN_DIR, name + ".npz")).items()}


def load_train_golden():
    """tests/golden/samplers_train.{npz,json} (oracle/make_golden_samplers_train.py): (arrays, meta).  meta["draws"][run] lists the
    reference's random draws of that run in order; ``train_draws`` returns the drawn tensors."""
    import json

    with open(os.path.join(GOLDEN_DIR, "samplers_train.json")) as f:
        meta = json.load(f)
    return load_golden("samplers_train"), meta


def train_draws(G, meta, run):
    return [G[f"{run}.draw{k}"] for k in range(len(meta["draws"][run]))]


def train_case_inputs():
    """The golden's rays (the first TRAIN_SAMPLER_RAYS of cases.TRAIN_SAMPLER_CASE) and the fp32 oracle field of that case."""
    spec, kw, o, d, cam, nears, fars = cases.case_inputs(cases.TRAIN_SAMPLER_CASE)
    n = cases.TRAIN_SAMPLER_RAYS
    oracle = OracleField(spec, init_params(spec, **cases.init_kwargs(kw)))
    return spec, kw, o[:n], d[:n], cam[:n], nears[:n], fars[:n], oracle


def product_field(spec: FieldSpec, params, kw, device="cuda", precision="fp32", table_dtype="fp32"):
    """sdfstudio_b200.SDFField with the oracle's seeded parameters loaded (names match the reference state_dict)."""
    import sdfstudio_b200 as sb

    cfg = sb.SDFFieldConfig(
        num_layers=spec.num_layers, hidden_dim=spec.hidden_dim, geo_feat_dim=spec.geo_feat_dim, num_layers_color=spec.num_layers_color,
        hidden_dim_color=spec.hidden_dim_color, appearance_embedding_dim=spec.appearance_embedding_dim,
        use_appearance_embedding=spec.use_appearance_embedding, bias=kw.get("bias", 0.5), inside_outside=kw.get("inside_outside", False),
        use_grid_feature=spec.use_grid_feature, weight_norm=spec.weight_norm, beta_init=kw.get("beta_init", 0.3), position_encoding_max_degree=spec.position_encoding_max_degree,
        use_diffuse_color=spec.use_diffuse_color, use_specular_tint=spec.use_specular_tint, use_reflections=spec.use_reflections,
        use_n_dot_v=spec.use_n_dot_v, rgb_padding=spec.rgb_padding, off_axis=spec.off_axis, use_numerical_gradients=spec.use_numerical_gradients,
        num_levels=spec.num_levels, max_res=spec.max_res, base_res=spec.base_res, log2_hashmap_size=spec.log2_hashmap_size,
        hash_features_per_level=spec.hash_features_per_level, hash_smoothstep=spec.hash_smoothstep, use_position_encoding=spec.use_position_encoding,
        grid_layout=spec.grid_layout, precision=precision, table_dtype=table_dtype,
    )  # fmt: skip

    class _Contraction:  # duck-typed SceneContraction (only `.order` is read)
        def __init__(self, order):
            self.order = order

    distortion = None
    if spec.contraction is not None:
        distortion = _Contraction(float("inf") if spec.contraction == "linf" else None)
    f = sb.SDFField(cfg, torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), num_images=49, spatial_distortion=distortion)
    sd = {}
    for k, v in params.items():
        if k == "hash_table":
            if spec.grid_layout == "torch":
                sd["encoding.hash_table"] = v
            else:
                sd["encoding.params"] = v.reshape(-1)
        else:
            sd[k] = v
    missing, unexpected = f.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert all(m.startswith("encoding") or m == "aabb" for m in missing), missing
    f = f.to(device).eval()
    if "mask_level" in kw:
        f.update_mask(kw["mask_level"])
    if "num_grad_delta" in kw:
        f.set_numerical_gradients_delta(kw["num_grad_delta"])
    return f


def build_case(name, device="cuda", precision="fp32", table_dtype="fp32"):
    spec, kw, o, d, cam, nears, fars = cases.case_inputs(name)
    params = init_params(spec, **cases.init_kwargs(kw))
    if table_dtype == "fp16" and "hash_table" in params:
        params["hash_table"] = params["hash_table"].half().float()   # the model IS the fp16-representable table (tcnn semantics)
    oracle = OracleField(spec, params)
    if "mask_level" in kw:
        oracle.update_mask(kw["mask_level"])
    if "num_grad_delta" in kw:
        oracle.numerical_gradients_delta = kw["num_grad_delta"]
    field = product_field(spec, params, kw, device, precision, table_dtype)
    return spec, kw, o, d, cam, nears, fars, oracle, field


@functools.lru_cache(maxsize=None)
def generic_chunk_points():
    """Points per pass of the generic field engine (kChunkPoints, csrc/field_plan.h), read off the library: the workspace of a generic-engine
    call grows with the point count up to one chunk and then stays (every pass reuses it).  Host logic only."""
    import sdfstudio_b200 as sb

    lib = sb._lib.load()
    d = sb.SDFField(sb.SDFFieldConfig(precision="fp32"), torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), 1)._field_desc()
    lo, hi = 1, 1 << 24
    top = lib.sdfb200_field_workspace_bytes(d, hi)
    assert top > 0 and lib.sdfb200_field_workspace_bytes(d, hi // 2) == top, "the workspace does not saturate: no chunked passes"
    while lo < hi:                      # the first point count whose workspace is the whole chunk's
        mid = (lo + hi) // 2
        lo, hi = (lo, mid) if lib.sdfb200_field_workspace_bytes(d, mid) == top else (mid + 1, hi)
    return lo


def assert_straddles_chunk(R, S, sl):
    """R rays of S samples cross the first chunk boundary of the generic engine, and the rays `sl` hold one that straddles it"""
    chunk = generic_chunk_points()
    assert R * S > chunk, f"{R * S} points fit in one {chunk}-point chunk"
    assert chunk % S != 0 and sl.start <= chunk // S < sl.stop, f"no ray of {sl} straddles the {chunk}-point chunk boundary at S = {S}"


def launches(fn):
    """library kernel launches of one call, after a first call has packed the weights"""
    from sdfstudio_b200 import _lib

    fn()
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    fn()
    torch.cuda.synchronize()
    return _lib.launch_count() - n0


def oracle_render(e, eu, from_density):
    """the renderers on the oracle's per-sample outputs `e` (OracleField.get_outputs on the euclidean bins `eu`): white background,
    expected depth"""
    ones = torch.ones(3, dtype=eu.dtype)
    if from_density:
        w, T = samplers.weights_from_density(eu[:, 1:] - eu[:, :-1], e["density"][..., 0])
    else:
        w, T = samplers.weights_from_alphas(e["alphas"][..., 0])
    w = w[..., None]
    return {"rgb": render.render_rgb(e["rgb"], w, ones), "depth": render.render_depth(w, eu[:, :-1, None], eu[:, 1:, None], "expected"),
            "normal": render.render_semantics(e["normals"], w), "accumulation": render.render_accumulation(w), "bg_transmittance": T[:, -1:],
            "weights": w}


def make_bundle(o, d, cam, nears, fars, device="cuda"):
    import sdfstudio_b200 as sb

    R = o.shape[0]
    return sb.RayBundle(origins=o.to(device), directions=d.to(device), pixel_area=torch.ones(R, 1, device=device),
                        directions_norm=torch.ones(R, 1, device=device), camera_indices=cam.view(R, 1).to(device), nears=nears.to(device),
                        fars=fars.to(device))


def rel_err(a, b, floor=1e-3):
    """max |a-b| / max(|b|, floor)"""
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float(((a - b).abs() / b.abs().clamp_min(floor)).max())


def oracle64(spec, params, kw):
    """float64 instance of the oracle: the 'exact' answer used to calibrate fp32 noise."""
    o = OracleField(spec, params, dtype=torch.float64)
    if "mask_level" in kw:
        o.update_mask(kw["mask_level"])
    if "num_grad_delta" in kw:
        o.numerical_gradients_delta = kw["num_grad_delta"]
    return o


# the fp64 parity tables (test_gpu_field_family.py, test_gpu_field_generic.py): one configuration per row, one switch from a base
# bias 0.9: the rays cross the zero level set or graze it, so the rendered accumulations spread over (0, 1) instead of all being ~0
FIELD_INIT = dict(bias=0.9, beta_init=0.3, perturb=0.02, hash_init_scale=0.05, seed=41)
RAY_SEED = 77
POINTS = 2048                                                # samples per call: 16 tiles of 128
UNBOUNDED = dict(near=0.2, far=30.0, spacing="piecewise")   # most samples lie outside the unit ball


class FieldCase:
    """One row of a configuration table: the product field at `precision` and the fp32 / fp64 oracles with the same parameters and
    switches.  `row` = (FieldSpec changes to `base`, options).  Options: table_dtype, near / far / spacing of the rays, appearance ("mean":
    eval mode with the mean embedding, "train": training mode with the per-camera rows), mask_level (update_mask), cos_anneal,
    inside_outside, num_grad_delta (the numerical-gradient step)."""

    _REF = {}

    def __init__(self, base, row, name, precision, device="cuda"):
        from dataclasses import replace

        changes, opt = row
        self.name, self.opt, self.precision = name, opt, precision
        self.spec = replace(base, **changes)
        self.kw = dict(FIELD_INIT, inside_outside=opt.get("inside_outside", False))
        for k in ("mask_level", "num_grad_delta"):
            if k in opt:
                self.kw[k] = opt[k]
        self.params = init_params(self.spec, **cases.init_kwargs(self.kw))
        if not self.spec.weight_norm:
            # a field without weight norm holds the folded weights as `{layer}.weight` (what the oracle then reads)
            for layer in [k[: -len(".weight_v")] for k in self.params if k.endswith(".weight_v")]:
                self.params[layer + ".weight"] = folded_weight(self.params, layer, True)
                del self.params[layer + ".weight_v"], self.params[layer + ".weight_g"]
        table_dtype = opt.get("table_dtype", "fp32")
        if table_dtype == "fp16" and "hash_table" in self.params:
            self.params["hash_table"] = self.params["hash_table"].half().float()   # the oracle holds the fp16-representable table
        f = product_field(self.spec, self.params, self.kw, device=device, precision=precision, table_dtype=table_dtype)
        f.set_cos_anneal_ratio(opt.get("cos_anneal", 1.0))
        if opt.get("appearance") == "mean":
            f.use_average_appearance_embedding = True
        elif opt.get("appearance") == "train":
            f.train()                                  # under no_grad: the inference kernels with the per-camera embedding rows
        self.field = f

    def oracle(self, dtype):
        o = OracleField(self.spec, self.params, dtype=dtype)
        if "mask_level" in self.kw:
            o.update_mask(self.kw["mask_level"])
        o.numerical_gradients_delta = self.kw.get("num_grad_delta", o.numerical_gradients_delta)
        o.cos_anneal_ratio = self.opt.get("cos_anneal", 1.0)
        o.use_average_appearance_embedding = self.opt.get("appearance") == "mean"
        o.training = self.opt.get("appearance") == "train"
        return o

    def samples(self, S, R=None, seed=RAY_SEED):
        """(origins, directions, camera indices, ray samples) of R rays (default: POINTS samples, or 48 rays) at S samples per ray"""
        import sdfstudio_b200 as sb

        R = R or (POINTS // S if POINTS % S == 0 else 48)
        o, d, cam = cases.synthetic_rays(R, seed)
        nears, fars = torch.full((R, 1), self.opt.get("near", 0.5)), torch.full((R, 1), self.opt.get("far", 4.5))
        rs = sb.SpacedSampler(self.opt.get("spacing", "uniform"), None, num_samples=S).eval()(make_bundle(o, d, cam, nears, fars))
        return o, d, cam, rs

    def points(self):
        """gradient() points (well outside the unit ball when the field contracts) and forward_geonetwork points"""
        g = torch.Generator().manual_seed(5)
        grad_pts = (torch.rand(200, 3, generator=g) * 2 - 1) * (4.0 if self.spec.contraction else 1.5)
        return grad_pts, (torch.rand(POINTS, 3, generator=g) * 2 - 1) * 1.5

    def reference(self, o, d, cam, rs):
        """(fp32, fp64 oracle outputs, euclidean bins) on the product's own bins: cached per configuration and S, since every precision
        samples the same bins"""
        import sdfstudio_b200 as sb

        eu = sb.rays.bins_of(rs).cpu()
        key = (repr(self.spec), repr(sorted(self.opt.items())), eu.shape[1])
        hit = FieldCase._REF.get(key)
        if hit is not None and torch.equal(hit[0], eu):
            return hit[1], hit[2], eu
        res = []
        for dt in (torch.float32, torch.float64):
            e = eu.to(dt)
            res.append(self.oracle(dt).get_outputs(o.to(dt), d.to(dt), e[:, :-1], e[:, 1:] - e[:, :-1], cam, return_alphas=True, return_occupancy=True))
        FieldCase._REF[key] = (eu, res[0], res[1])
        return res[0], res[1], eu


def scale(t):
    return float(t.abs().max())


# the rounding of one hash-grid level lookup (csrc/grid.cuh, level_prepare / encode_level), restated in fp64 for the element-wise bounds
# of the grid operator (test_gpu_grid_operator.py) and of the hash-MLP fields (test_gpu_hash_mlp.py)
def kernel_positions(x32, scales, layout):
    """[N, L, 3] fp32 positions exactly as level_prepare rounds them (CPU-checkable: torch's fp32 multiply, fma through fp64).  `scales`
    [L] fp32 are the descriptor's level scales, `layout` "torch" or "tcnn"."""
    s = scales.to(x32.device)
    if layout == "torch":
        return x32[:, None, :] * s[None, :, None]
    return (x32.double()[:, None, :] * s.double()[None, :, None] + 0.5).float()


def geometry(x32, scales, layout, smooth):
    """per (point, level, axis) in fp64: w, the magnitude of dw/dx and of d2w/dx2 ((6 + 12t) s^2).

    t = p - floor(p) is exact in fp32 except for p in (-1, 0) (points just below the grid), where floor(p) = -1 and the kernel rounds
    t (by <= u t).  dw = 6t(1 - t) then inherits 6|1 - 2t| u t from it, which its magnitude includes there."""
    p = kernel_positions(x32, scales, layout)
    t32 = p - torch.floor(p)
    t = p.double() - torch.floor(p).double()
    rounded = (t32.double() != t).double()
    s = scales.double().to(x32.device)[None, :, None]
    if smooth:
        return t * t * (3 - 2 * t), (6 * t * (1 - t) + 6 * (1 - 2 * t).abs() * t * rounded) * s, (6 + 12 * t) * s * s
    return t, torch.ones_like(t) * s, torch.zeros_like(t)


def corner_factors(w):
    """[N, L, 8, 3]: |per-axis weight factor| of corner k"""
    bits = torch.tensor([[(k >> d) & 1 for d in range(3)] for k in range(8)], device=w.device, dtype=torch.bool)
    return torch.where(bits[None, None], w[:, :, None, :], 1 - w[:, :, None, :]).abs()


def weight_mag(a):
    """|W_k| + sum of the 2-factor sub-products: the weight and the absolute rounding of each factor"""
    a0, a1, a2 = a.unbind(-1)
    return a0 * a1 * a2 + a1 * a2 + a0 * a2 + a0 * a1


def head_pairs(sb):
    """(product output key, oracle output key) of the per-sample heads of get_outputs, normals aside (see assert_heads_within_noise)"""
    H = sb.FieldHeadNames
    return ((H.SDF, "sdf"), (H.RGB, "rgb"), (H.DENSITY, "density"), (H.ALPHA, "alphas"), (H.OCCUPANCY, "occupancy"), (H.GRADIENT, "gradients"),
            ("points_norm", "points_norm"))


def assert_heads_within_noise(sb, out, e32, e64, tag, floor_rel):
    """every per-sample head of get_outputs within 4x the fp32 oracle's noise, with a floor of `floor_rel` of the quantity's scale.  A
    normal's error is its gradient's error over |grad sdf|, so normals are compared scaled by |grad sdf| under the gradients' floor (at
    |grad sdf| = 0.27 the bf16x3 gradient error, 1e-5 of the gradients' scale, is a 1.1e-4 error of the unit normal)."""
    for key, k in head_pairs(sb):
        assert_within_noise(out[key], e32[k], e64[k], f"{tag}/{k}", factor=4.0, floor=floor_rel * scale(e64[k]))
    gmag = e64["gradients"].norm(dim=-1, keepdim=True)
    n_cu, n32, n64 = (t.detach().double().cpu() * gmag for t in (out[sb.FieldHeadNames.NORMAL], e32["normals"], e64["normals"]))
    assert_within_noise(n_cu, n32, n64, f"{tag}/normals x |grad|", factor=4.0, floor=floor_rel * scale(e64["gradients"]))


def assert_within_noise(cuda, ref32, ref64, what, factor=4.0, floor=2e-6):
    """|cuda - exact| must not exceed `factor` x the reference's OWN fp32 rounding noise |ref32 - exact| (max-norm), with an
    absolute floor.  Used where the quantity is ill-conditioned in fp32 (numerical gradients, inverse-CDF sampling), so
    that a fixed relative bound would be either meaningless or unattainable by any fp32 implementation."""
    cuda, ref32, ref64 = (t.detach().double().cpu() for t in (cuda, ref32, ref64))
    noise = float((ref32 - ref64).abs().max())
    err = float((cuda - ref64).abs().max())
    bound = max(floor, factor * noise)
    assert err <= bound, f"{what}: |cuda-exact| = {err:.3e} > {bound:.3e} (reference fp32 noise {noise:.3e})"


def cdf_consistency(existing_spacing, weights, new_bins, u, hist_pad, eps=1e-5):
    """max |cdf(new_bin) - u| evaluated in float64: the forward map of PDF sampling is well conditioned even where its
    inverse (the bin position) is not."""
    w = weights.double() + hist_pad
    ws = w.sum(-1, keepdim=True)
    pad = torch.relu(eps - ws)
    w = w + pad / w.shape[-1]
    ws = ws + pad
    cdf = torch.cumsum(w / ws, -1).clamp(max=1.0)
    cdf = torch.cat([torch.zeros_like(cdf[:, :1]), cdf], -1)
    eb = existing_spacing.double()
    nb = new_bins.double()
    idx = torch.searchsorted(eb.contiguous(), nb.contiguous(), right=True).clamp(1, eb.shape[1] - 1)
    b0, b1 = torch.gather(eb, 1, idx - 1), torch.gather(eb, 1, idx)
    c0, c1 = torch.gather(cdf, 1, idx - 1), torch.gather(cdf, 1, idx)
    t = ((nb - b0) / (b1 - b0).clamp_min(1e-30)).clamp(0, 1)
    return float((c0 + t * (c1 - c0) - u.double()).abs().max())
