"""The generic field engine (csrc/field_simt.cu: the exact-fp32 GEMMs at precision 'fp32', the tensor-core Linear of tc_linear.cu at bf16x3 /
bf16) against the fp64 oracle over the shapes it accepts: a table of configurations one switch away from a base that no precision sends to
the fused kernel, the way test_gpu_field_family.py walks the fused kernel's family.

Every configuration runs at fp32 and bf16x3: the per-sample heads of get_outputs, the point-mode and narrow-output calls (forward_geonetwork,
get_sdf, get_density, get_alpha, gradient) and render().  Each quantity is held to 4x the fp32 oracle's own rounding noise from the fp64 one,
with a floor of 1e-4 (fp32) / 3e-4 (bf16x3) of the quantity's scale, the bounds of test_generic_shapes_on_the_tensor_core_engine.  bf16 is held
to the fast mode's bounds of test_tcnn_layout_fast_mode, or to twice the error of the oracle run on bf16-rounded operands where that alone
misses them.  The launch counter pins the engine: never the fused kernel; tensor-core GEMMs (one weight pack per GEMM chunk) at bf16x3 /
bf16; the exact GEMMs, and so fp32's bits, whenever the field uses numerical gradients.

The descriptor-against-weights checks at the end run without a GPU."""
import contextlib
import math

import pytest
import torch

from oracle import cases
from oracle.field import FieldSpec

from helpers import (POINTS, RAY_SEED, UNBOUNDED, FieldCase, assert_heads_within_noise, assert_straddles_chunk, assert_within_noise, launches,
                     make_bundle, oracle_render, rel_err, scale)

gpu = pytest.mark.gpu

# in_dim = 3 + 36 (PE) + 32 (grid) = 71: a layer feeding the skip concat has a 57-wide output, a multiple of no tile
BASE = FieldSpec(num_layers=2, hidden_dim=128, geo_feat_dim=64, num_layers_color=2, hidden_dim_color=128, use_grid_feature=True, log2_hashmap_size=15)
NUMGRAD = dict(num_grad_delta=0.002)
FLOOR = {"fp32": 1e-4, "bf16x3": 3e-4}

# name -> (FieldSpec changes, options of helpers.FieldCase).  The reference's skip concat (skip_in = [4]) feeds geo layer 4, which exists
# from num_layers = 4 on.
CONFIGS = {
    "base": ({}, {}),
    # depth
    "layers0": ({"num_layers": 0}, {}),                 # one geo layer: d sdf / d inputs is row 0 of W0
    "layers1": ({"num_layers": 1}, {}),                 # two: the reverse sweep is its seed and layer 0
    "layers4": ({"num_layers": 4}, {}),                 # the skip concat feeds the last layer: the seed runs the skip copy
    "layers5": ({"num_layers": 5}, {}),                 # the skip is the first step of the reverse loop
    "layers11": ({"num_layers": 11, "hidden_dim": 96}, {}),   # the 12-layer maximum
    # width
    "hidden100_layers5": ({"num_layers": 5, "hidden_dim": 100}, {}),   # softplus(0) padding columns, overwritten by the skip copy
    "hidden320": ({"hidden_dim": 320}, {}),             # N-chunked and K-accumulated tensor-core GEMMs
    "geo_feat15": ({"geo_feat_dim": 15}, {}),
    "geo_feat300": ({"geo_feat_dim": 300}, {}),         # a 301-wide last geo layer, a 365-wide colour input
    "hidden_color24": ({"hidden_dim_color": 24}, {}),
    "color_layers0": ({"num_layers_color": 0}, {}),     # one colour layer, no ReLU
    "color_layers4": ({"num_layers_color": 4}, {}),
    # heads
    "diffuse": ({"use_diffuse_color": True}, {}),       # specular 0.5 * rgb
    "diffuse_tint": ({"use_diffuse_color": True, "use_specular_tint": True}, {}),
    "tint_only": ({"use_specular_tint": True}, {}),     # the reference computes the tint and ignores it
    "reflections": ({"use_reflections": True}, {}),
    "n_dot_v": ({"use_n_dot_v": True}, {}),
    "off_axis": ({"off_axis": True}, {}),
    "off_axis_no_grid": ({"off_axis": True, "use_grid_feature": False}, {}),
    "diffuse_appearance_n_dot_v": ({"use_diffuse_color": True, "use_appearance_embedding": True, "use_n_dot_v": True}, {"appearance": "train"}),
    # inputs
    "no_grid": ({"use_grid_feature": False}, {}),
    "no_pe": ({"use_position_encoding": False}, {}),
    "pe1": ({"position_encoding_max_degree": 1}, {}),
    "off_axis_pe10": ({"off_axis": True, "position_encoding_max_degree": 10}, {}),   # in_pad = 464
    "features1": ({"hash_features_per_level": 1}, {}),
    "features4": ({"hash_features_per_level": 4}, {}),
    "features8": ({"hash_features_per_level": 8}, {}),
    "tcnn": ({"grid_layout": "tcnn"}, {}),
    "tcnn_fp16": ({"grid_layout": "tcnn"}, {"table_dtype": "fp16"}),
    "mask5": ({}, {"mask_level": 5}),
    "linear": ({"hash_smoothstep": False}, {}),
    # space
    "linf": ({"contraction": "linf"}, UNBOUNDED),
    "l2": ({"contraction": "l2"}, UNBOUNDED),
    # appearance
    "appearance_mean": ({"use_appearance_embedding": True}, {"appearance": "mean"}),
    "appearance_train": ({"use_appearance_embedding": True}, {"appearance": "train"}),
    # weights
    "no_weight_norm": ({"weight_norm": False}, {}),
    # numerical gradients
    "numgrad": ({"use_numerical_gradients": True}, NUMGRAD),
    "numgrad_layers5": ({"use_numerical_gradients": True, "num_layers": 5}, NUMGRAD),
    "numgrad_features8_mask5": ({"use_numerical_gradients": True, "hash_features_per_level": 8}, {**NUMGRAD, "mask_level": 5}),
    # NeuS knobs
    "anneal_padding_inside_out": ({"rgb_padding": 0.05}, {"cos_anneal": 0.3, "inside_outside": True}),
}
ANALYTIC = [n for n, (ch, _) in CONFIGS.items() if not ch.get("use_numerical_gradients")]


class _Case(FieldCase):
    def __init__(self, name, precision, device="cuda"):
        super().__init__(BASE, CONFIGS[name], name, precision, device)

    @property
    def numerical(self):
        return self.spec.use_numerical_gradients


def _calls(field, rs, grad_pts, geo_pts):
    """every inference entry point of the field on the same rays / points"""
    gp, xp = grad_pts.cuda(), geo_pts.cuda()
    return {
        "get_outputs": lambda: field(rs, return_alphas=True, return_occupancy=True),
        "forward_geonetwork": lambda: field.forward_geonetwork(xp),
        "get_sdf": lambda: field.get_sdf(rs),
        "get_density": lambda: field.get_density(rs),
        "get_alpha": lambda: field.get_alpha(rs),
        "gradient": lambda: field.gradient(gp),
        "gradient_skip": lambda: field.gradient(gp, skip_spatial_distortion=True),
    }


def _tensors(x):
    if isinstance(x, dict):
        return [v for v in x.values() if v is not None]
    return list(x) if isinstance(x, tuple) else [x]


def _at_starts(of, o, d, eu):
    """what get_sdf / get_density / get_alpha (no sdf or gradients passed) compute: forward_geonetwork at the un-contracted start positions,
    and NeuS alpha from autograd's gradient there (sdf_field.py:412-525)"""
    dt = of.dtype
    e, o, d = eu.to(dt), o.to(dt), d.to(dt)
    R, S = e.shape[0], e.shape[1] - 1
    pos = (o[:, None, :] + d[:, None, :] * e[:, :-1, None]).reshape(-1, 3)
    with torch.enable_grad():
        x = pos.clone().requires_grad_(True)
        h = of.forward_geonetwork(x)
        g = torch.autograd.grad(h[:, :1], x, torch.ones_like(h[:, :1]))[0]
    sdf, geo = h[:, :1].detach().view(R, S, 1), h[:, 1:].detach().view(R, S, -1)
    alpha = of.get_alpha(d[:, None, :].expand(R, S, 3), (e[:, 1:] - e[:, :-1])[..., None], sdf, g.view(R, S, 3))
    return {"sdf": sdf, "density": of.laplace_density(sdf), "geo_feature": geo, "alpha": alpha}


_POINT_REF = {}


def _point_reference(case, o, d, eu, grad_pts, geo_pts):
    hit = _POINT_REF.get(case.name)
    if hit is not None and torch.equal(hit[0], eu):
        return hit[1]
    res = {}
    for dt in (torch.float32, torch.float64):
        of = case.oracle(dt)
        r = _at_starts(of, o, d, eu)
        r["geo_points"] = of.forward_geonetwork(geo_pts.to(dt))
        for skip in (False, True):
            r[f"gradient(skip={skip})"] = of.gradient(grad_pts.to(dt), skip_spatial_distortion=skip)
        res[dt] = r
    _POINT_REF[case.name] = (eu, res)
    return res


def _check_engine(c, counts, got, rs, grad_pts, geo_pts):
    """never the fused kernel; against the same field at fp32: more launches (the tensor-core GEMMs' weight packs), or with numerical
    gradients the same launches and the same bits"""
    tag = f"{c.name}/{c.precision}"
    for k, n in counts.items():
        assert n > 1, f"{tag}/{k}: one launch, but the configuration is outside the fused kernel's family"
    if c.precision == "fp32":
        return
    calls32 = _calls(_Case(c.name, "fp32").field, rs, grad_pts, geo_pts)
    with torch.no_grad():
        for k, fn in calls32.items():
            n32 = launches(fn)
            if not c.numerical:
                assert counts[k] > n32, f"{tag}/{k}: {counts[k]} launches, fp32 {n32}: the GEMMs did not run on the tensor cores"
                continue
            assert counts[k] == n32, f"{tag}/{k}: {counts[k]} launches, fp32 {n32}: numerical gradients keep the exact engine"
            ours, exact = _tensors(got[k]), _tensors(fn())
            assert len(ours) == len(exact)
            for i, (a, b) in enumerate(zip(ours, exact)):
                assert torch.equal(a, b), f"{tag}/{k}: output {i} differs from fp32's"


# ----------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_outputs_and_point_mode_match_fp64_oracle(name, precision):
    import sdfstudio_b200 as sb

    c = _Case(name, precision)
    o, d, cam, rs = c.samples(32)
    grad_pts, geo_pts = c.points()
    calls = _calls(c.field, rs, grad_pts, geo_pts)
    with torch.no_grad():
        counts = {k: launches(fn) for k, fn in calls.items()}
        got = {k: fn() for k, fn in calls.items()}
    _check_engine(c, counts, got, rs, grad_pts, geo_pts)

    tag, fl = f"{name}/{precision}", FLOOR[precision]

    def close(cu, r32, r64, what):
        assert_within_noise(cu, r32, r64, f"{tag}/{what}", factor=4.0, floor=fl * scale(r64))

    # get_outputs: every per-sample head
    e32, e64, eu = c.reference(o, d, cam, rs)
    out = got["get_outputs"]
    assert_heads_within_noise(sb, out, e32, e64, tag, fl)
    if c.numerical:
        close(out["sampled_sdf"], e32["sampled_sdf"], e64["sampled_sdf"], "sampled_sdf")
    else:
        assert out["sampled_sdf"] is None

    # point mode and the narrow output sets
    p = _point_reference(c, o, d, eu, grad_pts, geo_pts)
    p32, p64 = p[torch.float32], p[torch.float64]
    geo = got["forward_geonetwork"]
    assert geo.shape == (POINTS, 1 + c.spec.geo_feat_dim)
    close(geo[:, :1], p32["geo_points"][:, :1], p64["geo_points"][:, :1], "forward_geonetwork sdf")
    close(geo[:, 1:], p32["geo_points"][:, 1:], p64["geo_points"][:, 1:], "forward_geonetwork geo_feature")
    close(got["get_sdf"], p32["sdf"], p64["sdf"], "get_sdf")
    dens, gfeat = got["get_density"]
    assert gfeat.shape == p64["geo_feature"].shape
    close(dens, p32["density"], p64["density"], "get_density density")
    close(gfeat, p32["geo_feature"], p64["geo_feature"], "get_density geo_feature")
    close(got["get_alpha"], p32["alpha"], p64["alpha"], "get_alpha")
    for skip in (False, True):
        k = f"gradient(skip={skip})"
        close(got["gradient_skip" if skip else "gradient"], p32[k], p64[k], k)


@gpu
@pytest.mark.parametrize("S", [32, 48])             # 48: rays do not tile the 128-row GEMM tiles
@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_render_matches_fp64_oracle(name, precision, S):
    c = _Case(name, precision)
    o, d, cam, rs = c.samples(S)
    bg = torch.ones(3, device="cuda")
    e32, e64, eu = c.reference(o, d, cam, rs)
    for from_density in (False, True):
        tag = f"{name}/{precision}/S={S}/{'density' if from_density else 'alpha'}"
        with torch.no_grad():
            n = launches(lambda: c.field.render(rs, bg, from_density=from_density, clip_depth=False))
            res = c.field.render(rs, bg, from_density=from_density)
        assert n > 1, f"{tag}: one launch, but the configuration is outside the fused kernel's family"
        r32, r64 = oracle_render(e32, eu, from_density), oracle_render(e64, eu.double(), from_density)
        for k in ("rgb", "depth", "normal", "accumulation", "bg_transmittance", "weights"):
            assert_within_noise(res[k], r32[k], r64[k], f"{tag}/{k}", factor=4.0, floor=FLOOR[precision] * scale(r64[k]))


@contextlib.contextmanager
def _bf16_operands():
    """every Linear of the oracle on bf16-rounded operands with fp32 accumulation: what a one-plane bf16 GEMM engine computes at best"""
    linear = torch.nn.functional.linear
    torch.nn.functional.linear = lambda x, w, b=None: linear(x.bfloat16().float(), w.bfloat16().float(), b)
    try:
        yield
    finally:
        torch.nn.functional.linear = linear


def _fast_mode_errors(sdf, rgb, rendered_rgb, e64, eu):
    """sdf error relative above |sdf| = 0.1 (bf16 rounds the MLP's operands, so its sdf error does not shrink where the sdf crosses zero),
    absolute per-sample rgb error, and the PSNR of the rendered rgb, against the fp64 oracle's outputs `e64` on the bins `eu`"""
    mse = float(((rendered_rgb.detach().double().cpu() - oracle_render(e64, eu.double(), False)["rgb"]) ** 2).mean())
    return rel_err(sdf, e64["sdf"], 1e-1), float((rgb.detach().double().cpu() - e64["rgb"]).abs().max()), -10.0 * math.log10(mse)


@gpu
@pytest.mark.parametrize("name", ANALYTIC)
def test_single_pass_bf16_within_fast_mode_bounds(name):
    """precision='bf16' (one bf16 plane per GEMM operand) on the generic engine, held to the bounds of test_tcnn_layout_fast_mode (sdf 2e-2
    relative, rgb 2e-2, rendered PSNR 55 dB), or to twice the error of the oracle evaluated with bf16 operands where that alone misses them.
    The rounding of the operands is all of it: measured on an H100, the base's sdf error is 2.1e-2 (emulated 2.1e-2), the 12-layer net's
    7.3e-2 (7.9e-2), five layers with the skip feeding the last one 5.4e-2 (6.2e-2), and the rgb of off-axis PE 10 0.105 (0.105)."""
    import sdfstudio_b200 as sb

    c, c32 = _Case(name, "bf16"), _Case(name, "fp32")
    o, d, cam, rs = c.samples(32)
    bg = torch.ones(3, device="cuda")
    H = sb.FieldHeadNames
    fwd = lambda f: f(rs, return_alphas=True, return_occupancy=True)   # noqa: E731
    with torch.no_grad():
        n, n32 = launches(lambda: fwd(c.field)), launches(lambda: fwd(c32.field))
        out = fwd(c.field)
        res = c.field.render(rs, bg)
    assert n > n32 > 1, f"{name}: {n} launches at bf16, {n32} at fp32: the GEMMs did not run on the tensor cores"
    _, e64, eu = c.reference(o, d, cam, rs)
    e = eu.float()
    with _bf16_operands():
        eb = c.oracle(torch.float32).get_outputs(o, d, e[:, :-1], e[:, 1:] - e[:, :-1], cam, return_alphas=True, return_occupancy=True)
    emul = _fast_mode_errors(eb["sdf"], eb["rgb"], oracle_render(eb, e, False)["rgb"], e64, eu)
    e_sdf, e_rgb, psnr = _fast_mode_errors(out[H.SDF], out[H.RGB], res["rgb"], e64, eu)
    assert e_sdf < max(2e-2, 2 * emul[0]), f"{name}: bf16 sdf rel err {e_sdf:.3e} (bf16 operands alone: {emul[0]:.3e})"
    assert e_rgb < max(2e-2, 2 * emul[1]), f"{name}: bf16 rgb err {e_rgb:.3e} (bf16 operands alone: {emul[1]:.3e})"
    assert psnr > min(55.0, emul[2] - 20 * math.log10(2)), f"{name}: bf16 rendered PSNR {psnr:.1f} dB (bf16 operands alone: {emul[2]:.1f} dB)"


CHUNK_CALL = (1500, 50, slice(1330, 1380))    # rays, samples per ray, the rays compared: 75 000 points


@gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
@pytest.mark.parametrize("name", ["hidden320", "numgrad"])
def test_chunk_boundary_does_not_show(name, precision):
    """more points than one pass of the generic engine holds, with a ray straddling the first chunk boundary: every head of the rays around
    it is bit-equal to a separate call on those rays alone"""
    import sdfstudio_b200 as sb

    R, S, sl = CHUNK_CALL
    assert_straddles_chunk(R, S, sl)
    c = _Case(name, precision)
    o, d, cam, rs = c.samples(S, R=R, seed=123)
    nears, fars = torch.full((R, 1), 0.5), torch.full((R, 1), 4.5)
    small_rs = sb.SpacedSampler("uniform", None, num_samples=S).eval()(make_bundle(o[sl], d[sl], cam[sl], nears[sl], fars[sl]))
    with torch.no_grad():
        big = c.field(rs, return_alphas=True, return_occupancy=True)
        small = c.field(small_rs, return_alphas=True, return_occupancy=True)
    assert (big["sampled_sdf"] is not None) == c.numerical
    for k, v in small.items():
        if v is not None:
            assert torch.equal(big[k][sl], v), f"{name}/{precision}/{k}"


# ----------------------------------------------------------------------------------------------------------------
# the descriptor against the module's weights (host side, no GPU)
# ----------------------------------------------------------------------------------------------------------------
AABB = [[-1.0, -1, -1], [1, 1, 1]]


def test_every_configuration_is_a_descriptor_the_library_plans():
    from sdfstudio_b200 import _lib

    lib = _lib.load()
    for name in CONFIGS:
        d = _Case(name, "bf16x3", device="cpu").field._field_desc()
        assert lib.sdfb200_field_packed_bytes(d) > 0, name
        assert lib.sdfb200_field_workspace_bytes(d, POINTS) > 0, name


def test_weights_the_descriptor_does_not_describe_are_refused():
    """num_layers = 3: the reference's skip_in = [4] narrows the last geo layer to 1 + geo_feat_dim - in_dim rows ([186, 128] here), but the
    descriptor has no skip below 5 geo layers and reads it as [257, 128]"""
    import sdfstudio_b200 as sb

    f = sb.SDFField(sb.SDFFieldConfig(num_layers=3, hidden_dim=128, geo_feat_dim=256), torch.tensor(AABB), 4)
    assert tuple(f.glin3.weight_v.shape) == (186, 128)
    with pytest.raises(ValueError, match=r"glin3\.weight_v is \[186, 128\].*\[257, 128\]"):
        f._field_desc()
    # a layer replaced by one of another shape, on a field without weight norm (colour dims [129, 128, 128, 3])
    f = sb.SDFField(sb.SDFFieldConfig(num_layers=2, hidden_dim=128, geo_feat_dim=64, num_layers_color=2, hidden_dim_color=128, weight_norm=False),
                    torch.tensor(AABB), 4)
    f._field_desc()
    f.clin1 = torch.nn.Linear(128, 100)
    with pytest.raises(ValueError, match=r"clin1\.weight is \[100, 128\].*\[128, 128\]"):
        f._field_desc()


def test_more_layers_than_the_engine_holds_is_not_implemented():
    import sdfstudio_b200 as sb

    sb.SDFField(sb.SDFFieldConfig(num_layers=11, hidden_dim=96), torch.tensor(AABB), 4)._field_desc()   # 12 geo layers: the maximum
    with pytest.raises(NotImplementedError):
        sb.SDFField(sb.SDFFieldConfig(num_layers=12, hidden_dim=96), torch.tensor(AABB), 4)._field_desc()


def test_chunk_call_straddles_the_library_chunk():
    """the chunk test's rays still straddle the generic engine's chunk boundary as the library sizes it (checked without a GPU)"""
    assert_straddles_chunk(*CHUNK_CALL)


class _NoDevice:
    """stands in for the library: any use of it fails on the host"""

    def __getattr__(self, name):
        raise AssertionError(f"{name} reached with a field the descriptor does not describe")


def test_refused_field_reaches_no_library_call(monkeypatch):
    """the num_layers = 3 field: every entry point raises before it packs a weight or calls into the library.  The field stays on the host,
    the library is replaced by one that fails on any use and packing fails outright, so a regression fails here without touching a device."""
    import sdfstudio_b200 as sb
    from sdfstudio_b200 import _lib

    def no_packing(self, desc):
        raise AssertionError("weights packed for a field the descriptor does not describe")

    monkeypatch.setattr(_lib, "load", lambda: _NoDevice())
    monkeypatch.setattr(_lib, "require_cuda", lambda dev, what: None)
    monkeypatch.setattr(sb.SDFField, "_packed_weights", no_packing)
    f = sb.SDFField(sb.SDFFieldConfig(num_layers=3, hidden_dim=128, geo_feat_dim=256), torch.tensor(AABB), 4).eval()
    R, S = 4, 8
    o, d, cam = cases.synthetic_rays(R, RAY_SEED)
    bins = torch.linspace(0.5, 4.5, S + 1).expand(R, S + 1).contiguous()

    class _Frustums:                    # the fields of a RaySamples the entry points read
        origins, directions = o[:, None].expand(R, S, 3), d[:, None].expand(R, S, 3)
        starts, ends = bins[:, :-1, None], bins[:, 1:, None]
        shape = (R, S)

    class _Samples:
        frustums, camera_indices, _euclid_bins = _Frustums, cam.view(R, 1), bins

    pts = torch.zeros(16, 3)
    with torch.no_grad():
        for call in (lambda: f(_Samples), lambda: f.get_sdf(_Samples), lambda: f.get_density(_Samples), lambda: f.get_alpha(_Samples),
                     lambda: f.forward_geonetwork(pts), lambda: f.gradient(pts), lambda: f.render(_Samples, torch.ones(3))):
            with pytest.raises(ValueError, match="glin3"):
                call()
    assert f._packed is None
