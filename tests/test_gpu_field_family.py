"""-m gpu: the fused tensor-core field kernel (k_field_tc) against the fp64 oracle over the whole shape family it accepts
(`fused_family` in csrc/field_tc.cu), one switch at a time from a neus-facto field, and the configurations just outside the family,
which must fall back to the generic engine and still match.  Every configuration runs at bf16x3 (the fused kernel) and at fp32 (the
exact generic engine); the two tcnn-layout configurations also at bf16.  Then the two goldens minted from the unmodified reference
that only the oracle had been pinned on (`cases.CPU_CASES`) go through the CUDA product.

Every per-sample head and every rendered quantity is held to the bound the bf16x3 tests use for the heads and depth: |cuda - fp64
oracle| within 4x the fp32 oracle's own rounding noise, with a floor of 1e-4 of the quantity's scale (normals: see the forward test).  The bench tests hold
rendered RGB and normal to 1e-4 relative instead, but their field is nearly transparent (accumulation ~1e-2).  Here the rays reach the
surface, and the fp32 oracle itself then misses that relative bound: on these rays its rendered normal is 6e-4 (torch layout) to 4e-2
(L-inf contraction) relative from the fp64 one, and its alpha-composited RGB 5e-3 relative behind the L-inf contraction, where the NeuS
alpha divides two small sigmoids."""
import pytest
import torch

from oracle import cases, render, samplers
from oracle.field import FieldSpec

from helpers import (UNBOUNDED, FieldCase, assert_heads_within_noise, assert_within_noise, build_case, launches, load_golden, make_bundle, oracle64,
                     oracle_render, rel_err, scale)

pytestmark = pytest.mark.gpu

BASE = FieldSpec(num_layers=2, num_layers_color=2, hidden_dim=256, use_grid_feature=True, log2_hashmap_size=15)

# name -> (FieldSpec changes, options of helpers.FieldCase)
FAMILY = {
    "torch": ({}, {}),
    "tcnn": ({"grid_layout": "tcnn"}, {}),             # log2T = 15, base 16: the coarse levels are dense, the fine ones hashed
    "tcnn_fp16": ({"grid_layout": "tcnn"}, {"table_dtype": "fp16"}),
    "linf": ({"contraction": "linf"}, UNBOUNDED),
    "l2": ({"contraction": "l2"}, UNBOUNDED),
    "appearance_mean": ({"use_appearance_embedding": True}, {"appearance": "mean"}),
    "appearance_train": ({"use_appearance_embedding": True}, {"appearance": "train"}),
    "appearance58_n_dot_v": ({"use_appearance_embedding": True, "appearance_embedding_dim": 58, "use_n_dot_v": True}, {"appearance": "train"}),
    "n_dot_v": ({"use_n_dot_v": True}, {}),
    "pe10": ({"position_encoding_max_degree": 10}, {}),
    "pe1": ({"position_encoding_max_degree": 1}, {}),
    "no_pe": ({"use_position_encoding": False}, {}),
    "levels8": ({"num_levels": 8}, {}),
    "mask5": ({}, {"mask_level": 5}),
    "no_grid": ({"use_grid_feature": False}, {}),
    "anneal_padding_inside_out": ({"rgb_padding": 0.05}, {"cos_anneal": 0.3, "inside_outside": True}),
}
# one step past a limit of the family: PE columns (kMaxPe = 60), the misc operand (38 + appearance <= kInK = 96), 2 features per level
OUTSIDE = {
    "pe11": ({"position_encoding_max_degree": 11}, {}),
    "appearance59": ({"use_appearance_embedding": True, "appearance_embedding_dim": 59}, {"appearance": "train"}),
    "features4": ({"hash_features_per_level": 4}, {}),
}
CONFIGS = {**FAMILY, **OUTSIDE}


class _Case(FieldCase):
    def __init__(self, name, precision):
        super().__init__(BASE, CONFIGS[name], name, precision)

    def fused(self, precision):
        return self.name in FAMILY and precision != "fp32"


def _assert_engine(case, precision, n, what):
    if case.fused(precision):
        assert n == 1, f"{case.name}/{precision}/{what}: {n} launches, the fused kernel is one"
    elif precision != "fp32":
        assert n > 1, f"{case.name}/{precision}/{what}: one launch, but the configuration is outside the fused family"


# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_forward_get_sdf_and_point_mode_match_fp64_oracle(name, precision):
    import sdfstudio_b200 as sb

    c = _Case(name, precision)
    o, d, cam, rs = c.samples(32)
    tag = f"{name}/{precision}"
    with torch.no_grad():
        _assert_engine(c, precision, launches(lambda: c.field(rs, return_alphas=True, return_occupancy=True)), "forward")
        _assert_engine(c, precision, launches(lambda: c.field.get_sdf(rs)), "get_sdf")
        out = c.field(rs, return_alphas=True, return_occupancy=True)
        sdf_u = c.field.get_sdf(rs)
    e32, e64, eu = c.reference(o, d, cam, rs)
    assert_heads_within_noise(sb, out, e32, e64, tag, 1e-4)
    # sdf-only mode: un-contracted start positions
    o32, o64 = c.oracle(torch.float32), c.oracle(torch.float64)
    s32, s64 = o32.get_sdf(o, d, eu[:, :-1]), o64.get_sdf(o.double(), d.double(), eu[:, :-1].double())
    assert_within_noise(sdf_u[..., 0], s32, s64, f"{tag}/get_sdf", factor=4.0, floor=1e-4 * scale(s64))
    # point mode: gradient() with and without the contraction (points well outside the unit ball when the field contracts)
    pts, _ = c.points()
    for skip in (False, True):
        with torch.no_grad():
            gp = c.field.gradient(pts.cuda(), skip_spatial_distortion=skip)
        g64 = o64.gradient(pts.double(), skip_spatial_distortion=skip)
        assert_within_noise(gp, o32.gradient(pts, skip_spatial_distortion=skip), g64, f"{tag}/gradient(skip={skip})", factor=4.0,
                            floor=1e-4 * scale(g64))


def _check_render(name, precision, S, from_density):
    c = _Case(name, precision)
    o, d, cam, rs = c.samples(S)
    bg = torch.ones(3, device="cuda")
    tag = f"{name}/{precision}/S={S}/{'density' if from_density else 'alpha'}"
    fused_render = c.fused(precision) and 128 % S == 0
    with torch.no_grad():
        n = launches(lambda: c.field.render(rs, bg, from_density=from_density, clip_depth=False))
        res = c.field.render(rs, bg, from_density=from_density)
    if fused_render:
        assert n == 1, f"{tag}: {n} launches, the fused render is one"
    elif precision != "fp32":
        assert n > 1, f"{tag}: one launch, but this render cannot be fused"
    e32, e64, eu = c.reference(o, d, cam, rs)
    r32, r64 = oracle_render(e32, eu, from_density), oracle_render(e64, eu.double(), from_density)
    for k in ("rgb", "depth", "normal", "accumulation", "bg_transmittance", "weights"):
        assert_within_noise(res[k], r32[k], r64[k], f"{tag}/{k}", factor=4.0, floor=1e-4 * scale(r64[k]))


@pytest.mark.parametrize("from_density", [False, True])
@pytest.mark.parametrize("S", [32, 128])             # 128: every ray spans the four 32-row chunks of a tile
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_render_matches_fp64_oracle(name, precision, S, from_density):
    _check_render(name, precision, S, from_density)


@pytest.mark.parametrize("from_density", [False, True])
def test_composed_render_of_the_default_layout(from_density):
    """S = 48 does not divide the 128-point tile: the fused field call is followed by the compositing kernels"""
    _check_render("tcnn", "bf16x3", 48, from_density)


@pytest.mark.parametrize("name", ["tcnn", "tcnn_fp16"])
def test_tcnn_layout_fast_mode(name):
    """precision='bf16' runs the single-pass instantiation of the tcnn layout: held to the fast mode's bounds"""
    import sdfstudio_b200 as sb

    c = _Case(name, "bf16")
    o, d, cam, rs = c.samples(32)
    bg = torch.ones(3, device="cuda")
    H = sb.FieldHeadNames
    with torch.no_grad():
        assert launches(lambda: c.field(rs, return_alphas=True, return_occupancy=True)) == 1
        assert launches(lambda: c.field.render(rs, bg, clip_depth=False)) == 1
        out = c.field(rs, return_alphas=True, return_occupancy=True)
        res = c.field.render(rs, bg)
    _, e64, eu = c.reference(o, d, cam, rs)
    # bf16 rounds the MLP's operands, so its sdf error does not shrink where the sdf crosses zero: relative above |sdf| = 0.1
    assert rel_err(out[H.SDF], e64["sdf"], 1e-1) < 2e-2
    assert float((out[H.RGB].cpu().double() - e64["rgb"]).abs().max()) < 2e-2
    mse = float(((res["rgb"].cpu().double() - oracle_render(e64, eu.double(), False)["rgb"]) ** 2).mean())
    psnr = -10.0 * torch.log10(torch.tensor(mse)).item()
    assert psnr > 55.0, f"{name}: fast-mode PSNR vs the fp64 oracle {psnr:.1f} dB"


# ----------------------------------------------------------------------------------------------------------------
# the goldens minted from the unmodified reference for neusfacto_l2 (L2 contraction, unbounded far plane) and mixed_heads (128 / 192 / 96-wide
# layers, reflections + n.v, appearance, F = 4, lindisp spacing)
# ----------------------------------------------------------------------------------------------------------------
def _run_golden_case(name, precision):
    import sdfstudio_b200 as sb

    G = load_golden(name)
    spec, kw, o, d, cam, nears, fars, oracle, field = build_case(name, precision=precision)
    rs = sb.SpacedSampler(kw["spacing"], None, num_samples=kw["S"]).eval()(make_bundle(o, d, cam, nears, fars))
    assert torch.equal(sb.rays.spacing_bins_of(rs).cpu(), G["spacing_bins"])  # bit-exact bin edges
    assert torch.equal(sb.rays.bins_of(rs).cpu(), G["euclid_bins"])
    with torch.no_grad():
        out = field(rs, return_alphas=True, return_occupancy=True)
    o64 = oracle64(spec, oracle.p, kw)
    eu = G["euclid_bins"].double()
    e64 = o64.get_outputs(o.double(), d.double(), eu[:, :-1], eu[:, 1:] - eu[:, :-1], cam, return_alphas=True, return_occupancy=True)
    return sb, G, spec, o, d, cam, rs, field, out, o64, e64


@pytest.mark.parametrize("name", list(cases.CPU_CASES))
def test_oracle_only_golden_on_the_exact_engine(name):
    """the checks of test_field_matches_reference_golden, at fp32"""
    sb, G, spec, o, d, cam, rs, field, out, o64, e64 = _run_golden_case(name, "fp32")
    H = sb.FieldHeadNames

    def assert_rel(a, b, floor=1e-3, what=""):
        e = rel_err(a, b, floor)
        assert e <= 1e-4, f"{name}/{what}: rel err {e:.3e}"

    assert_rel(out[H.SDF], G["sdf"], what="sdf")
    assert_rel(out[H.DENSITY], G["density"], floor=1e-2, what="density")
    assert_rel(out["points_norm"], G["points_norm"], what="points_norm")
    assert_rel(out[H.OCCUPANCY], G["occupancy"], floor=1e-2, what="occupancy")
    assert_within_noise(out[H.GRADIENT], G["gradients"], e64["gradients"], f"{name}/gradients")
    assert_within_noise(out[H.NORMAL], G["normals"], e64["normals"], f"{name}/normals")
    if spec.contraction:
        # unbounded far plane: the NeuS alpha of the long far bins divides two small sigmoids, and the reference's own fp32 rgb / alpha
        # are 1.7e-4 / 7.6e-3 relative from the fp64 oracle here
        assert_within_noise(out[H.RGB], G["rgb"], e64["rgb"], f"{name}/rgb")
        assert_within_noise(out[H.ALPHA], G["alphas"], e64["alphas"], f"{name}/alpha")
    else:
        assert_rel(out[H.RGB], G["rgb"], floor=1e-2, what="rgb")
        assert_rel(out[H.ALPHA], G["alphas"], floor=1e-2, what="alpha")
    with torch.no_grad():
        assert_rel(field.get_sdf(rs), G["get_sdf"], what="get_sdf")
        assert_rel(field.forward_geonetwork(G["points"].cuda()), G["geo_points"], floor=1e-2, what="forward_geonetwork")
        gp = field.gradient(G["points"].cuda())
    assert_within_noise(gp, G["grad_points"], o64.gradient(G["points"].double()), f"{name}/gradient()")


@pytest.mark.parametrize("name", list(cases.CPU_CASES))
def test_oracle_only_golden_on_the_tensor_core_engines(name):
    """the checks of test_generic_shapes_on_the_tensor_core_engine, at bf16x3: neusfacto_l2 is a fused-family field behind the L2
    contraction, mixed_heads drives the generic tensor-core engine off 256-wide shapes"""
    sb, G, spec, o, d, cam, rs, field, out, o64, e64 = _run_golden_case(name, "bf16x3")
    H = sb.FieldHeadNames
    with torch.no_grad():
        n = launches(lambda: field(rs, return_alphas=True, return_occupancy=True))
    assert (n == 1) == (name == "neusfacto_l2"), f"{name}: {n} launches"
    for key, gk in ((H.SDF, "sdf"), (H.RGB, "rgb"), (H.ALPHA, "alphas"), (H.DENSITY, "density"), (H.GRADIENT, "gradients"), (H.NORMAL, "normals")):
        assert_within_noise(out[key], G[gk], e64[gk], f"{name}/{gk}", factor=4.0, floor=3e-4 * scale(e64[gk]))
    # rendered RGB against the reference's own fp32 render (7e-4 relative from the fp64 one for neusfacto_l2, see above)
    w = rs.get_weights_from_alphas(out[H.ALPHA])
    img = sb.render_all(w, out[H.RGB], out[H.NORMAL], rs, torch.ones(3, device="cuda"))
    ow, _ = samplers.weights_from_alphas(e64["alphas"][..., 0])
    orgb = render.render_rgb(e64["rgb"], ow[..., None], torch.ones(3, dtype=torch.float64))
    gw, _ = samplers.weights_from_alphas(G["alphas"][..., 0])
    grgb = render.render_rgb(G["rgb"], gw[..., None], torch.ones(3))
    assert_within_noise(img["rgb"], grgb, orgb, f"{name}/rendered rgb", factor=4.0, floor=1e-4)
