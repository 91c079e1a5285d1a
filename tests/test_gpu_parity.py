"""-m gpu parity tests: the CUDA path (through sdfstudio_b200's reference-shaped modules and the C-ABI) against
(1) golden vectors minted from the unmodified reference and (2) the CPU oracle on seeded inputs.
Tolerances: floating point outputs 1e-4 relative (BASELINE.json north_star); indices bit-exact."""
import pytest
import torch

from oracle import cases, hashgrid, render, samplers
from oracle.field import FieldSpec, OracleField, init_params

from helpers import assert_straddles_chunk, assert_within_noise, build_case, cdf_consistency, load_golden, make_bundle, oracle64, product_field, rel_err

pytestmark = pytest.mark.gpu
RTOL = 1e-4
FIELD_CASES = list(cases.CASES)
SAMPLER_CASES = ["neusfacto_c1", "neusfacto_c1_init", "volsdf_stock"]


def assert_rel(a, b, tol=RTOL, floor=1e-3, what=""):
    e = rel_err(a, b, floor)
    assert e <= tol, f"{what}: rel err {e:.3e} > {tol:.1e}"


# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["torch", "tcnn"])
@pytest.mark.parametrize("F,smooth", [(2, True), (2, False), (8, False), (4, True), (1, False)])
def test_grid_encode_matches_oracle(layout, F, smooth):
    import sdfstudio_b200 as sb

    L, log2T, base, maxres = 8, 12, 4, 256
    g = hashgrid.growth_factor(L, base, maxres)
    enc = sb.Encoding(3, {"otype": "HashGrid", "n_levels": L, "n_features_per_level": F, "log2_hashmap_size": log2T, "base_resolution": base,
                          "per_level_scale": g, "interpolation": "Smoothstep" if smooth else "Linear"}, layout=layout).cuda()
    gen = torch.Generator().manual_seed(7)
    x = torch.rand(4097, 3, generator=gen)
    x[:8] = torch.tensor([[0, 0, 0], [1, 1, 1], [0.5, 0.25, 0.125], [1, 0, 0.5], [0.999999, 0.5, 0.5], [1e-7, 0.3, 0.9], [0.25, 0.25, 0.25], [0.75, 1, 0]])
    table = enc.table.detach().cpu()
    table = ((torch.rand(table.shape, generator=gen) * 2 - 1) * 0.1)
    with torch.no_grad():
        enc.table.copy_(table.cuda())
    xo = x.clone().requires_grad_(True)
    if layout == "torch":
        scal = hashgrid.torch_layout_scalings(L, base, base * g ** (L - 1))
        ref = hashgrid.encode_torch_layout(xo, table.view(-1, F), scal, 1 << log2T, smooth)
    else:
        meta = hashgrid.tcnn_grid_meta(L, F, log2T, base, g)
        ref = hashgrid.encode_tcnn_layout(xo, table.view(-1, F), meta, F, smooth)
    out = enc(x.cuda())
    assert out.shape == (4097, L * F)
    torch.testing.assert_close(out.cpu(), ref.detach(), rtol=1e-5, atol=2e-7)
    # d out / d x through the dout_dx side output vs autograd of the oracle
    lib = sb._lib.load()
    o2 = torch.empty(4097, L * F, device="cuda")
    J = torch.empty(4097, L * F, 3, device="cuda")
    xc = x.cuda().contiguous()
    sb._lib.check(lib.sdfb200_grid_encode(enc._desc_ref(), enc.table.data_ptr(), xc.data_ptr(), 4097, o2.data_ptr(), L * F, J.data_ptr(), 0))
    torch.cuda.synchronize()
    w = torch.randn(L * F, generator=gen)
    gref = torch.autograd.grad((ref * w).sum(), xo)[0]
    gcu = (J.cpu() * w[None, :, None]).sum(1)
    torch.testing.assert_close(gcu, gref, rtol=1e-4, atol=1e-4 * float(gref.abs().max()))   # the eight edge points included
    # masked levels
    enc.set_active_levels(5)
    out_m = enc(x.cuda()).cpu()
    assert torch.equal(out_m[:, : 5 * F], out.cpu()[:, : 5 * F]) and float(out_m[:, 5 * F:].abs().max()) == 0.0


def test_grid_encode_backward_matches_autograd():
    import sdfstudio_b200 as sb

    L, F, log2T, base, maxres = 6, 2, 10, 4, 64
    g = hashgrid.growth_factor(L, base, maxres)
    for layout in ("torch", "tcnn"):
        enc = sb.Encoding(3, {"n_levels": L, "n_features_per_level": F, "log2_hashmap_size": log2T, "base_resolution": base, "per_level_scale": g,
                              "interpolation": "Smoothstep"}, layout=layout).cuda()
        gen = torch.Generator().manual_seed(3)
        x = torch.rand(513, 3, generator=gen)
        table = ((torch.rand(enc.table.shape, generator=gen) * 2 - 1) * 0.1)
        with torch.no_grad():
            enc.table.copy_(table.cuda())
        w = torch.randn(513, L * F, generator=gen)
        xg = x.cuda().requires_grad_(True)
        (enc(xg) * w.cuda()).sum().backward()
        to = table.clone().view(-1, F).requires_grad_(True)
        xo = x.clone().requires_grad_(True)
        if layout == "torch":
            ref = hashgrid.encode_torch_layout(xo, to, hashgrid.torch_layout_scalings(L, base, base * g ** (L - 1)), 1 << log2T, True)
        else:
            ref = hashgrid.encode_tcnn_layout(xo, to, hashgrid.tcnn_grid_meta(L, F, log2T, base, g), F, True)
        (ref * w).sum().backward()
        torch.testing.assert_close(enc.table.grad.cpu().view(-1, F), to.grad, rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(xg.grad.cpu(), xo.grad, rtol=1e-3, atol=1e-3 * float(xo.grad.abs().max()))


# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", FIELD_CASES)
def test_field_matches_reference_golden(name):
    import sdfstudio_b200 as sb

    G = load_golden(name)
    spec, kw, o, d, cam, nears, fars, oracle, field = build_case(name)
    rb = make_bundle(o, d, cam, nears, fars)
    sampler = sb.SpacedSampler(kw.get("spacing", "uniform"), None, num_samples=kw["S"]).eval()
    rs = sampler(rb)
    assert torch.equal(sb.rays.spacing_bins_of(rs).cpu(), G["spacing_bins"])  # bit-exact bin edges
    assert torch.equal(sb.rays.bins_of(rs).cpu(), G["euclid_bins"])
    out = field(rs, return_alphas=True, return_occupancy=True)
    H = sb.FieldHeadNames
    # fp64 oracle on the same samples: calibrates the reference's own fp32 noise for ill-conditioned outputs
    o64 = oracle64(spec, oracle.p, kw)
    eu = G["euclid_bins"].double()
    e64 = o64.get_outputs(o.double(), d.double(), eu[:, :-1], eu[:, 1:] - eu[:, :-1], cam, return_alphas=True, return_occupancy=True)
    assert_rel(out[H.SDF], G["sdf"], what="sdf")
    assert_rel(out[H.DENSITY], G["density"], floor=1e-2, what="density")
    assert_rel(out["points_norm"], G["points_norm"], what="points_norm")
    assert_rel(out[H.OCCUPANCY], G["occupancy"], floor=1e-2, what="occupancy")
    assert_within_noise(out[H.GRADIENT], G["gradients"], e64["gradients"], "gradients")
    assert_within_noise(out[H.NORMAL], G["normals"], e64["normals"], "normals")
    if spec.use_numerical_gradients:
        # central differences over 2*delta amplify the fp32 rounding of sdf by 1/delta (sdf_field.py:446-453); every
        # fp32 implementation (the reference included) carries that noise into rgb / alpha
        assert_within_noise(out[H.RGB], G["rgb"], e64["rgb"], "rgb")
        assert_within_noise(out[H.ALPHA], G["alphas"], e64["alphas"], "alpha")
        assert_rel(out["sampled_sdf"], G["sampled_sdf"], what="sampled_sdf")
    else:
        assert_rel(out[H.RGB], G["rgb"], floor=1e-2, what="rgb")
        assert_rel(out[H.ALPHA], G["alphas"], floor=1e-2, what="alpha")
    assert_rel(field.get_sdf(rs), G["get_sdf"], what="get_sdf")
    geo = field.forward_geonetwork(G["points"].cuda())
    assert_rel(geo, G["geo_points"], floor=1e-2, what="forward_geonetwork")
    g64 = o64.gradient(G["points"].double())
    assert_within_noise(field.gradient(G["points"].cuda()), G["grad_points"], g64, "gradient()")


@pytest.mark.parametrize("name", FIELD_CASES)
def test_weights_and_renderers_match_reference_golden(name):
    import sdfstudio_b200 as sb

    G = load_golden(name, "cuda")
    eu = G["euclid_bins"].contiguous()
    w_a, T_a = sb.rays.weights_from_alphas(G["alphas"], True)
    assert torch.equal(w_a, G["weights_alpha"]) and torch.equal(T_a, G["trans_alpha"])  # double-accumulated cumprod => bit-exact
    w_d, T_d = sb.rays.weights_from_density(eu, G["density"], True)
    torch.testing.assert_close(w_d, G["weights_density"], rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(T_d, G["trans_density"], rtol=1e-5, atol=1e-7)

    class RS:  # minimal duck-typed RaySamples for DepthRenderer
        _euclid_bins = eu

    w = G["weights_alpha"]
    close = lambda a, b: torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
    close(sb.RGBRenderer(background_color=torch.ones(3)).eval()(G["rgb"], w), G["render_rgb_white"])
    close(sb.RGBRenderer(background_color="last_sample").eval()(G["rgb"], w), G["render_rgb_last"])
    close(sb.RGBRenderer(background_color=torch.ones(3)).train()(G["rgb"], G["weights_density"]), G["render_rgb_white_train"])
    close(sb.DepthRenderer("expected")(w, RS()), G["render_depth_expected"])
    assert torch.equal(sb.DepthRenderer("median")(w, RS()), G["render_depth_median"])
    close(sb.AccumulationRenderer()(w), G["render_acc"])
    close(sb.SemanticRenderer()(G["normals"], w), G["render_normal"])
    fused = sb.render_from_alphas(G["alphas"], G["rgb"], G["normals"], RS(), torch.ones(3, device="cuda"))
    torch.testing.assert_close(fused["weights"], G["weights_alpha"], rtol=2e-6, atol=1e-9)
    torch.testing.assert_close(fused["bg_transmittance"], G["trans_alpha"][:, -1], rtol=2e-6, atol=1e-9)
    for k, gk in (("rgb", "render_rgb_white"), ("depth", "render_depth_expected"), ("normal", "render_normal"), ("accumulation", "render_acc")):
        close(fused[k], G[gk])
    allr = sb.render_all(w, G["rgb"], G["normals"], RS(), torch.ones(3))
    close(allr["rgb"], G["render_rgb_white"])
    close(allr["depth"], G["render_depth_expected"])
    close(allr["normal"], G["render_normal"])
    close(allr["accumulation"], G["render_acc"])


# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SAMPLER_CASES)
def test_pdf_and_merge_indices_bit_exact(name):
    import sdfstudio_b200 as sb

    G = load_golden(name, "cuda")
    spec, kw, o, d, cam, nears, fars, oracle, field = build_case(name)
    rb = make_bundle(o, d, cam, nears, fars)
    rs = sb.UniformSampler(num_samples=kw["S"]).eval()(rb)
    new, inds = sb.PDFSampler(include_original=False, histogram_padding=0.01).eval()(rb, rs, G["pdf_weights"], num_samples=24, return_indices=True)
    assert torch.equal(inds, G["pdf_inds"])  # searchsorted indices: bit-exact
    nb = sb.rays.spacing_bins_of(new)
    # bin positions: the reference's weights_sum is a torch.sum whose rounding depends on the host's vector width, and
    # the inverse CDF is ill-conditioned where the pdf ~ 0 -> require (a) the overwhelming majority bit-equal and
    # (b) cdf(bin) == u to fp32 accuracy everywhere
    assert (nb == G["pdf_spacing"]).float().mean() > 0.5  # the rest differ in the last bits (1-ulp weights_sum)
    u = (torch.linspace(0.0, 1.0 - 1.0 / 25, 25) + 1.0 / 50)[None].expand(nb.shape[0], -1)
    sp0 = sb.rays.spacing_bins_of(rs)
    assert cdf_consistency(sp0.cpu(), G["pdf_weights"][..., 0].cpu(), nb.cpu(), u, 0.01) < 2e-6
    new2, inds2 = sb.PDFSampler(include_original=True, histogram_padding=1e-5).eval()(rb, rs, G["pdf_weights"], num_samples=16, return_indices=True)
    assert torch.equal(inds2, G["pdf_inc_inds"])
    assert sb.rays.spacing_bins_of(new2).shape == G["pdf_inc_spacing"].shape
    assert (sb.rays.spacing_bins_of(new2)[:, 1:] >= sb.rays.spacing_bins_of(new2)[:, :-1]).all()  # sorted merge with the originals
    torch.testing.assert_close(sb.rays.spacing_bins_of(new2), G["pdf_inc_spacing"], rtol=0, atol=2e-2)
    # merge: feed the reference's own new bins so the inputs are identical -> indices and bins bit-exact
    ref_new = sb.rays.make_ray_samples(rb, G["pdf_spacing"].contiguous(), G["pdf_euclid"].contiguous(), rs.spacing_to_euclidean_fn)
    merged, sidx = sb.ray_samplers.merge_ray_samples(rb, rs, ref_new)
    assert torch.equal(sidx, G["merge_sorted_index"])
    assert torch.equal(sb.rays.spacing_bins_of(merged), G["merge_spacing"])
    assert torch.equal(sb.rays.bins_of(merged), G["merge_euclid"])


@pytest.mark.parametrize("name", SAMPLER_CASES)
def test_field_driven_samplers_match_reference_golden(name):
    import sdfstudio_b200 as sb

    G = load_golden(name, "cuda")
    spec, kw, o, d, cam, nears, fars, oracle, field = build_case(name)
    rb = make_bundle(o, d, cam, nears, fars)
    # fp64 run of the same samplers calibrates how far fp32 rounding of the sdf alone moves the samples
    o64 = oracle64(spec, oracle.p, kw)
    n64, f64_ = nears.double(), fars.double()
    sdf64 = lambda starts: o64.get_sdf(o.double(), d.double(), starts)
    sdf32 = lambda starts: oracle.get_sdf(o, d, starts)

    rs_n = sb.NeuSSampler().eval()(rb, sdf_fn=field.get_sdf)
    assert_within_noise(sb.rays.spacing_bins_of(rs_n), samplers.neus_sampler(nears, fars, sdf32).spacing, samplers.neus_sampler(n64, f64_, sdf64).spacing,
                        "NeuSSampler spacing bins", factor=6.0, floor=4e-6)
    assert sb.rays.bins_of(rs_n).shape == G["neus_euclid"].shape
    rs_e = sb.ErrorBoundedSampler(num_samples=64, num_samples_eval=128, num_samples_extra=32).eval()(rb, density_fn=field.laplace_density,
                                                                                                   sdf_fn=field.get_sdf, return_eikonal_points=False)
    assert sb.rays.bins_of(rs_e).shape == G["eb_euclid"].shape
    e32 = samplers.error_bounded_sampler(nears, fars, sdf32, oracle.get_beta())
    e64 = samplers.error_bounded_sampler(n64, f64_, sdf64, o64.get_beta())
    if e64.spacing.shape == e32.spacing.shape:
        assert_within_noise(sb.rays.spacing_bins_of(rs_e), e32.spacing, e64.spacing, "ErrorBoundedSampler spacing bins", factor=6.0, floor=2e-5)
    torch.testing.assert_close(sb.rays.bins_of(rs_e), G["eb_euclid"], rtol=0, atol=5e-3)
    rs_u, surf = sb.UniSurfSampler().eval()(make_bundle(o, d, cam, nears, fars), occupancy_fn=field.get_occupancy, sdf_fn=field.get_sdf,
                                            return_surface_points=True)
    u32, s32, m32 = samplers.unisurf_sampler(o, d, nears, fars, sdf32)
    u64, s64, m64 = samplers.unisurf_sampler(o.double(), d.double(), n64, f64_, sdf64)
    assert_within_noise(sb.rays.bins_of(rs_u), u32.euclid, u64.euclid, "UniSurfSampler euclid bins", factor=6.0, floor=1e-5)
    if bool(m32.any()) and surf.shape == s32.shape:
        torch.testing.assert_close(surf.cpu(), s32, rtol=1e-4, atol=1e-4)


def test_samplers_bit_exact_vs_oracle_on_shared_inputs():
    """Per-kernel bit-exactness: identical sdf / weights in, identical indices + bins out (config-2 sized rays)."""
    import sdfstudio_b200 as sb

    R, S = 4096, 128
    gen = torch.Generator().manual_seed(11)
    nears, fars = torch.full((R, 1), 0.5), torch.full((R, 1), 4.5)
    o, d, cam = cases.synthetic_rays(R, 99)
    rb = make_bundle(o, d, cam, nears, fars)
    rs = sb.UniformSampler(num_samples=S).eval()(rb)
    ob = samplers.spaced_sampler(nears, fars, S, "uniform")
    assert torch.equal(sb.rays.bins_of(rs).cpu(), ob.euclid)
    w = torch.rand(R, S, generator=gen) ** 6
    w[:7] = 0.0  # all-zero weights rows (padding path)
    new, inds = sb.PDFSampler(include_original=False, histogram_padding=1e-5).eval()(rb, rs, w.cuda()[..., None], num_samples=64, return_indices=True)
    onew, oinds = samplers.pdf_sampler(ob, w, 64, histogram_padding=1e-5, return_indices=True)
    mism = (inds.cpu() != oinds)
    # the reference's torch.sum is not associative-order stable across CPUs; tolerate tie-level flips only
    assert mism.float().mean() <= 1e-5, f"index mismatch fraction {mism.float().mean():.2e}"
    nbins = sb.rays.spacing_bins_of(new).cpu()
    assert (nbins == onew.spacing).float().mean() > 0.5
    u = (torch.linspace(0.0, 1.0 - 1.0 / 65, 65) + 1.0 / 130)[None].expand(R, -1)
    assert cdf_consistency(ob.spacing, w, nbins, u, 1e-5) < 2e-6
    merged, sidx = sb.ray_samplers.merge_ray_samples(rb, rs, new)
    om, osidx = samplers.merge_bins(ob, samplers.Bins(sb.rays.spacing_bins_of(new).cpu(), sb.rays.bins_of(new).cpu(), ob.to_euclid))
    # identical sorted values; the index choice may differ only between EQUAL keys (torch.sort is not stable by default)
    cat = torch.cat([ob.spacing[:, :-1], sb.rays.spacing_bins_of(new).cpu()[:, :-1]], -1)
    assert torch.equal(cat.gather(1, sidx.cpu()), cat.gather(1, osidx))
    diff = sidx.cpu() != osidx
    srt = cat.gather(1, osidx)
    tie = torch.zeros_like(diff)
    tie[:, 1:] |= srt[:, 1:] == srt[:, :-1]
    tie[:, :-1] |= srt[:, :-1] == srt[:, 1:]
    assert not bool((diff & ~tie).any())
    assert torch.equal(sb.rays.spacing_bins_of(merged).cpu(), om.spacing)
    # NeuS fixed-inv_s weights on a shared sdf
    sdf = (torch.rand(R, S, generator=gen) - 0.3) * torch.linspace(1, -1, S)[None]
    wk = torch.empty(R, S, device="cuda")
    lib = sb._lib.load()
    eu = sb.rays.bins_of(rs)
    sb._lib.check(lib.sdfb200_neus_upsample_weights(eu.data_ptr(), sdf.cuda().contiguous().data_ptr(), R, S, 64.0, wk.data_ptr(), 0))
    al = samplers.neus_fixed_inv_s_alpha(ob.deltas, sdf, 64.0)
    ow, _ = samplers.weights_from_alphas(al)
    torch.testing.assert_close(wk.cpu()[:, :-1], ow, rtol=2e-5, atol=5e-7)
    assert float(wk[:, -1].abs().max()) == 0.0


# ----------------------------------------------------------------------------------------------------------------
def test_render_pipeline_parity_config2_shape():
    """neus-facto field (BASELINE configs[1] shape: L=16, F=2, T=2^19, MLP 2x256) on 512 rays x 128 samples:
    rendered RGB / depth / normal within 1e-4 rel of the CPU oracle on identical rays."""
    import sdfstudio_b200 as sb

    spec = FieldSpec(num_layers=2, num_layers_color=2, hidden_dim=256, use_grid_feature=True)
    kw = dict(bias=0.5, beta_init=0.3, perturb=0.02, hash_init_scale=0.05, seed=21)
    params = init_params(spec, **kw)
    oracle = OracleField(spec, params)
    field = product_field(spec, params, kw)
    R, S = 512, 128
    o, d, cam = cases.synthetic_rays(R, 5)
    nears, fars = torch.full((R, 1), 0.5), torch.full((R, 1), 4.5)
    rb = make_bundle(o, d, cam, nears, fars)
    rs = sb.UniformSampler(num_samples=S).eval()(rb)
    out = field(rs, return_alphas=True)
    H = sb.FieldHeadNames
    w = rs.get_weights_from_alphas(out[H.ALPHA])
    img = sb.render_all(w, out[H.RGB], out[H.NORMAL], rs, torch.ones(3))
    ob = samplers.spaced_sampler(nears, fars, S, "uniform")
    oo = oracle.get_outputs(o, d, ob.starts, ob.deltas, cam, return_alphas=True)
    ow, _ = samplers.weights_from_alphas(oo["alphas"][..., 0])
    orgb = render.render_rgb(oo["rgb"], ow[..., None], torch.ones(3))
    odepth = render.render_depth(ow[..., None], ob.starts[..., None], ob.ends[..., None], "expected")
    onormal = render.render_semantics(oo["normals"], ow[..., None])
    assert_rel(img["rgb"], orgb, floor=1e-2, what="rendered rgb")
    assert_rel(img["depth"], odepth, floor=1e-2, what="rendered depth")
    assert_rel(img["normal"], onormal, floor=1e-1, what="rendered normal")
    assert_rel(out[H.SDF], oo["sdf"], what="sdf")


def test_empty_and_ragged_inputs():
    import sdfstudio_b200 as sb

    spec, kw, o, d, cam, nears, fars, oracle, field = build_case("neusfacto_c1_init")
    # zero rays
    rb0 = make_bundle(o[:0], d[:0], cam[:0], nears[:0], fars[:0])
    rs0 = sb.UniformSampler(num_samples=8).eval()(rb0)
    assert sb.rays.bins_of(rs0).shape == (0, 9)
    # a ray count that is not a multiple of any tile size, 1 sample per ray
    rb = make_bundle(o[:37], d[:37], cam[:37], nears[:37], fars[:37])
    rs = sb.UniformSampler(num_samples=1).eval()(rb)
    out = field(rs, return_alphas=True)
    ob = samplers.spaced_sampler(nears[:37], fars[:37], 1, "uniform")
    oo = oracle.get_outputs(o[:37], d[:37], ob.starts, ob.deltas, cam[:37], return_alphas=True)
    assert_rel(out[sb.FieldHeadNames.RGB], oo["rgb"], floor=1e-2, what="rgb")
    assert_rel(out[sb.FieldHeadNames.ALPHA], oo["alphas"], floor=1e-2, what="alpha")


def test_large_batch_crosses_chunks():
    """N > the generic engine's chunk: a slice of rays around the first chunk boundary, one of them straddling it, must match a small call
    on that slice bit for bit."""
    import sdfstudio_b200 as sb

    spec, kw, o, d, cam, nears, fars, oracle, field = build_case("neusfacto_c1_init")
    R, S, sl = 1500, 50, slice(1330, 1380)      # 75 000 points
    assert_straddles_chunk(R, S, sl)
    o, d, cam = cases.synthetic_rays(R, 123)
    nears, fars = torch.full((R, 1), 0.5), torch.full((R, 1), 4.5)
    rb = make_bundle(o, d, cam, nears, fars)
    rs = sb.UniformSampler(num_samples=S).eval()(rb)
    big = field(rs, return_alphas=True)
    rb2 = make_bundle(o[sl], d[sl], cam[sl], nears[sl], fars[sl])
    small = field(sb.UniformSampler(num_samples=S).eval()(rb2), return_alphas=True)
    for k in (sb.FieldHeadNames.RGB, sb.FieldHeadNames.SDF, sb.FieldHeadNames.ALPHA, sb.FieldHeadNames.GRADIENT):
        assert torch.equal(big[k][sl], small[k]), k


# ----------------------------------------------------------------------------------------------------------------
# proposal density field + ProposalNetworkSampler (SURVEY section 8f row 1)
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hidden,layers,contraction", [(16, 2, None), (64, 3, "linf"), (32, 2, "l2")])
def test_density_field_matches_oracle(hidden, layers, contraction):
    import sdfstudio_b200 as sb
    from oracle import density as odensity

    class _C:
        def __init__(self, order):
            self.order = order

    sd = None if contraction is None else _C(float("inf") if contraction == "linf" else None)
    aabb = torch.tensor([[-1.0, -1, -1], [1, 1, 1]])
    f = sb.HashMLPDensityField(aabb, num_layers=layers, hidden_dim=hidden, spatial_distortion=sd, num_levels=5, max_res=256, log2_hashmap_size=12).cuda().eval()
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        nb = f.mlp_base
        nb.params[nb.n_net:] = ((torch.rand(nb.n_grid, generator=g) * 2 - 1) * 0.5).cuda()
    pos = (torch.rand(37, 11, 3, generator=g) * 2 - 1) * (3.0 if contraction else 1.0)
    dens, pre = f.density_from_positions(pos.cuda(), return_pre_activation=True)
    p = f.mlp_base.params.detach().cpu()
    growth = hashgrid.growth_factor(5, 16, 256)
    od, opre = odensity.density_field(pos, p[: nb.n_net], p[nb.n_net:], hidden, layers - 1, 5, 2, 12, 16, growth,
                                      aabb=None if contraction else aabb, contraction=contraction)
    assert dens.shape == (37, 11, 1)
    torch.testing.assert_close(pre.cpu(), opre, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(dens.cpu(), od, rtol=1e-4, atol=1e-6)


def test_proposal_network_sampler_matches_oracle():
    """neus-facto's sampler (ray_samplers.py:537-578 with the preset numbers neus_facto.py:47-64): (256, 96) proposal samples
    through two HashMLPDensityFields, 48 final samples -- this library end to end vs the CPU oracle."""
    import numpy as np

    import sdfstudio_b200 as sb
    from oracle import density as odensity

    aabb = torch.tensor([[-1.0, -1, -1], [1, 1, 1]])
    g = torch.Generator().manual_seed(9)
    nets = []
    for max_res in (64, 256):
        f = sb.HashMLPDensityField(aabb, num_layers=2, hidden_dim=16, num_levels=5, max_res=max_res, log2_hashmap_size=17).cuda().eval()
        with torch.no_grad():
            nb = f.mlp_base
            nb.params[nb.n_net:] = ((torch.rand(nb.n_grid, generator=g) * 2 - 1) * 2.0).cuda()
        nets.append(f)
    R = 200
    o, d, cam = cases.synthetic_rays(R, 77)
    nears, fars = torch.full((R, 1), 0.5), torch.full((R, 1), 4.5)
    rb = make_bundle(o, d, cam, nears, fars)
    sampler = sb.ProposalNetworkSampler(num_proposal_samples_per_ray=(256, 96), num_nerf_samples_per_ray=48, num_proposal_network_iterations=2).eval()
    rs, weights_list, rs_list = sampler(rb, density_fns=[n.density_fn for n in nets])
    assert sb.rays.bins_of(rs).shape == (R, 49) and len(weights_list) == 2

    def ofn(net, max_res):
        nb = net.mlp_base
        p = nb.params.detach().cpu()
        gf = float(np.exp((np.log(max_res) - np.log(16)) / 4))
        return lambda pos: odensity.density_field(pos, p[: nb.n_net], p[nb.n_net:], 16, 1, 5, 2, 17, 16, gf, aabb=aabb)[0][..., 0]

    ob, owl, obl = samplers.proposal_sampler(o, d, nears, fars, [ofn(nets[0], 64), ofn(nets[1], 256)], (256, 96), 48)
    torch.testing.assert_close(weights_list[0][..., 0].cpu(), owl[0], rtol=2e-4, atol=1e-6)
    # sample positions: inverse-CDF conditioning -> compare at the level of the oracle's own sensitivity
    torch.testing.assert_close(sb.rays.bins_of(rs_list[1]).cpu(), obl[1].euclid, rtol=0, atol=5e-3)
    torch.testing.assert_close(sb.rays.bins_of(rs).cpu(), ob.euclid, rtol=0, atol=2e-2)
    assert (sb.rays.bins_of(rs)[:, 1:] >= sb.rays.bins_of(rs)[:, :-1]).all()


# ----------------------------------------------------------------------------------------------------------------
# packed samples: the `ray_indices` / `num_rays` branch of the renderers (renderers.py:74-79,192-194,249-253)
# ----------------------------------------------------------------------------------------------------------------
def test_packed_renderers_match_dense_and_reference_formulas():
    """A ragged packed sample list (different sample counts per ray, one ray with no sample) against (a) the fp64 restatement of
    nerfacc.accumulate_along_rays = per-ray index_add and (b) the dense renderers on a zero-padded copy."""
    import sdfstudio_b200 as sb

    g = torch.Generator().manual_seed(17)
    R, Smax = 301, 23
    counts = torch.randint(0, Smax + 1, (R,), generator=g)
    counts[5] = 0
    N = int(counts.sum())
    ray_indices = torch.repeat_interleave(torch.arange(R), counts)
    w = torch.rand(N, 1, generator=g) * 0.2
    rgb = torch.rand(N, 3, generator=g)
    nrm = torch.randn(N, 3, generator=g)
    starts = torch.rand(N, 1, generator=g) * 3 + 0.5
    ends = starts + torch.rand(N, 1, generator=g) * 0.1
    bg = torch.tensor([0.2, 0.7, 0.4])

    class _Fr:
        pass

    class _RS:
        frustums = _Fr()

    _RS.frustums.starts, _RS.frustums.ends = starts.cuda(), ends.cuda()
    o_rgb = sb.RGBRenderer(background_color=bg.cuda()).eval()(rgb.cuda(), w.cuda(), ray_indices=ray_indices.cuda(), num_rays=R)
    o_acc = sb.AccumulationRenderer.forward(w.cuda(), ray_indices=ray_indices.cuda(), num_rays=R)
    o_dep = sb.DepthRenderer("expected")(w.cuda(), _RS, ray_indices=ray_indices.cuda(), num_rays=R)
    # (a) fp64 index_add
    w64 = w.double()
    acc = torch.zeros(R, 1, dtype=torch.float64).index_add_(0, ray_indices, w64)
    crgb = torch.zeros(R, 3, dtype=torch.float64).index_add_(0, ray_indices, w64 * rgb.double()) + bg.double() * (1 - acc)
    steps = (starts.double() + ends.double()) / 2
    dep = (torch.zeros(R, 1, dtype=torch.float64).index_add_(0, ray_indices, w64 * steps) / (acc + 1e-10)).clip(steps.min(), steps.max())
    torch.testing.assert_close(o_acc.cpu().double(), acc, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(o_rgb.cpu().double(), crgb.clamp(0, 1), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(o_dep.cpu().double(), dep, rtol=1e-5, atol=1e-5)
    assert o_rgb.shape == (R, 3) and o_acc.shape == (R, 1) and o_dep.shape == (R, 1)
    with pytest.raises(NotImplementedError):
        sb.RGBRenderer(background_color="last_sample")(rgb.cuda(), w.cuda(), ray_indices=ray_indices.cuda(), num_rays=R)


# ----------------------------------------------------------------------------------------------------------------
# samplers driven by IDENTICAL sdf values (the oracle's, evaluated on the product's own sample positions): what remains is the
# arithmetic of the sampler kernels themselves, so the bounds are tight (no field rounding to absorb)
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["neusfacto_c1"])
def test_samplers_on_shared_sdf_function(name):
    import sdfstudio_b200 as sb

    spec, kw, o, d, cam, nears, fars, oracle, field = build_case(name)
    rb = make_bundle(o, d, cam, nears, fars)

    def shared_sdf(rs):                                   # the ORACLE's fp32 sdf at the product's sample starts
        starts = sb.rays.bins_of(rs)[:, :-1].cpu()
        return oracle.get_sdf(o, d, starts).cuda()[..., None]

    sdf32 = lambda starts: oracle.get_sdf(o, d, starts)  # noqa: E731
    rs_n = sb.NeuSSampler().eval()(rb, sdf_fn=shared_sdf)
    on = samplers.neus_sampler(nears, fars, sdf32)
    pn = sb.rays.spacing_bins_of(rs_n).cpu()
    # every upsampling round inverts a CDF: bins agree to a few ulp of the [0,1] spacing domain and the ORDER of the merged samples
    # (the sorted_index stream of merge_ray_samples) is identical
    assert float((pn - on.spacing).abs().max()) < 2e-6, float((pn - on.spacing).abs().max())
    assert float((pn == on.spacing).float().mean()) > 0.5      # the rest differs by 1-2 ulp (inverse-CDF arithmetic order)
    assert torch.equal(torch.argsort(pn[:, :-1], dim=-1, stable=True), torch.argsort(on.spacing[:, :-1], dim=-1, stable=True))
    rs_e = sb.ErrorBoundedSampler(num_samples=64, num_samples_eval=128, num_samples_extra=32).eval()(rb, density_fn=field.laplace_density, sdf_fn=shared_sdf,
                                                                                                   return_eikonal_points=False)
    oe = samplers.error_bounded_sampler(nears, fars, sdf32, oracle.get_beta())
    pe = sb.rays.spacing_bins_of(rs_e).cpu()
    assert pe.shape == oe.spacing.shape
    # the final inverse-CDF draw divides by density weights that sit next to a saturating exp(-sum): a few 1e-5 in the [0,1] spacing
    # domain (measured 3.3e-5) -- two orders of magnitude below the bound needed when the sdf itself differs (eb_euclid golden: 5e-3)
    assert float((pe - oe.spacing).abs().max()) < 1e-4, float((pe - oe.spacing).abs().max())
    assert float((sb.rays.bins_of(rs_e).cpu() - oe.euclid).abs().max()) < 4e-4
