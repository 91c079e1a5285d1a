"""-m gpu: tensor-core building blocks (bf16 split-plane wgmma GEMM tile, A operand in shared memory or in registers) against torch fp64."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("ts", [0, 1])
@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("K,N", [(32, 16), (96, 256), (256, 256), (256, 96), (64, 80)])
def test_tc_gemm_tile(ts, planes, K, N):
    import sdfstudio_b200 as sb

    lib = sb._lib.load_debug()
    g = torch.Generator().manual_seed(K * 1000 + N)
    A = torch.randn(128, K, generator=g).cuda()
    W = (torch.randn(N, K, generator=g) / K**0.5).cuda()
    Np = (N + 15) // 16 * 16
    D = torch.full((128, Np), float("nan"), device="cuda")
    Np64 = (N + 63) // 64 * 64
    scratch = torch.zeros((K // 32) * planes * Np64 * 64, dtype=torch.uint8, device="cuda")
    rc = lib.sdfb200_debug_tc_gemm(A.data_ptr(), W.data_ptr(), K, N, ts, planes, D.data_ptr(), scratch.data_ptr(), 0)
    assert rc == 0, lib.sdfb200_last_error_string()
    torch.cuda.synchronize()
    ref = (A.double() @ W.double().t()).float()
    scale = float((A.abs().double() @ W.abs().double().t()).max())
    err = float((D[:, :N] - ref).abs().max()) / scale
    assert Np == N or float(D[:, N:].abs().max()) == 0.0
    tol = 2e-5 if planes == 2 else 6e-3
    assert err < tol, f"relative-to-|A||W| error {err:.3e} (planes={planes}, ts={ts})"
    if planes == 2:
        # the split must actually buy precision: error well below a single bf16 pass
        assert err < 1e-4


# ----------------------------------------------------------------------------------------------------------------
# fused tensor-core field kernel (k_field_tc): bf16x3 must sit at the fp32 reference's own noise level, bf16 is the
# fast mode reported with PSNR
# ----------------------------------------------------------------------------------------------------------------
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from helpers import assert_within_noise, build_case, load_golden, make_bundle, oracle64, rel_err  # noqa: E402
from oracle import render, samplers  # noqa: E402


def _run_case(name, precision):
    import sdfstudio_b200 as sb

    spec, kw, o, d, cam, nears, fars, oracle, field = build_case(name, precision=precision)
    rb = make_bundle(o, d, cam, nears, fars)
    rs = sb.UniformSampler(num_samples=kw["S"]).eval()(rb)
    out = field(rs, return_alphas=True, return_occupancy=True)
    torch.cuda.synchronize()
    eu = sb.rays.bins_of(rs).cpu().double()
    o64 = oracle64(spec, oracle.p, kw)
    e64 = o64.get_outputs(o.double(), d.double(), eu[:, :-1], eu[:, 1:] - eu[:, :-1], cam, return_alphas=True, return_occupancy=True)
    return sb, field, rs, out, e64, (o, d, cam, eu, o64)


@pytest.mark.parametrize("name", ["neusfacto_c1", "neusfacto_c1_init"])
def test_field_tc_bf16x3_matches_reference(name):
    sb, field, rs, out, e64, (o, d, cam, eu, o64) = _run_case(name, "bf16x3")
    G = load_golden(name)  # the unmodified reference's fp32 outputs on the same samples
    H = sb.FieldHeadNames
    # per-sample heads: error vs the fp64 oracle bounded by max(1e-4 of the head's scale, 4x the reference's own fp32 noise)
    for key, gk in ((H.SDF, "sdf"), (H.RGB, "rgb"), (H.ALPHA, "alphas"), (H.DENSITY, "density"), (H.GRADIENT, "gradients"),
                    (H.NORMAL, "normals"), (H.OCCUPANCY, "occupancy")):
        assert_within_noise(out[key], G[gk], e64[gk], f"{name}/{gk}", factor=4.0, floor=1e-4 * float(e64[gk].abs().max()))
    # rendered image quantities: BASELINE north_star bound (1e-4 relative)
    w = rs.get_weights_from_alphas(out[H.ALPHA])
    img = sb.render_all(w, out[H.RGB], out[H.NORMAL], rs, torch.ones(3, device="cuda"))
    ow, _ = samplers.weights_from_alphas(e64["alphas"][..., 0])
    orgb = render.render_rgb(e64["rgb"], ow[..., None], torch.ones(3, dtype=torch.float64))
    assert rel_err(img["rgb"], orgb, 1e-2) < 1e-4
    gw, _ = samplers.weights_from_alphas(G["alphas"][..., 0])
    gdep = render.render_depth(gw[..., None], eu[:, :-1, None].float(), eu[:, 1:, None].float(), "expected")
    odep = render.render_depth(ow[..., None], eu[:, :-1, None], eu[:, 1:, None], "expected")
    assert_within_noise(img["depth"], gdep, odep, f"{name}/depth", factor=4.0, floor=1e-4 * float(odep.abs().max()))
    # sdf-only mode of the kernel (sampler path): un-contracted positions, same arithmetic
    sdf_u = field.get_sdf(rs)
    e_sdf = o64.get_sdf(o.double(), d.double(), eu[:, :-1])
    assert_within_noise(sdf_u[..., 0], G["get_sdf"][..., 0], e_sdf, f"{name}/get_sdf", factor=4.0, floor=1e-4 * float(e_sdf.abs().max()))


def test_field_tc_bf16_fast_mode_psnr():
    sb, field, rs, out, e64, _ = _run_case("neusfacto_c1", "bf16")
    H = sb.FieldHeadNames
    w = rs.get_weights_from_alphas(out[H.ALPHA])
    img = sb.render_all(w, out[H.RGB], out[H.NORMAL], rs, torch.ones(3, device="cuda"))
    ow, _ = samplers.weights_from_alphas(e64["alphas"][..., 0])
    orgb = render.render_rgb(e64["rgb"], ow[..., None], torch.ones(3, dtype=torch.float64))
    mse = float(((img["rgb"].cpu().double() - orgb) ** 2).mean())
    psnr = -10.0 * torch.log10(torch.tensor(mse)).item()
    assert psnr > 60.0, f"fast-mode PSNR vs reference {psnr:.1f} dB"


def test_field_tc_ragged_tail_and_point_mode():
    """N not a multiple of the 128-point tile; point-mode entry (forward_geonetwork / gradient)."""
    import sdfstudio_b200 as sb

    spec, kw, o, d, cam, nears, fars, oracle, field = build_case("neusfacto_c1", precision="bf16x3")
    G = load_golden("neusfacto_c1")
    pts = G["points"].cuda()  # 200 points
    geo = field.forward_geonetwork(pts)
    o64 = oracle64(spec, oracle.p, kw)
    assert_within_noise(geo, G["geo_points"], o64.forward_geonetwork(G["points"].double()), "forward_geonetwork", factor=4.0, floor=2e-5)
    assert_within_noise(field.gradient(pts), G["grad_points"], o64.gradient(G["points"].double()), "gradient()", factor=4.0, floor=2e-5)
    rb = make_bundle(o[:37], d[:37], cam[:37], nears[:37], fars[:37])
    rs = sb.UniformSampler(num_samples=5).eval()(rb)  # 185 points
    out = field(rs, return_alphas=True)
    ob = samplers.spaced_sampler(nears[:37], fars[:37], 5, "uniform")
    oo = oracle.get_outputs(o[:37], d[:37], ob.starts, ob.deltas, cam[:37], return_alphas=True)
    assert rel_err(out[sb.FieldHeadNames.RGB], oo["rgb"], 1e-2) < 1e-3
    assert rel_err(out[sb.FieldHeadNames.SDF], oo["sdf"], 1e-3) < 1e-3


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_field_fp16_table_matches_oracle_on_the_same_quantised_table(precision):
    """table_dtype="fp16" (tiny-cuda-nn's storage precision): the kernels gather half-precision entries; against the oracle
    holding the same fp16-representable values the field must agree as tightly as with an fp32 table."""
    import sdfstudio_b200 as sb

    spec, kw, o, d, cam, nears, fars, oracle, field = build_case("neusfacto_c1", precision=precision, table_dtype="fp16")
    assert field.encoding.compute_table().dtype == torch.float16
    rb = make_bundle(o, d, cam, nears, fars)
    rs = sb.UniformSampler(num_samples=kw["S"]).eval()(rb)
    out = field(rs, return_alphas=True)
    eu = sb.rays.bins_of(rs).cpu()
    oo = oracle.get_outputs(o, d, eu[:, :-1], eu[:, 1:] - eu[:, :-1], cam, return_alphas=True)
    H = sb.FieldHeadNames
    o64 = oracle64(spec, oracle.p, kw)
    e64 = o64.get_outputs(o.double(), d.double(), eu[:, :-1].double(), (eu[:, 1:] - eu[:, :-1]).double(), cam, return_alphas=True)
    for key, k in ((H.SDF, "sdf"), (H.RGB, "rgb"), (H.ALPHA, "alphas"), (H.GRADIENT, "gradients")):
        assert_within_noise(out[key], oo[k], e64[k], f"fp16-table/{precision}/{k}", factor=4.0, floor=1e-4 * float(e64[k].abs().max()))


# ----------------------------------------------------------------------------------------------------------------
# generic tensor-core Linear (csrc/tc_linear.cu): the GEMM engine of every field shape outside the fused kernel's family
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("epi", [0, 1, 2, 3])
@pytest.mark.parametrize("M,Kp,Np", [(128, 80, 256), (1000, 384, 272), (333, 256, 16), (4097, 528, 320)])
def test_tc_linear_matches_fp64(planes, epi, M, Kp, Np):
    import sdfstudio_b200 as sb

    lib = sb._lib.load_debug()
    g = torch.Generator().manual_seed(M + Kp + Np + epi)
    ldx, ldy = Kp + 16, Np + 32
    X = (torch.randn(M, ldx, generator=g) * 0.5).cuda()
    W = (torch.randn(Np, Kp, generator=g) / Kp**0.5).cuda()
    b = (torch.randn(Np, generator=g) * 0.1).cuda()
    aux = (torch.rand(M, Np, generator=g) * 0.05).cuda()               # "h" values whose softplus' scales the result (epi 3)
    aux_cols = Np - 16
    Y = torch.full((M, ldy), float("nan"), device="cuda")
    scratch = torch.zeros(1 << 18, dtype=torch.uint8, device="cuda")
    rc = lib.sdfb200_debug_tc_linear(planes, epi, X.data_ptr(), ldx, W.data_ptr(), b.data_ptr(), Y.data_ptr(), ldy, M, Np, Kp, aux.data_ptr(), Np, aux_cols,
                                     scratch.data_ptr(), 0)
    assert rc == 0, lib.sdfb200_last_error_string()
    torch.cuda.synchronize()
    z = X[:, :Kp].double() @ W.double().t()
    if epi != 3:
        z = z + b.double()
    if epi == 1:
        z = torch.nn.functional.softplus(z, beta=100)
    elif epi == 2:
        z = torch.relu(z)
    elif epi == 3:
        z[:, :aux_cols] = z[:, :aux_cols] * (-torch.expm1(-100.0 * aux.double()[:, :aux_cols]))
    scale = float((X[:, :Kp].abs().double() @ W.abs().double().t()).max())
    err = float((Y[:, :Np].double() - z).abs().max()) / scale
    assert torch.isnan(Y[:, Np:]).all()                                 # nothing written outside [0, Np)
    assert err < (3e-5 if planes == 2 else 8e-3), f"relative-to-|X||W| error {err:.3e}"


@pytest.mark.parametrize("name", ["bakedsdf_small", "volsdf_stock", "angelo_small"])
def test_generic_shapes_on_the_tensor_core_engine(name):
    """Field shapes outside the fused family at precision='bf16x3': the generic kernels with tensor-core GEMMs must sit at the fp32
    reference's own noise level, like the fused kernel does for neus-facto."""
    sb, field, rs, out, e64, (o, d, cam, eu, o64) = _run_case(name, "bf16x3")
    G = load_golden(name)
    H = sb.FieldHeadNames
    # floor 3e-4 of the head's scale: the stock 8x256 network chains 16 bf16x3 GEMMs (forward + reverse sweep), each ~2^-16 relative,
    # and the angelo shape divides sdf differences by 2 delta (numerical gradients)
    for key, gk in ((H.SDF, "sdf"), (H.RGB, "rgb"), (H.ALPHA, "alphas"), (H.DENSITY, "density"), (H.GRADIENT, "gradients"), (H.NORMAL, "normals")):
        assert_within_noise(out[key], G[gk], e64[gk], f"{name}/{gk}", factor=4.0, floor=3e-4 * float(e64[gk].abs().max()))
    w = rs.get_weights_from_alphas(out[H.ALPHA])
    img = sb.render_all(w, out[H.RGB], out[H.NORMAL], rs, torch.ones(3, device="cuda"))
    ow, _ = samplers.weights_from_alphas(e64["alphas"][..., 0])
    orgb = render.render_rgb(e64["rgb"], ow[..., None], torch.ones(3, dtype=torch.float64))
    assert rel_err(img["rgb"], orgb, 1e-2) < 1e-4
