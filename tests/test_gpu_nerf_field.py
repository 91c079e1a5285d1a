"""GPU: the vanilla NeRF background field (background_model="mlp") against the fp64 oracle (oracle/nerf_field.py).

The oracle in fp64 is fed the fp32 contracted positions (what the reference's fp32 SceneContraction hands to the encoding); the PE reaches
arguments of ~1000 rad, so fp32 itself is the noise source.  Every bound is a factor of the fp32 oracle's own distance to fp64, plus a floor.
"""
import math

import pytest
import torch

import sdfstudio_b200 as sb
from oracle import nerf_field as onf
from oracle.field import scene_contraction
from oracle.make_golden_nerf_field import seeded_params

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
FACTOR = 4.0


def make_field(norm="linf", precision="bf16x3", pe=(10, 0.0, 9.0, True), de=(4, 0.0, 3.0, True), seed=3, **kw):
    pe_enc = sb.NeRFEncoding(3, pe[0], pe[1], pe[2], include_input=pe[3])
    de_enc = sb.NeRFEncoding(3, de[0], de[1], de[2], include_input=de[3])
    sd = None if norm == "none" else sb.SceneContraction(order=float("inf") if norm == "linf" else None)
    f = sb.NeRFField(position_encoding=pe_enc, direction_encoding=de_enc, spatial_distortion=sd, precision=precision, **kw)
    params = seeded_params({k: tuple(v.shape) for k, v in f.state_dict().items()}, seed)
    f.load_state_dict(params)
    spec = onf.NerfSpec(pe=pe, de=de, base_layers=len(f.mlp_base.layers), head_layers=len(f.mlp_head.layers), skips=tuple(f.mlp_base._skip_connections),
                        contraction=None if norm == "none" else norm)
    return f.to(DEV).eval(), params, spec


def ray_case(R, S, seed=0):
    g = torch.Generator().manual_seed(seed)
    o = torch.randn(R, 3, generator=g) * 0.3
    d = torch.randn(R, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True)
    fars = 1.5 + 2.0 * torch.rand(R, 1, generator=g)
    rb = sb.RayBundle(origins=o.to(DEV), directions=d.to(DEV), pixel_area=torch.ones(R, 1, device=DEV), camera_indices=torch.zeros(R, 1, dtype=torch.long, device=DEV),
                      nears=fars.to(DEV), fars=torch.full((R, 1), 1000.0, device=DEV))
    return sb.LinearDisparitySampler(num_samples=S).eval()(rb), o, d


def point_samples(N, seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, 3, generator=g) * torch.logspace(-1, 1.8, max(N, 1))[:N, None]
    d = torch.randn(N, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True).clamp_min(1e-6)
    fr = sb.Frustums(origins=x.to(DEV), directions=d.to(DEV), starts=torch.zeros(N, 1, device=DEV), ends=torch.zeros(N, 1, device=DEV),
                     pixel_area=torch.ones(N, 1, device=DEV))
    return sb.RaySamples(frustums=fr, camera_indices=torch.zeros(N, 1, dtype=torch.long, device=DEV)), x, d


def oracle_pair(positions, directions, params, spec):
    """(fp32 oracle, fp64 oracle fed the fp32 contracted positions)"""
    o32 = onf.field(positions, directions, params, spec)
    p64 = {k: v.double() for k, v in params.items()}
    o64 = onf.field(o32["contracted"].double(), directions.double(), p64, spec, contracted=True)
    return o32, o64


def check(name, got, o32, o64, floor):
    got = got.double().cpu()
    assert torch.isfinite(got).all(), name
    ref_err = float((o32.double() - o64).abs().max()) if got.numel() else 0.0
    err = float((got - o64).abs().max()) if got.numel() else 0.0
    assert err <= FACTOR * ref_err + floor, f"{name}: {err:.3e} vs fp32 oracle {ref_err:.3e} (+ floor {floor:.1e})"
    return err


# (density, rgb): absolute, on O(1) outputs.  The same at fp32: ATen's CUDA L2 norm can differ from the CPU's by an ulp, and the PE's 512 x
# frequency turns that into ~1e-5 on the outputs
FLOOR = {"bf16x3": (2e-4, 5e-5), "fp32": (2e-4, 5e-5)}


def compare(f, rs, pos, dirs, params, spec, precision):
    with torch.no_grad():
        out = f(rs)
    o32, o64 = oracle_pair(pos, dirs, params, spec)
    fd, fr = FLOOR[precision]
    d_err = check("density", out[sb.FieldHeadNames.DENSITY], o32["density"], o64["density"], fd * max(1.0, float(o64["density"].abs().max())))
    r_err = check("rgb", out[sb.FieldHeadNames.RGB], o32["rgb"], o64["rgb"], fr)
    return out, d_err, r_err


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
@pytest.mark.parametrize("norm", ["linf", "l2", "none"])
def test_ray_mode_matches_oracle(norm, precision):
    f, params, spec = make_field(norm, precision)
    rs, o, d = ray_case(64, 32)
    eu = sb.rays.bins_of(rs).cpu()
    pos = onf.midpoints(o[:, None], d[:, None], eu[:, :-1, None], eu[:, 1:, None])
    compare(f, rs, pos, d[:, None].expand(*pos.shape), params, spec, precision)


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
@pytest.mark.parametrize("N", [0, 1, 127, 128, 129, 1000])
def test_point_mode_sizes(N, precision):
    f, params, spec = make_field("linf", precision)
    rs, x, d = point_samples(N)
    if N == 0:
        with torch.no_grad():
            out = f(rs)
        assert out[sb.FieldHeadNames.DENSITY].shape == (0, 1) and out[sb.FieldHeadNames.RGB].shape == (0, 3)
        return
    compare(f, rs, x, d, params, spec, precision)


@pytest.mark.parametrize("pe,de", [((6, 0.0, 5.0, False), (2, 0.0, 1.0, True)), ((10, 0.0, 9.0, True), (10, 0.0, 9.0, False)),
                                   ((3, 1.0, 2.5, True), (0, 0.0, 0.0, True))])
def test_encoding_variants(pe, de):
    f, params, spec = make_field("l2", "bf16x3", pe=pe, de=de)
    assert f._engine() == "kernel"
    rs, x, d = point_samples(700)
    compare(f, rs, x, d, params, spec, "bf16x3")


@pytest.mark.parametrize("R", [4096, 65536])
def test_large_batches_one_launch_deterministic(R):
    f, params, spec = make_field("linf", "bf16x3")
    rs, o, d = ray_case(R, 32, seed=5)
    with torch.no_grad():
        f(rs)
        torch.cuda.synchronize()
        n0 = sb._lib.launch_count()
        a = f(rs)
        torch.cuda.synchronize()
        assert sb._lib.launch_count() - n0 == 1
        b = f(rs)
    for k in a:
        assert torch.isfinite(a[k]).all() and torch.equal(a[k], b[k]), k
    idx = torch.arange(0, R, R // 64)
    eu = sb.rays.bins_of(rs).cpu()[idx]
    pos = onf.midpoints(o[idx, None], d[idx, None], eu[:, :-1, None], eu[:, 1:, None])
    o32, o64 = oracle_pair(pos, d[idx, None].expand(*pos.shape), params, spec)
    check("density", a[sb.FieldHeadNames.DENSITY][idx.to(DEV)], o32["density"], o64["density"], 2e-4 * max(1.0, float(o64["density"].abs().max())))
    check("rgb", a[sb.FieldHeadNames.RGB][idx.to(DEV)], o32["rgb"], o64["rgb"], 5e-5)


def test_bf16_background_psnr():
    """The package states PSNR >= 60 dB for its bf16 mode; this measures it on the rendered background colour."""
    f16, params, spec = make_field("linf", "bf16")
    rs, o, d = ray_case(4096, 32, seed=9)
    with torch.no_grad():
        out = f16(rs)
        ref = make_field("linf", "fp32")[0](rs)
        w16 = rs.get_weights(out[sb.FieldHeadNames.DENSITY])
        w32 = rs.get_weights(ref[sb.FieldHeadNames.DENSITY])
        bg = torch.tensor([0.2, 0.5, 0.9], device=DEV)
        c16 = sb.RGBRenderer(bg).eval()(out[sb.FieldHeadNames.RGB], w16)
        c32 = sb.RGBRenderer(bg).eval()(ref[sb.FieldHeadNames.RGB], w32)
    mse = float(((c16 - c32) ** 2).mean())
    psnr = 10 * math.log10(1.0 / max(mse, 1e-30))
    print(f"bf16 background rgb PSNR vs fp32: {psnr:.1f} dB")
    assert psnr >= 60.0, psnr


@pytest.mark.parametrize("kw", [{"head_mlp_layer_width": 64}, {"skip_connections": (3,)}])
def test_outside_family_runs_composition(kw):
    f, params, spec = make_field("linf", "bf16x3", **kw)
    assert f._engine() == "compose"
    rs, x, d = point_samples(500)
    compare(f, rs, x, d, params, spec, "bf16x3")


def _kink_free(pre, margin):
    """rows whose every ReLU pre-activation is at least `margin` from 0"""
    return torch.stack([(p.abs() > margin).all(-1) for p in pre]).all(0)


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_training_gradients_match_fp64_autograd(precision):
    f, params, spec = make_field("linf", precision)
    f.train()
    rs, x, d = point_samples(384, seed=4)
    # fp64 oracle on the fp32-contracted positions; keep the samples away from ReLU kinks
    c = scene_contraction(x, "linf")
    p64 = {k: v.double().requires_grad_(True) for k, v in params.items()}
    pre = []
    orig_relu = torch.relu

    def relu_rec(t):
        pre.append(t.detach())
        return orig_relu(t)

    torch.relu = relu_rec
    try:
        o64 = onf.field(c.double(), d.double(), p64, spec, contracted=True)
    finally:
        torch.relu = orig_relu
    keep = _kink_free(pre, 1e-4)
    assert keep.sum() > 100
    g = torch.Generator().manual_seed(2)
    wd, wr = torch.randn(384, 1, generator=g), torch.randn(384, 3, generator=g)
    m = keep[:, None].double()
    loss64 = (o64["density"] * wd * m).sum() * 1e-2 + (o64["rgb"] * wr * m).sum()
    loss64.backward()
    out = f(rs)
    md = keep[:, None].to(DEV).float()
    loss = (out[sb.FieldHeadNames.DENSITY] * wd.to(DEV) * md).sum() * 1e-2 + (out[sb.FieldHeadNames.RGB] * wr.to(DEV) * md).sum()
    loss.backward()
    tol = 2e-4 if precision == "bf16x3" else 2e-5
    assert abs(loss.item() - loss64.item()) <= tol * max(1.0, abs(float(loss64))) * 10
    for name, p in f.named_parameters():
        ref = p64[name].grad
        got = p.grad.double().cpu()
        rel = float((got - ref).norm() / ref.norm().clamp_min(1e-12))
        assert rel < (3e-3 if precision == "bf16x3" else 1e-4), (name, rel)


def _sdf_setup(kind):
    from oracle.field import FieldSpec  # noqa: F401  (the SDF field is the foreground only; its values are not checked here)
    from sdfstudio_b200.synthetic import dtu_like_rays, perturb_field_

    torch.manual_seed(0)
    cfg = sb.SDFFieldConfig(use_grid_feature=True, num_layers=2, num_layers_color=2, hidden_dim=256, bias=0.5, beta_init=0.3, inside_outside=False,
                            log2_hashmap_size=15, grid_layout="torch", precision="bf16x3")
    field = perturb_field_(sb.SDFField(cfg, torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), 49), 0).to(DEV).eval()
    R = 256
    o, d, cam, nears, fars = dtu_like_rays(R, 7)
    rb = sb.RayBundle(origins=o.to(DEV), directions=d.to(DEV), pixel_area=torch.ones(R, 1, device=DEV), directions_norm=torch.ones(R, 1, device=DEV),
                      camera_indices=cam.view(R, 1).to(DEV), nears=nears.to(DEV), fars=fars.to(DEV))
    if kind == "neus":
        sampler = sb.NeuSSampler(num_samples=32, num_samples_importance=32).eval()
    else:
        sampler = sb.ErrorBoundedSampler(num_samples=64, num_samples_eval=128, num_samples_extra=32).eval()
    return field, sampler, rb


@pytest.mark.parametrize("kind", ["neus", "volsdf"])
def test_surface_renderer_background_branch(kind):
    field, sampler, rb = _sdf_setup(kind)
    bgf, params, spec = make_field("linf", "bf16x3")
    bg_color = torch.tensor([0.2, 0.5, 0.9], device=DEV)
    plain = sb.SurfaceRenderer(field, sampler, kind=kind, background_color=bg_color).eval()
    with_bg = sb.SurfaceRenderer(field, sampler, kind=kind, background_color=bg_color, field_background=bgf).eval()
    nears, fars = rb.nears.clone(), rb.fars.clone()
    with torch.no_grad():
        a = plain.get_outputs(rb)
        b = plain.get_outputs(rb)
        c = with_bg.get_outputs(rb)
    assert torch.equal(rb.nears, nears) and torch.equal(rb.fars, fars)              # the caller's bundle is left as it is
    for k in ("rgb", "depth", "normal", "accumulation"):
        assert torch.equal(a[k], b[k]), k
    for k in ("depth", "normal", "accumulation"):
        assert torch.equal(a[k], c[k]), k                                          # the background only touches rgb
    bgT = c["bg_transmittance"].cpu()
    o = onf.background_branch(rb.origins.cpu(), rb.directions.cpu(), rb.fars.cpu(), bgT, a["rgb"].cpu(), params, spec, bg_color.cpu())
    p64 = {k: v.double() for k, v in params.items()}
    o64 = onf.background_branch(rb.origins.cpu().double(), rb.directions.cpu().double(), rb.fars.cpu().double(), bgT.double(), a["rgb"].cpu().double(), p64,
                                spec, bg_color.cpu().double())
    check("merged rgb", c["rgb"], o["rgb"], o64["rgb"], 1e-4)
    if kind == "volsdf":      # bg_transmittance = the transmittance before the last sample (volsdf.py:67-68)
        rs, _ = sampler(rb, density_fn=field.laplace_density, sdf_fn=field.get_sdf)
        _, T = rs.get_weights_and_transmittance(field(rs)[sb.FieldHeadNames.DENSITY])
        assert torch.equal(c["bg_transmittance"], T[:, -1, :])


def test_neus_facto_style_merge():
    """forward_background_field_and_merge (base_surface_model.py:266-290) on the field's outputs: alpha and rgb outside the unit sphere."""
    f, params, spec = make_field("linf", "bf16x3")
    rs, o, d = ray_case(32, 48, seed=11)
    with torch.no_grad():
        out = f(rs)
    inside = (rs.frustums.get_start_positions().norm(dim=-1, keepdim=True) < 1.0).float()
    alpha_bg = rs.get_alphas(out[sb.FieldHeadNames.DENSITY])
    alpha_fg, rgb_fg = torch.full_like(alpha_bg, 0.3), torch.full_like(out[sb.FieldHeadNames.RGB], 0.7)
    alpha = alpha_fg * inside + (1.0 - inside) * alpha_bg
    rgb = rgb_fg * inside + (1.0 - inside) * out[sb.FieldHeadNames.RGB]
    eu = sb.rays.bins_of(rs).cpu()
    pos = onf.midpoints(o[:, None], d[:, None], eu[:, :-1, None], eu[:, 1:, None])
    o32, o64 = oracle_pair(pos, d[:, None].expand(*pos.shape), params, spec)
    ins = inside.cpu().double()
    deltas = (eu[:, 1:] - eu[:, :-1])[..., None].double()
    a64 = 0.3 * ins + (1 - ins) * (1 - torch.exp(-deltas * o64["density"]))
    a32 = 0.3 * ins + (1 - ins) * (1 - torch.exp(-deltas.float() * o32["density"]))
    check("merged alpha", alpha, a32, a64, 2e-4)
    check("merged rgb", rgb, 0.7 * ins + (1 - ins) * o32["rgb"], 0.7 * ins + (1 - ins) * o64["rgb"], 5e-5)
    assert float((1 - inside).sum()) > 0
