"""-m gpu: the fused tensor-core field kernel in the regime bench.py runs it in -- many 128-point tiles per persistent CTA
(BASELINE configs[1]: 4096 rays x 128 samples, hash L=16 F=2 T=2^19, MLP 2x256, i.e. 4096 tiles on 132 CTAs = 31.0 tiles
per CTA), the tile loop / operand double buffering / mbarrier phase carry-over included.  The oracle (fp64) is evaluated on a
strided ray subset; rays are independent, so the subset pins the whole batch statistically while the oracle finishes in
seconds.  Reference: nerfstudio/fields/sdf_field.py:614-689 (get_outputs), cameras/rays.py:194-230, renderers.py:53-118,215-261.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from helpers import assert_within_noise, make_bundle, rel_err  # noqa: E402
from oracle import render, samplers  # noqa: E402
from oracle.field import FieldSpec, OracleField  # noqa: E402

pytestmark = pytest.mark.gpu

BENCH_SPEC = FieldSpec(num_layers=2, num_layers_color=2, hidden_dim=256, use_grid_feature=True, grid_layout="torch")


def _bench_field(precision, table_dtype="fp32"):
    import bench

    field = bench.make_field(torch.device("cuda", 0), precision, table_dtype=table_dtype)
    sd = {k: v.detach().cpu() for k, v in field.state_dict().items()}
    sd["hash_table"] = sd.pop("encoding.hash_table")
    if table_dtype == "fp16":
        sd["hash_table"] = sd["hash_table"].half().float()
    return field, OracleField(BENCH_SPEC, sd), OracleField(BENCH_SPEC, sd, dtype=torch.float64)


def _oracle_subset(o32, o64, o, d, cam, eu, idx):
    eu = eu[idx]
    e32 = o32.get_outputs(o[idx], d[idx], eu[:, :-1], eu[:, 1:] - eu[:, :-1], cam[idx], return_alphas=True)
    eu64 = eu.double()
    e64 = o64.get_outputs(o[idx].double(), d[idx].double(), eu64[:, :-1], eu64[:, 1:] - eu64[:, :-1], cam[idx], return_alphas=True)
    return e32, e64, eu64


def _check_heads(sb, out, e32, e64, idx, tag, floor_rel=1e-4):
    H = sb.FieldHeadNames
    for key, gk in ((H.SDF, "sdf"), (H.RGB, "rgb"), (H.ALPHA, "alphas"), (H.DENSITY, "density"), (H.GRADIENT, "gradients"), (H.NORMAL, "normals")):
        assert_within_noise(out[key][idx], e32[gk], e64[gk], f"{tag}/{gk}", factor=4.0, floor=floor_rel * float(e64[gk].abs().max()))


@pytest.mark.parametrize("precision,table_dtype", [("bf16x3", "fp32"), ("bf16x3", "fp16")])
def test_bench_config_multi_tile_parity(precision, table_dtype):
    """4096 rays x 128 samples at the benchmark's dtype: per-sample heads at the reference's fp32 noise level, rendered
    RGB / depth within 1e-4 relative of the oracle, on every 16th ray (256 rays, spread over all 132 CTAs and all tile slots)."""
    import sdfstudio_b200 as sb
    from sdfstudio_b200.synthetic import dtu_like_rays

    field, o32, o64 = _bench_field(precision, table_dtype)
    R, S = 4096, 128
    o, d, cam, nears, fars = dtu_like_rays(R, 1000)
    rb = make_bundle(o, d, cam, nears, fars)
    with torch.no_grad():
        rs = sb.UniformSampler(num_samples=S).eval()(rb)
        out = field(rs, return_alphas=True)
        img = sb.render_from_alphas(out[sb.FieldHeadNames.ALPHA], out[sb.FieldHeadNames.RGB], out[sb.FieldHeadNames.NORMAL], rs, torch.ones(3, device="cuda"))
    torch.cuda.synchronize()
    idx = torch.arange(5, R, 16)
    eu = sb.rays.bins_of(rs).cpu()
    e32, e64, eu64 = _oracle_subset(o32, o64, o, d, cam, eu, idx)
    _check_heads(sb, out, e32, e64, idx.cuda(), f"bench/{precision}/{table_dtype}")
    ow, _ = samplers.weights_from_alphas(e64["alphas"][..., 0])
    orgb = render.render_rgb(e64["rgb"], ow[..., None], torch.ones(3, dtype=torch.float64))
    assert rel_err(img["rgb"][idx.cuda()], orgb, 1e-2) < 1e-4
    gw, _ = samplers.weights_from_alphas(e32["alphas"][..., 0])
    gdep = render.render_depth(gw[..., None], eu[idx][:, :-1, None], eu[idx][:, 1:, None], "expected")
    odep = render.render_depth(ow[..., None], eu64[:, :-1, None], eu64[:, 1:, None], "expected")
    assert_within_noise(img["depth"][idx.cuda()], gdep, odep, "bench/depth", factor=4.0, floor=1e-4 * float(odep.abs().max()))
    onrm = render.render_semantics(e64["normals"], ow[..., None])
    assert rel_err(img["normal"][idx.cuda()], onrm, 1e-1) < 1e-4


def test_bench_config_fast_mode_psnr():
    """precision='bf16' (single pass) on the benchmark batch: reported with PSNR vs the oracle, like BASELINE's metric."""
    import sdfstudio_b200 as sb
    from sdfstudio_b200.synthetic import dtu_like_rays

    field, o32, o64 = _bench_field("bf16")
    R, S = 4096, 128
    o, d, cam, nears, fars = dtu_like_rays(R, 1000)
    rb = make_bundle(o, d, cam, nears, fars)
    with torch.no_grad():
        rs = sb.UniformSampler(num_samples=S).eval()(rb)
        out = field(rs, return_alphas=True)
        img = sb.render_from_alphas(out[sb.FieldHeadNames.ALPHA], out[sb.FieldHeadNames.RGB], out[sb.FieldHeadNames.NORMAL], rs, torch.ones(3, device="cuda"))
    idx = torch.arange(3, R, 16)
    _, e64, _ = _oracle_subset(o32, o64, o, d, cam, sb.rays.bins_of(rs).cpu(), idx)
    ow, _ = samplers.weights_from_alphas(e64["alphas"][..., 0])
    orgb = render.render_rgb(e64["rgb"], ow[..., None], torch.ones(3, dtype=torch.float64))
    mse = float(((img["rgb"][idx.cuda()].cpu().double() - orgb) ** 2).mean())
    psnr = -10.0 * torch.log10(torch.tensor(mse)).item()
    assert psnr > 55.0, f"fast-mode PSNR vs oracle {psnr:.1f} dB"


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_ragged_multi_tile_and_tile_boundaries(precision):
    """N = 3 * 132 * 128 + 39 points (a ragged last tile after three full waves), S = 37 so that rays straddle tile boundaries: a strided
    subset and the very last rays against the fp64 oracle.  That slices of this batch equal the whole bit for bit is checked in
    test_gpu_tc_placement.py."""
    import sdfstudio_b200 as sb
    from sdfstudio_b200.synthetic import dtu_like_rays

    field, o32, o64 = _bench_field(precision)
    R, S = 1371, 37
    assert R * S == 3 * 132 * 128 + 39
    o, d, cam, nears, fars = dtu_like_rays(R, 77)
    rb = make_bundle(o, d, cam, nears, fars)
    H = sb.FieldHeadNames
    with torch.no_grad():
        rs = sb.UniformSampler(num_samples=S).eval()(rb)
        out = field(rs, return_alphas=True)
    idx = torch.cat([torch.arange(0, R, 11), torch.arange(R - 3, R)])
    e32, e64, _ = _oracle_subset(o32, o64, o, d, cam, sb.rays.bins_of(rs).cpu(), idx)
    if precision == "bf16x3":
        _check_heads(sb, out, e32, e64, idx.cuda(), f"ragged/{precision}")
    else:
        assert rel_err(out[H.SDF][idx.cuda()], e64["sdf"], 1e-2) < 2e-2
        assert float((out[H.RGB][idx.cuda()].cpu().double() - e64["rgb"]).abs().max()) < 2e-2


def test_sdf_only_mode_multi_tile():
    """get_sdf (the samplers' sdf_fn: geo layers only, un-contracted positions) over > 3 waves of tiles."""
    import sdfstudio_b200 as sb
    from sdfstudio_b200.synthetic import dtu_like_rays

    field, o32, o64 = _bench_field("bf16x3")
    R, S = 2048, 64
    o, d, cam, nears, fars = dtu_like_rays(R, 31)
    rb = make_bundle(o, d, cam, nears, fars)
    with torch.no_grad():
        rs = sb.UniformSampler(num_samples=S).eval()(rb)
        sdf = field.get_sdf(rs)
    idx = torch.arange(1, R, 16)
    eu = sb.rays.bins_of(rs).cpu()[idx]
    s32 = o32.get_sdf(o[idx], d[idx], eu[:, :-1])
    s64 = o64.get_sdf(o[idx].double(), d[idx].double(), eu[:, :-1].double())
    assert_within_noise(sdf[idx.cuda()][..., 0], s32, s64, "get_sdf multi-tile", factor=4.0, floor=1e-4 * float(s64.abs().max()))


def test_fused_render_bench_config_vs_oracle():
    """The benchmark step itself (4096 x 128, one fused launch) against the fp64 oracle on every 16th ray: rendered RGB / depth /
    normal within 1e-4 relative (BASELINE north_star bound)."""
    import sdfstudio_b200 as sb
    from sdfstudio_b200.synthetic import dtu_like_rays

    field, o32, o64 = _bench_field("bf16x3")
    R, S = 4096, 128
    o, d, cam, nears, fars = dtu_like_rays(R, 1000)
    rb = make_bundle(o, d, cam, nears, fars)
    with torch.no_grad():
        rs = sb.UniformSampler(num_samples=S).eval()(rb)
        res = field.render(rs, torch.ones(3, device="cuda"))
    idx = torch.arange(7, R, 16)
    eu = sb.rays.bins_of(rs).cpu()
    e32, e64, eu64 = _oracle_subset(o32, o64, o, d, cam, eu, idx)
    ow, _ = samplers.weights_from_alphas(e64["alphas"][..., 0])
    orgb = render.render_rgb(e64["rgb"], ow[..., None], torch.ones(3, dtype=torch.float64))
    assert rel_err(res["rgb"][idx.cuda()], orgb, 1e-2) < 1e-4
    gw, _ = samplers.weights_from_alphas(e32["alphas"][..., 0])
    gdep = render.render_depth(gw[..., None], eu[idx][:, :-1, None], eu[idx][:, 1:, None], "expected")
    odep = render.render_depth(ow[..., None], eu64[:, :-1, None], eu64[:, 1:, None], "expected")
    assert_within_noise(res["depth"][idx.cuda()], gdep, odep, "fused/depth", factor=4.0, floor=1e-4 * float(odep.abs().max()))
    assert rel_err(res["normal"][idx.cuda()], render.render_semantics(e64["normals"], ow[..., None]), 1e-1) < 1e-4
    assert_within_noise(res["weights"][idx.cuda()][..., 0], gw, ow, "fused/weights", factor=4.0, floor=1e-5)
