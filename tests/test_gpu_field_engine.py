"""-m gpu: which engine runs a field call, seen through the library's kernel-launch counter.  The fused kernel is one launch per call; the
generic kernels launch one kernel per stage and GEMM, plus a weight pack per GEMM chunk when the GEMMs run on the tensor cores."""
import pytest
import torch

from helpers import launches

pytestmark = pytest.mark.gpu

SHAPES = {
    "neus-facto": dict(use_grid_feature=True, num_layers=2, num_layers_color=2, log2_hashmap_size=12),
    "volsdf": dict(num_layers=8, num_layers_color=4),
    "bakedsdf": dict(use_grid_feature=True, num_layers=2, num_layers_color=2, position_encoding_max_degree=8, use_diffuse_color=True,
                     use_specular_tint=True, use_reflections=True, use_n_dot_v=True, off_axis=True, log2_hashmap_size=12),
    "angelo": dict(use_grid_feature=True, num_layers=1, num_layers_color=4, use_numerical_gradients=True, hash_features_per_level=8,
                   hash_smoothstep=False, use_position_encoding=False, log2_hashmap_size=12, base_res=64, max_res=4096),
}
HEADS = ("sdf", "gradients", "normals", "rgb", "alpha")


def _samples(n_samples, n_rays=64):
    import sdfstudio_b200 as sb
    from sdfstudio_b200.synthetic import dtu_like_rays

    o, d, cam, nears, fars = dtu_like_rays(n_rays, 3)
    dev = torch.device("cuda")
    rb = sb.RayBundle(origins=o.to(dev), directions=d.to(dev), pixel_area=torch.ones(n_rays, 1, device=dev),
                      directions_norm=torch.ones(n_rays, 1, device=dev), camera_indices=cam.view(n_rays, 1).to(dev), nears=nears.to(dev),
                      fars=fars.to(dev))
    return sb.UniformSampler(num_samples=n_samples).eval()(rb)


def _field(shape, precision):
    import sdfstudio_b200 as sb

    torch.manual_seed(0)
    return sb.SDFField(sb.SDFFieldConfig(**SHAPES[shape], precision=precision), torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), 49).cuda().eval()


def _forward_launches(shape, precision, wants=HEADS, n_samples=32):
    import sdfstudio_b200 as sb

    field, rs = _field(shape, precision), _samples(n_samples)
    origins, directions = sb.rays.rays_of(rs)
    bins = sb.rays.bins_of(rs)
    return launches(lambda: field._run(origins, directions, bins, n_samples, wants, True))


def _render_launches(shape, precision, n_samples, clip_depth):
    field, rs = _field(shape, precision), _samples(n_samples)
    return launches(lambda: field.render(rs, torch.ones(3, device="cuda"), clip_depth=clip_depth))


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_fused_family_runs_one_launch(precision):
    assert _forward_launches("neus-facto", precision) == 1
    assert _forward_launches("neus-facto", precision, wants=("sdf",)) == 1
    assert _render_launches("neus-facto", precision, 32, clip_depth=False) == 1
    assert _render_launches("neus-facto", precision, 32, clip_depth=True) == 2             # + the global depth clip


def test_exact_engine_launches_like_fp32():
    """the fused family asking for geo_feature, and numerical gradients, run the exact-fp32 engine at a tensor-core precision"""
    geo = HEADS + ("geo_feature",)
    assert _forward_launches("neus-facto", "bf16x3", wants=geo) == _forward_launches("neus-facto", "fp32", wants=geo)
    assert _forward_launches("angelo", "bf16x3") == _forward_launches("angelo", "fp32")


@pytest.mark.parametrize("shape", ["volsdf", "bakedsdf"])
def test_generic_tensor_core_engine_packs_per_gemm_chunk(shape):
    assert _forward_launches(shape, "bf16x3") > _forward_launches(shape, "fp32")


def test_render_without_whole_rays_per_tile_is_composed():
    """S = 96 does not divide the 128-point tile: the field call (fused, one launch) is followed by the compositing kernels"""
    assert _render_launches("neus-facto", "bf16x3", 96, clip_depth=False) > 1
