"""-m gpu: the heads and the per-ray compositing of the fused tensor-core field kernel run on the three encoder warps, 32-row chunks
each, with the chunks of a ray longer than 32 samples spread over different warps.  A ray's rendered outputs must not depend on which
CTA, staging-slot parity, chunk or warp it lands in, nor on the run."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from helpers import make_bundle  # noqa: E402

pytestmark = pytest.mark.gpu

TILES = 300                         # > 2 x 132: CTAs with two and three tiles
KEYS = ["rgb", "depth", "normal", "accumulation", "weights", "bg_transmittance"]


def _field(precision):
    import bench

    return bench.make_field(torch.device("cuda", 0), precision)


def _render(sb, field, rays, S, from_density):
    o, d, cam, nears, fars = rays
    with torch.no_grad():
        rs = sb.UniformSampler(num_samples=S).eval()(make_bundle(o, d, cam, nears, fars))
        return field.render(rs, torch.ones(3, device="cuda"), from_density=from_density)


def _roll(rays, k):
    return tuple(torch.roll(t, k, dims=0) for t in rays)


@pytest.mark.parametrize("S", [128, 64, 32, 16])
@pytest.mark.parametrize("from_density", [False, True], ids=["alpha", "density"])
@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_render_equal_when_rays_move(S, from_density, precision):
    """The batch against the same batch with its ray order rotated by one ray and by 7 tiles (not a multiple of 132 CTAs): every ray
    lands in another CTA, slot parity, chunk and owning warp.  The set of rays is the same, so the depth range and the depth clip are
    too, and every per-ray output must be bit-identical once the order is undone."""
    import sdfstudio_b200 as sb
    from sdfstudio_b200.synthetic import dtu_like_rays

    field = _field(precision)
    R = TILES * (128 // S) + 1          # a ragged last tile
    rays = dtu_like_rays(R, 23 + S)
    base = _render(sb, field, rays, S, from_density)
    for k in (1, 7 * (128 // S)):
        moved = _render(sb, field, _roll(rays, k), S, from_density)
        for key in KEYS:
            assert torch.equal(torch.roll(moved[key], -k, dims=0), base[key]), (key, k)


def test_bench_size_render_is_deterministic():
    """The benchmark batch (4096 x 128, 31 tiles per CTA) rendered twice: the chunk sums of a ray are added in a fixed order whatever
    warp produced them, so any difference is a race between the encoder warps."""
    import sdfstudio_b200 as sb
    from sdfstudio_b200.synthetic import dtu_like_rays

    field = _field("bf16x3")
    rays = dtu_like_rays(4096, 1000)
    first = _render(sb, field, rays, 128, False)
    second = _render(sb, field, rays, 128, False)
    for key in KEYS:
        assert torch.equal(first[key], second[key]), key
