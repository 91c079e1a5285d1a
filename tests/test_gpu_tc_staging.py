"""-m gpu: the encoder warps of the fused tensor-core field kernel stage a tile in 32-row batches.  A batch whose rows are all samples of
one ray evaluates the direction encoding once and shares it across the warp; a batch holding several rays evaluates it per row.  That
may not show in the outputs: a sample's and a ray's outputs must not depend on where in a batch or tile the ray lands."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from helpers import make_bundle  # noqa: E402

pytestmark = pytest.mark.gpu

TILES = 300                         # > 2 x 132: CTAs with two and three tiles
RENDER_KEYS = ["rgb", "depth", "normal", "accumulation", "weights", "bg_transmittance"]


def _field():
    import bench

    return bench.make_field(torch.device("cuda", 0), "bf16x3")


def _samples(sb, rays, S):
    o, d, cam, nears, fars = rays
    with torch.no_grad():
        return sb.UniformSampler(num_samples=S).eval()(make_bundle(o, d, cam, nears, fars))


def _roll(rays, k):
    return tuple(torch.roll(t, k, dims=0) for t in rays)


def _undo(t, k, R, S):
    """t of the batch rotated by k rays, back in the original ray order (per-ray or per-sample leading dimension)."""
    if t.shape[0] == R:
        return torch.roll(t, -k, dims=0)
    assert t.shape[0] == R * S, t.shape
    return torch.roll(t, -k * S, dims=0)


@pytest.mark.parametrize("S", [128, 64, 32, 24, 16, 7])
def test_staging_equal_when_rays_move(S):
    """Forward (per-sample outputs), get_sdf and, where a tile holds whole rays (128 % S == 0), the fused render of a batch against the
    same batch with its ray order rotated by one ray and by 7 tiles' worth of rays.  S >= 32 with 128 % S == 0 gives one-ray batches,
    S = 16 two rays per batch, S = 24 and 7 rays that straddle batches and tiles (unfused).  Bit-identical once the order is undone."""
    import sdfstudio_b200 as sb
    from sdfstudio_b200.synthetic import dtu_like_rays

    field = _field()
    R = TILES * max(1, 128 // S) + 1    # a ragged last tile
    rays = dtu_like_rays(R, 31 + S)
    base_rs = _samples(sb, rays, S)
    with torch.no_grad():
        base_fwd = field(base_rs, return_alphas=True)
        base_sdf = field.get_sdf(base_rs)
        base_img = field.render(base_rs, torch.ones(3, device="cuda")) if 128 % S == 0 else None
    for k in (1, 7 * max(1, 128 // S)):
        rs = _samples(sb, _roll(rays, k), S)
        with torch.no_grad():
            fwd = field(rs, return_alphas=True)
            sdf = field.get_sdf(rs)
            img = field.render(rs, torch.ones(3, device="cuda")) if base_img is not None else None
        for key, v in base_fwd.items():
            if torch.is_tensor(v):
                assert torch.equal(_undo(fwd[key], k, R, S), v), (key, k)
        assert torch.equal(_undo(sdf, k, R, S), base_sdf), k
        if img is not None:
            for key in RENDER_KEYS:
                assert torch.equal(_undo(img[key], k, R, S), base_img[key]), (key, k)
