"""-m gpu: the per-point heads and the fused compositing of the tensor-core field kernel, which run in an encoder warp one tile behind
the consumers (head inputs double-buffered by tile parity, the last tile drained after the tile loop).  Rays longer than 32 samples
span several 32-row chunks of a tile; their sums are combined chunk by chunk in a fixed order, so a render is deterministic."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from helpers import make_bundle  # noqa: E402

pytestmark = pytest.mark.gpu

RENDER_KEYS = ("rgb", "depth", "normal", "accumulation", "bg_transmittance", "weights")


def _field(precision="bf16x3"):
    import bench

    return bench.make_field(torch.device("cuda", 0), precision)


def _samples(sb, R, S, seed):
    from sdfstudio_b200.synthetic import dtu_like_rays

    o, d, cam, nears, fars = dtu_like_rays(R, seed)
    with torch.no_grad():
        return sb.UniformSampler(num_samples=S).eval()(make_bundle(o, d, cam, nears, fars))


@pytest.mark.parametrize("S,R", [(128, 4096), (64, 601), (32, 1001), (8, 4001)])
@pytest.mark.parametrize("from_density", [False, True])
def test_fused_render_is_deterministic(S, R, from_density):
    """Two identical fused renders agree bit for bit, per-ray sums included (no atomics in the compositing)."""
    import sdfstudio_b200 as sb

    field = _field()
    rs = _samples(sb, R, S, 7 + S)
    bg = torch.tensor([0.9, 0.5, 0.1], device="cuda")
    with torch.no_grad():
        first = field.render(rs, bg, from_density=from_density)
        second = field.render(rs, bg, from_density=from_density)
    for k in RENDER_KEYS:
        assert torch.equal(first[k], second[k]), k


# S = 64: two rays per tile, an odd ray count leaves a ragged last tile.  2, 133 and 265 tiles on min(tiles, 132) CTAs: the CTAs run
# 1, 2 and 3 tiles, so the heads warp drains a last tile of either head-input parity
@pytest.mark.parametrize("R", [3, 265, 529])
@pytest.mark.parametrize("from_density", [False, True])
def test_fused_render_tiles_per_cta(R, from_density):
    import sdfstudio_b200 as sb

    H = sb.FieldHeadNames
    field = _field()
    rs = _samples(sb, R, 64, 31 + R)
    bg = torch.tensor([0.9, 0.5, 0.1], device="cuda")
    with torch.no_grad():
        out = field(rs, return_alphas=True)
        if from_density:
            w, T = rs.get_weights_and_transmittance(out[H.DENSITY])
            ref = sb.render_all(w, out[H.RGB], out[H.NORMAL], rs, bg)
            ref["weights"], ref["bg_transmittance"] = w, T[:, -1, :]
        else:
            ref = sb.render_from_alphas(out[H.ALPHA], out[H.RGB], out[H.NORMAL], rs, bg)
        res = field.render(rs, bg, from_density=from_density, sample_outputs=("sdf", "gradients", "alpha"))
    assert torch.equal(res["sdf"], out[H.SDF]) and torch.equal(res["gradients"], out[H.GRADIENT]) and torch.equal(res["alpha"], out[H.ALPHA])
    torch.testing.assert_close(res["weights"], ref["weights"], rtol=2e-6, atol=1e-7)
    for k in ("rgb", "depth", "normal", "accumulation", "bg_transmittance"):
        torch.testing.assert_close(res[k], ref[k], rtol=1e-5, atol=2e-6, msg=lambda m, k=k: f"{k}: {m}")


FULL = ["rgb", "density", "sdf", "normals", "gradients", "alpha"]


@pytest.mark.parametrize("mode", ["full", "sdf_only"])
def test_unfused_heads_match_a_big_call(mode):
    """37 samples per ray (rays straddle tiles, 290 tiles: up to 3 per CTA): slices of the batch against the whole batch, bit for bit.
    In sdf-only mode the kernel runs no heads at all."""
    import sdfstudio_b200 as sb

    field = _field()
    R, S = 1000, 37
    rs = _samples(sb, R, S, 3)
    o, d = sb.rays.rays_of(rs)
    eu = sb.rays.bins_of(rs)
    wants = FULL if mode == "full" else ["sdf"]
    with torch.no_grad():
        whole = field._run(o, d, eu, S, wants, apply_contraction=True)
        for a, b in ((1, R), (R - 5, R), (0, 3)):
            part = field._run(o[a:b], d[a:b], eu[a:b], S, wants, apply_contraction=True)
            for k in wants:
                assert torch.equal(whole[k][a * S:b * S], part[k]), (k, a, b)
