"""-m gpu: hand-offs between tiles in the fused tensor-core field kernel.  The encoder warps stage tile n + 1 (geo input, Jacobians,
colour-static columns) in one of two per-CTA scratch slots while the consumers run tile n, so a row's result must not depend on
which CTA, which slot parity or which position in a CTA's tile sequence it lands in, nor on the run."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from helpers import make_bundle  # noqa: E402

pytestmark = pytest.mark.gpu

S = 64   # two rays per 128-point tile: an odd ray count leaves a ragged half tile at the end


def _field(precision):
    import bench

    return bench.make_field(torch.device("cuda", 0), precision)


def _samples(sb, R, seed):
    from sdfstudio_b200.synthetic import dtu_like_rays

    o, d, cam, nears, fars = dtu_like_rays(R, seed)
    with torch.no_grad():
        return sb.UniformSampler(num_samples=S).eval()(make_bundle(o, d, cam, nears, fars))


def _slice(sb, rs, a, b):
    o, d = sb.rays.rays_of(rs)
    eu = sb.rays.bins_of(rs)
    return o[a:b], d[a:b], eu[a:b]


def _run(field, o, d, eu, wants):
    with torch.no_grad():
        return field._run(o, d, eu, eu.shape[1] - 1, wants, apply_contraction=True)


FULL = ["rgb", "density", "sdf", "normals", "gradients", "alpha", "points", "points_norm"]


# tiles = full + 1 (ragged): 2, 132, 133, 134, 265 and 266 tiles on min(tiles, 132) CTAs, i.e. CTAs with 1, 2 and 3 tiles
@pytest.mark.parametrize("full", [1, 131, 132, 133, 264, 265])
@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("mode", ["full", "sdf_only"])
def test_tiles_equal_across_ctas_and_slot_parity(full, precision, mode):
    """The whole batch against slices of it that start one ray (half a tile) later or a whole number of tiles later: every row
    moves to another CTA, another staging slot parity or another position in its CTA's tile sequence, and must not change."""
    import sdfstudio_b200 as sb

    field = _field(precision)
    R = 2 * full + 1
    rs = _samples(sb, R, 11 + full)
    o, d, eu = _slice(sb, rs, 0, R)
    wants = FULL if mode == "full" else ["sdf"]
    whole = _run(field, o, d, eu, wants)
    for a, b in ((1, R), (2 * 131 % R, R), (0, max(1, R - 3)), (R - 1, R)):
        if a >= b:
            continue
        part = _run(field, o[a:b], d[a:b], eu[a:b], wants)
        for k in wants:
            assert torch.equal(whole[k][a * S:b * S], part[k]), (k, a, b)


def test_bench_size_call_is_deterministic():
    """The benchmark batch (4096 x 128, 31 tiles per CTA) twice: per-sample outputs carry no atomics, so any difference is a race in
    the staging of the next tile."""
    import sdfstudio_b200 as sb
    from sdfstudio_b200.synthetic import dtu_like_rays

    field = _field("bf16x3")
    o, d, cam, nears, fars = dtu_like_rays(4096, 1000)
    with torch.no_grad():
        rs = sb.UniformSampler(num_samples=128).eval()(make_bundle(o, d, cam, nears, fars))
    o, d = sb.rays.rays_of(rs)
    eu = sb.rays.bins_of(rs)
    first = _run(field, o, d, eu, FULL)
    second = _run(field, o, d, eu, FULL)
    for k in FULL:
        assert torch.equal(first[k], second[k]), k


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_points_match_generic_path(precision):
    """points / points_norm (written by the encoder warps) against the exact-fp32 engine on the same samples."""
    import sdfstudio_b200 as sb

    rs = _samples(sb, 2 * 133 + 1, 5)
    o, d = sb.rays.rays_of(rs)
    eu = sb.rays.bins_of(rs)
    tc = _run(_field(precision), o, d, eu, ["sdf", "points", "points_norm"])
    ref = _run(_field("fp32"), o, d, eu, ["sdf", "points", "points_norm"])
    assert torch.equal(tc["points"], ref["points"])
    assert torch.equal(tc["points_norm"], ref["points_norm"])
