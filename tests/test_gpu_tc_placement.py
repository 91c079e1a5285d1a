"""-m gpu: placement and determinism of the fused tensor-core field kernel (k_field_tc) on the benchmark's field, at bf16x3 and bf16.

A row's outputs must not depend on which CTA, staging slot parity, 32-row chunk or encoder warp it lands in, nor on the run.  Each test
moves the rays, undoes the move and compares bit for bit:
- *rotate*: the ray order rolled by one ray, by 7 tiles' worth of rays and by one wave of 132 tiles' worth.  The set of rays stays the
  same, and so do the batch's depth range and depth clip, so this is the placement renders are held to.
- *slice*: sub-batches evaluated on their own against the whole batch (forward and sdf-only calls).

| axis | mechanism it exercises |
|---|---|
| rotate by one ray | every row in another 32-row chunk, encoder warp and staging-batch position; rays that straddle tiles in another tile |
| rotate by 7 tiles | the same rows per tile in another CTA (7 is not a multiple of 132) |
| rotate by one wave (132 tiles) | the same CTA one step later in its tile sequence: the other staging slot parity (tile n + 1 is staged while tile n runs) |
| slice from one ray (half a tile at S = 64) or from a tile boundary | another CTA, staging slot parity or position in the CTA's tile sequence |
| R = 2 * full + 1 at S = 64 (2 .. 266 tiles) | CTAs running 1, 2 and 3 tiles: the drain of the last tile after the loop at either head-input parity, ragged last tile |
| S = 128, 64, 32 | one ray per 32-row staging batch (direction encoding shared by shuffle); S > 32 spreads a ray over chunks of different warps, whose sums are added in chunk order |
| S = 16, 8 | several rays per staging batch and chunk, per-row direction encoding |
| S = 37, 24, 7 | rays straddle batches and tiles: the unfused field call, the ragged tile at R * S = 3 * 132 * 128 + 39 |
| determinism | no atomics in per-sample outputs or compositing: a difference is a race in the staging of the next tile or between encoder warps |

The fused render is also checked against the separate field and renderer calls of the same library (same per-sample bits, per-ray sums
within summation-order tolerance), and the points the encoder warps write against the exact-fp32 engine's."""
import pytest
import torch

from helpers import make_bundle

pytestmark = pytest.mark.gpu

PRECISIONS = ["bf16x3", "bf16"]
MODES = ["forward", "sdf_only", "render_alpha", "render_density"]
# every per-sample output the kernel writes
FORWARD = ["rgb", "density", "sdf", "normals", "gradients", "alpha", "occupancy", "points", "points_norm"]
RENDER = ["rgb", "depth", "normal", "accumulation", "bg_transmittance", "weights"]
BG = (0.9, 0.5, 0.1)
SEED = 7


def _tiles(S):
    """rays per 128-point tile (1 when a ray spans tiles)"""
    return max(1, 128 // S)


# (S, R): R = 300 tiles + one ray (> 2 x 132 CTAs: CTAs with two and three tiles, a ragged last tile)
ROTATE = [(S, 300 * _tiles(S) + 1) for S in (128, 64, 32, 24, 16, 7)]
# (S, R, slices [a, b)).  S = 64 puts two rays in a tile: R = 2 * full + 1 rays are full + 1 tiles on min(tiles, 132) CTAs, sliced from
# one ray (half a tile) or a whole number of tiles later
SLICE = [(64, R, ((1, R), (2 * 131 % R, R), (0, max(1, R - 3)), (R - 1, R))) for R in (2 * full + 1 for full in (1, 131, 132, 133, 264, 265))]
SLICE += [(37, 1000, ((1, 1000), (995, 1000), (0, 3))),               # 290 tiles
          (37, 1371, ((0, 7), (700, 763), (1330, 1371)))]            # 3 * 132 * 128 + 39 points: three full waves, a ragged tile
DETERMINISM = [(64, 601), (32, 1001), (8, 4001)]
BENCH = (128, 4096)                 # the benchmark batch, 31 tiles per CTA


@pytest.fixture(scope="module")
def field():
    """field(precision): the benchmark's SDFField, one per precision for the module"""
    import bench

    made = {}

    def at(precision):
        if precision not in made:
            made[precision] = bench.make_field(torch.device("cuda", 0), precision)
        return made[precision]

    return at


def _rays(R, seed=SEED):
    from sdfstudio_b200.synthetic import dtu_like_rays

    return dtu_like_rays(R, seed)


def _samples(rays, S):
    import sdfstudio_b200 as sb

    with torch.no_grad():
        return sb.UniformSampler(num_samples=S).eval()(make_bundle(*rays))


def _call(field, mode, rs):
    """the outputs of one call in `mode`, each viewed as [R, ...] so that a ray's outputs are one row"""
    import sdfstudio_b200 as sb

    R = sb.rays.bins_of(rs).shape[0]
    with torch.no_grad():
        if mode == "forward":
            o, d = sb.rays.rays_of(rs)
            eu = sb.rays.bins_of(rs)
            out = field._run(o, d, eu, eu.shape[1] - 1, FORWARD, apply_contraction=True)
        elif mode == "sdf_only":
            out = {"sdf": field.get_sdf(rs)}
        else:
            out = field.render(rs, torch.tensor(BG, device="cuda"), from_density=mode == "render_density")
            assert sorted(out) == sorted(RENDER)
    return {k: v.reshape(R, -1) for k, v in out.items()}


def _rotate_params():
    for S, R in ROTATE:
        for mode in MODES:
            if mode.startswith("render") and 128 % S:
                continue                    # the fused render needs whole rays per tile
            yield pytest.param(mode, S, R, id=f"{mode}-S{S}-R{R}")


@pytest.mark.parametrize("mode,S,R", list(_rotate_params()))
@pytest.mark.parametrize("precision", PRECISIONS)
def test_rotated_rays(field, precision, mode, S, R):
    """the batch against the same batch with its ray order rotated by one ray, 7 tiles' and 132 tiles' worth of rays"""
    f = field(precision)
    rays = _rays(R)
    base = _call(f, mode, _samples(rays, S))
    for k in (1, 7 * _tiles(S), 132 * 128 // S):
        moved = _call(f, mode, _samples(tuple(torch.roll(t, k, dims=0) for t in rays), S))
        for key, v in base.items():
            assert torch.equal(torch.roll(moved[key], -k, dims=0), v), (key, k)


@pytest.mark.parametrize("S,R,slices", [pytest.param(S, R, sl, id=f"S{S}-R{R}") for S, R, sl in SLICE])
@pytest.mark.parametrize("mode", ["forward", "sdf_only"])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_slices_equal_the_whole(field, precision, mode, S, R, slices):
    """slices of the batch evaluated on their own against the whole batch"""
    f = field(precision)
    rays = _rays(R)
    whole = _call(f, mode, _samples(rays, S))
    for a, b in slices:
        if a >= b:
            continue
        part = _call(f, mode, _samples(tuple(t[a:b] for t in rays), S))
        for key, v in part.items():
            assert torch.equal(whole[key][a:b], v), (key, a, b)


@pytest.mark.parametrize("S,R", DETERMINISM, ids=[f"S{S}-R{R}" for S, R in DETERMINISM])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("precision", PRECISIONS)
def test_deterministic(field, precision, mode, S, R):
    """the same call twice"""
    _assert_deterministic(field(precision), mode, S, R)


def test_bench_size_call_is_deterministic(field):
    """the benchmark batch's forward and sdf-only calls twice, at every precision"""
    for precision in PRECISIONS:
        for mode in ("forward", "sdf_only"):
            _assert_deterministic(field(precision), mode, *BENCH)


def test_bench_size_render_is_deterministic(field):
    """the benchmark batch's renders twice, at every precision"""
    for precision in PRECISIONS:
        for mode in ("render_alpha", "render_density"):
            _assert_deterministic(field(precision), mode, *BENCH)


def _assert_deterministic(f, mode, S, R):
    rs = _samples(_rays(R), S)
    first, second = _call(f, mode, rs), _call(f, mode, rs)
    for key, v in first.items():
        assert torch.equal(second[key], v), (mode, S, R, key)


# ----------------------------------------------------------------------------------------------------------------
# field + compositing in one call (sdfb200_field_render): fused into the kernel when 128 % S == 0
# ----------------------------------------------------------------------------------------------------------------
def _unfused(field, rs, bg, from_density, training=False):
    import sdfstudio_b200 as sb

    H = sb.FieldHeadNames
    out = field(rs, return_alphas=True)
    if from_density:
        w, T = rs.get_weights_and_transmittance(out[H.DENSITY])
        img = sb.render_all(w, out[H.RGB], out[H.NORMAL], rs, bg, training=training)
        img["weights"], img["bg_transmittance"] = w, T[:, -1, :]
    else:
        img = sb.render_from_alphas(out[H.ALPHA], out[H.RGB], out[H.NORMAL], rs, bg, training=training)
    return out, img


# S = 64 with R = 3, 265 and 529: 2, 133 and 265 tiles, CTAs with 1, 2 and 3 tiles whose last tile is drained at either head-input parity
FUSED = [(128, 300), (64, 601), (32, 77), (16, 1000), (8, 33), (1, 200), (37, 50), (64, 3), (64, 265), (64, 529)]


@pytest.mark.parametrize("S,R", FUSED, ids=[f"S{S}-R{R}" for S, R in FUSED])
@pytest.mark.parametrize("from_density", [False, True], ids=["alpha", "density"])
def test_fused_render_equals_field_plus_renderers(field, S, R, from_density):
    """field.render (one kernel: heads + compositing in registers) against the separate field + renderer calls of the same
    library on the same samples: identical per-sample arithmetic, compositing sums differ only in summation order."""
    import sdfstudio_b200 as sb

    f = field("bf16x3")
    rs = _samples(_rays(R), S)
    bg = torch.tensor(BG, device="cuda")
    with torch.no_grad():
        out, ref = _unfused(f, rs, bg, from_density)
        res = f.render(rs, bg, from_density=from_density, sample_outputs=("sdf", "gradients", "alpha"))
    H = sb.FieldHeadNames
    assert torch.equal(res["sdf"], out[H.SDF]) and torch.equal(res["gradients"], out[H.GRADIENT]) and torch.equal(res["alpha"], out[H.ALPHA])
    torch.testing.assert_close(res["weights"], ref["weights"], rtol=2e-6, atol=1e-7)
    for k in ("rgb", "depth", "normal", "accumulation", "bg_transmittance"):
        torch.testing.assert_close(res[k], ref[k], rtol=1e-5, atol=2e-6, msg=lambda m, k=k: f"{k}: {m}")


@pytest.mark.parametrize("background", ["last_sample", "per_ray"])
def test_fused_render_backgrounds_and_training_mode(field, background):
    f = field("bf16x3")
    R, S = 257, 64
    rs = _samples(_rays(R), S)
    bg = "last_sample" if background == "last_sample" else torch.rand(R, 3, generator=torch.Generator().manual_seed(3)).cuda()
    with torch.no_grad():
        out, ref = _unfused(f, rs, bg, False, training=True)
        res = f.render(rs, bg, training=True, want_weights=False)
    assert "weights" not in res
    for k in ("rgb", "depth", "normal", "accumulation"):
        torch.testing.assert_close(res[k], ref[k], rtol=1e-5, atol=2e-6, msg=lambda m, k=k: f"{k}: {m}")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_points_match_fp32_engine(field, precision):
    """points / points_norm (written by the encoder warps) against the exact-fp32 engine on the same samples"""
    rs = _samples(_rays(2 * 133 + 1), 64)
    tc, ref = _call(field(precision), "forward", rs), _call(field("fp32"), "forward", rs)
    assert torch.equal(tc["points"], ref["points"])
    assert torch.equal(tc["points_norm"], ref["points_norm"])
