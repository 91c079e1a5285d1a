"""GPU: the marching-cubes kernel against its numpy restatement (oracle/marching_cubes.py), the mesh-extraction drop-ins against the
golden minted from the unmodified reference, and extract_mesh on an SDFField."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import marching_cubes as omc
from test_meshing_cpu import (GOLDEN_CASES, directed_edges_balance, noise_volume, read_ply, sphere_volume, torus_volume,
                                    two_spheres_volume, undirected_edge_counts)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def kernel(vol, level=0.0, spacing=(1.0, 1.0, 1.0), mask=None):
    from sdfstudio_b200 import meshing

    m = None if mask is None else torch.from_numpy(np.asarray(mask)).cuda()
    v, f, n = meshing.marching_cubes(torch.from_numpy(np.ascontiguousarray(vol)).cuda(), level, spacing, m)
    return v.cpu().numpy(), f.cpu().numpy(), n.cpu().numpy()


def assert_same(vol, level=0.0, spacing=(1.0, 1.0, 1.0), mask=None):
    V, F, N = kernel(vol, level, spacing, mask)
    v, f, n = omc.marching_cubes(vol, level, spacing, mask)
    assert V.shape == v.shape and F.shape == f.shape
    assert np.array_equal(V, v), np.abs(V - v).max()
    assert np.array_equal(F.astype(np.int64), f)
    assert np.abs(N - n).max(initial=0.0) <= 1e-6
    return V, F, N


def _volumes():
    rng = np.random.default_rng(5)
    ex = rng.standard_normal((17, 33, 9)).astype(np.float32)
    return {
        "sphere": (sphere_volume(64), 0.0, (0.1, 0.2, 0.3)),
        "torus": (torus_volume(48), 0.0, (1.0, 1.0, 1.0)),
        "two_spheres": (two_spheres_volume(40), 0.0, (1.0, 1.0, 1.0)),
        "noise": (noise_volume(60), 0.5, (1.0, 1.0, 1.0)),
        "non_cubic": (ex, 0.1, (0.5, 1.0, 2.0)),
        "extent_2": (rng.standard_normal((2, 2, 2)).astype(np.float32) + np.array([-1, 1], np.float32), 0.0, (1.0, 1.0, 1.0)),
        "extent_2x7x2": (rng.standard_normal((2, 7, 2)).astype(np.float32), 0.0, (1.0, 1.0, 1.0)),
        "at_level": (np.round(sphere_volume(30) * 4).astype(np.float32), 0.0, (1.0, 1.0, 1.0)),
    }


@pytest.mark.parametrize("name", list(_volumes()))
def test_kernel_matches_oracle(name):
    vol, level, spacing = _volumes()[name]
    V, F, N = assert_same(vol, level, spacing)
    assert np.isfinite(V).all() and np.isfinite(N).all()
    if name in ("sphere", "torus", "two_spheres"):
        assert (undirected_edge_counts(F) == 2).all()
    if name == "noise":
        assert directed_edges_balance(F)


def test_kernel_masks_match_oracle():
    rng = np.random.default_rng(1)
    for vol, level in ((sphere_volume(40), 0.0), (noise_volume(30), 0.5)):
        for p in (0.1, 0.5, 0.9):
            mask = (rng.random(vol.shape) < p).astype(np.uint8)
            V, F, _ = assert_same(vol, level, mask=mask)
            assert len(np.unique(F)) == len(V)


def test_kernel_empty_extents_and_reruns():
    for shape in ((1, 8, 8), (8, 1, 8), (8, 8, 1), (1, 1, 1)):
        V, F, N = kernel(np.random.default_rng(0).standard_normal(shape).astype(np.float32))
        assert V.shape == (0, 3) and F.shape == (0, 3)
    assert kernel(np.ones((9, 9, 9), np.float32))[1].shape == (0, 3)
    vol = noise_volume(50)
    a, b = kernel(vol, 0.5), kernel(vol, 0.5)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))


def test_nonfinite_volume_raises():
    from sdfstudio_b200 import meshing

    vol = torch.zeros(8, 8, 8, device="cuda")
    for bad in (float("nan"), float("inf"), -float("inf")):
        v = vol.clone()
        v[3, 4, 5] = bad
        with pytest.raises(ValueError):
            meshing.marching_cubes(v)


def _field(precision="fp32"):
    import sdfstudio_b200 as sb
    from sdfstudio_b200 import synthetic

    # an object-centred sphere of radius 0.5 at initialisation (inside_outside=False), perturbed: a closed surface inside the box
    cfg = sb.SDFFieldConfig(use_grid_feature=True, num_layers=2, num_layers_color=2, inside_outside=False, bias=0.5, precision=precision)
    torch.manual_seed(0)                                                 # the geometric initialisation draws from the global RNG
    f = sb.SDFField(cfg, torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), num_images=49).cuda().eval()
    return recentre_(synthetic.perturb_field_(f, seed=0))


def recentre_(field):
    """shifts the SDF head's bias so that the SDF is -0.5 at the origin: the perturbation moves the initial sphere's level by up to ~0.8,
    which can leave the box without a surface."""
    from sdfstudio_b200 import meshing

    with torch.no_grad():
        s0 = meshing.sdf_fn(field)(torch.zeros(1, 3, device="cuda")).item()
        getattr(field, f"glin{field.num_layers - 2}").bias[0] -= s0 + 0.5
    return field


def test_kernel_matches_oracle_on_a_field_block():
    from sdfstudio_b200 import meshing

    vol = meshing.evaluate_sdf_grid(_field("bf16x3"), 512, chunk=1 << 20).cpu().numpy()
    assert vol.min() < 0 < vol.max(), (vol.min(), vol.max())
    h = 2.0 / 511
    V, F, _ = assert_same(vol, 0.0, (h, h, h))
    assert len(F) > 10000


def test_more_than_2_31_points():
    """a 1300^3 volume (2.2e9 points) holding a sphere in its last slab meshes like the slab alone, shifted by the slab offset."""
    n, i0 = 1300, 1240
    vol = torch.empty(n, n, n, device="cuda")
    j = torch.arange(n, device="cuda", dtype=torch.float32)
    c = (1270.0, 650.0, 650.0)
    for s in range(0, n, 100):
        i = j[s:s + 100]
        vol[s:s + 100] = torch.sqrt((i[:, None, None] - c[0]) ** 2 + (j[None, :, None] - c[1]) ** 2 + (j[None, None, :] - c[2]) ** 2) - 20.0
    from sdfstudio_b200 import meshing

    V, F, N = (t.cpu().numpy() for t in meshing.marching_cubes(vol))
    slab = vol[i0:].contiguous()
    del vol
    v, f, nn = (t.cpu().numpy() for t in meshing.marching_cubes(slab))
    assert len(F) > 1000 and np.array_equal(F, f)
    assert np.array_equal(V[:, 1:], v[:, 1:]) and np.abs(V[:, 0] - (v[:, 0] + i0)).max() <= 1e-3
    assert np.abs(N - nn).max() <= 1e-6


# ---------------------------------------------------------------------------------------------------------------------------------
# the drop-ins against the reference golden
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_dropins_match_reference_golden(name, monkeypatch, tmp_path):
    from oracle import make_golden_marching_cubes as mk
    from sdfstudio_b200 import meshing

    with open(os.path.join(ROOT, "tests", "golden", "marching_cubes.json")) as fh:
        want = json.load(fh)["cases"][name]
    arr = np.load(os.path.join(ROOT, "tests", "golden", "marching_cubes.npz"))
    calls = []
    block_mesh = meshing._block_mesh

    def record(volume, level, spacing, mask, offset):
        calls.append(dict(volume=volume.cpu().numpy(), level=level, spacing=list(spacing), mask=None if mask is None else mask.cpu().numpy(),
                          offset=[float(o) for o in offset]))
        return block_mesh(volume, level, spacing, mask, offset)

    monkeypatch.setattr(meshing, "_block_mesh", record)
    fn, kw, f = mk.cases()[name]
    kw = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in kw.items()}
    f_cuda = lambda x: f(x)
    out = tmp_path / "m.ply"
    if fn == "get_surface_occupancy":
        mesh = meshing.get_surface_occupancy(f_cuda, **kw, output_path=out, return_mesh=True)
    else:
        mesh = getattr(meshing, fn)(f_cuda, **kw, output_path=out, return_mesh=True, simplify_mesh=False)
    assert len(calls) == len(want) > 0
    flips = total = 0
    for n, (g, w) in enumerate(zip(calls, want)):
        assert g["level"] == w["level"] and g["spacing"] == w["spacing"] and g["offset"] == w["offset"]
        assert list(g["volume"].shape) == w["shape"]
        # CUDA's AvgPool3d sums in another order than the CPU's: a pyramid point within that noise of a threshold may flip its mask
        got = np.concatenate([g["volume"].reshape(-1)[arr[f"{name}/{n}/cross_idx"]], g["volume"][g["volume"].shape[0] // 2, ::4, ::4].reshape(-1)])
        ref = np.concatenate([arr[f"{name}/{n}/cross_val"], arr[f"{name}/{n}/slice"].reshape(-1)])
        # the analytic callables themselves round differently on the device (norm, sqrt, sigmoid): a few ulp of their inputs' scale
        close = np.abs(got - ref) <= 8 * np.finfo(np.float32).eps * np.maximum(1.0, np.abs(ref))
        flips += int((~close).sum())
        total += got.size
        if w["mask_count"] is not None:
            assert abs(int(g["mask"].sum()) - w["mask_count"]) <= 1e-4 * w["mask_count"]
    assert flips <= 1e-3 * total, (flips, total)
    assert len(mesh.faces) > 0 and np.isfinite(mesh.vertices).all()


# ---------------------------------------------------------------------------------------------------------------------------------
# extract_mesh on an SDFField
# ---------------------------------------------------------------------------------------------------------------------------------
def test_sdf_callable_matches_forward_geonetwork():
    """sdf_fn (the sdf-only mode) against the reference's callable, forward_geonetwork(x)[:, 0] (sdf + geo features).  Bound found on
    the H100: bit-identical at fp32; at bf16x3 the two modes differ by up to 1.2e-5 (SDF values of order 1)."""
    from sdfstudio_b200 import meshing

    for precision, bound in (("fp32", 0.0), ("bf16x3", 5e-5)):
        field = _field(precision)
        x = torch.rand(1 << 18, 3, device="cuda", generator=torch.Generator("cuda").manual_seed(0)) * 2 - 1
        with torch.no_grad():
            a = meshing.sdf_fn(field)(x)
            b = field.forward_geonetwork(x)[:, 0].contiguous()
        assert (a - b).abs().max().item() <= bound, (precision, (a - b).abs().max().item())


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_extract_mesh_on_a_field(precision, tmp_path):
    from sdfstudio_b200 import meshing

    field = _field(precision)
    out = tmp_path / "sub" / "mesh.ply"
    meshing.extract_mesh(field, resolution=512, output_path=out)
    V, F, N = read_ply(out)
    assert len(F) > 10000
    # Vertices lie within the edge-interpolation bound of the zero level, a lattice step h times the SDF's slope (~1; bound 2h), where the
    # pyramid evaluated both ends of the edge at the finest level.  Where it stopped at a coarser level (|coarse SDF| above that level's
    # threshold, at most 2 * 2 / 512 * 8) the edge carries values upsampled from up to 8 fine steps away.  Measured on an H100: 99.7 % of
    # the vertices within 2h at fp32 and at bf16x3, the largest miss 0.046.
    h = 2.0 / 511
    s = meshing.sdf_fn(field)(torch.from_numpy(V).cuda()).abs()
    assert s.max().item() <= 2 * 2 / 512 * 8 + 8 * h
    assert (s <= 2 * h).float().mean().item() >= 0.98
    # where the surface is closed in the box (no vertex on the box's faces) the welded mesh is closed
    if (np.abs(V) < 1 - h / 2).all():
        assert (undirected_edge_counts(F.astype(np.int64)) == 2).all()


def test_extract_mesh_occupancy(tmp_path):
    from sdfstudio_b200 import meshing

    field = _field("fp32")
    out = tmp_path / "occ.ply"
    mesh = meshing.get_surface_occupancy(lambda x: torch.sigmoid(10 * meshing.sdf_fn(field)(x)), resolution=200, level=0.5,
                                         output_path=out, return_mesh=True)
    meshing.extract_mesh(field, resolution=200, output_path=tmp_path / "occ2.ply", is_occupancy=True)
    V, F, _ = read_ply(tmp_path / "occ2.ply")
    assert len(F) == len(mesh.faces) > 0
    occ = torch.sigmoid(10 * meshing.sdf_fn(field)(torch.from_numpy(V).cuda()))
    assert (occ - 0.5).abs().max().item() < 0.05
