"""CPU: the two restatements of the reference's TSDF fusion (oracle/tsdf.py) against the golden minted from the unmodified reference
(oracle/make_golden_tsdf.py), and the host side of sdfstudio_b200/tsdf.py: signatures and defaults, the Cameras additions, the
argument errors and the C-ABI error codes.

(b), the kernel's op order in numpy float32, differs from (a), the reference's ATen ops, in the summation order inside ``bmm`` and in
the CPU ``grid_sample``'s unnormalisation.  The camera coordinates then differ by a few ulp of their magnitude, so the voxel depth does
too: with |camera coordinates| <= 4 and a truncation >= 0.6 here, a fused value moves by at most ~4 * 2^-23 * 4 / 0.6 ~ 3e-6 per image,
and a running average of such values stays within VALUE_ATOL.  A pixel or validity decision differs only where the two orders straddle
a rounding tie (a pixel coordinate within a few ulp of .5) or the validity boundary (dist within a few ulp of -truncation, or 0)."""
import dataclasses
import inspect
import json
import os
import types

import numpy as np
import pytest
import torch

from oracle import tsdf as ot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
VALUE_ATOL = 2e-5
EPS = float(np.finfo(np.float32).eps)


def golden():
    return np.load(os.path.join(GOLDEN, "tsdf.npz")), json.load(open(os.path.join(GOLDEN, "tsdf.json")))


GOLDEN_CASES = sorted(golden()[1]["cases"])


def case(name):
    """(aabb, dims, c2w, K, depth [B,1,H,W], color [B,3,H,W], batch_size) of a golden case as CPU tensors."""
    z, meta = golden()
    g = lambda k: torch.from_numpy(z[f"{name}/{k}"])  # noqa: E731
    return g("aabb"), g("dims"), g("c2w"), g("K"), g("depth"), g("color"), meta["cases"][name]["batch_size"]


def oracle_a(name, device="cpu"):
    """(voxel_coords, values, weights, colors, voxel_size, origin) after the reference's batches, by restatement (a)."""
    aabb, dims, c2w, K, depth, color, bs = case(name)
    st = [t.to(device) for t in ot.from_aabb(aabb, dims)]
    ot.integrate_batched(st[:4], ot.truncation(st[4]), c2w.to(device), K.to(device), depth.to(device), color.to(device), bs)
    return st


def oracle_b(name):
    """(values [N], weights [N], colors [N,3], per-image trace) by restatement (b), all images in order from the initial state."""
    aabb, dims, c2w, K, depth, color, _ = case(name)
    vc, v, w, c, vs, _ = ot.from_aabb(aabb, dims)
    return ot.integrate_ops(vc.reshape(3, -1).numpy(), v.reshape(-1).numpy(), w.reshape(-1).numpy(), c.reshape(-1, 3).numpy(),
                            np.float32(ot.truncation(vs)), ot.pack_cams(c2w, K).numpy(), depth[:, 0].numpy(), color.numpy())


def near_boundary(name, voxels, ulps=8):
    """For each voxel index, whether some image puts it within ``ulps`` ulp of a pixel rounding tie or of the validity boundary."""
    aabb, dims, c2w, K, depth, color, _ = case(name)
    vc, _, _, _, vs, _ = ot.from_aabb(aabb, dims)
    xyz = vc.reshape(3, -1).numpy()[:, voxels].astype(np.float64)
    cams = ot.pack_cams(c2w, K).numpy().astype(np.float64)
    trunc = float(ot.truncation(vs))
    B, _, H, W = depth.shape
    near = np.zeros(len(voxels), bool)
    with np.errstate(all="ignore"):
        for b in range(B):
            m = cams[b]
            cx, cy, cz = (m[r] * xyz[0] + m[r + 1] * xyz[1] + m[r + 2] * xyz[2] + m[r + 3] for r in (0, 4, 8))
            cy, cz = -cy, -cz
            vd = np.sqrt(cx * cx + cy * cy + cz * cz)
            for p, size in ((m[12] * cx / cz + m[13] * cy / cz + m[14], W), (m[15] * cx / cz + m[16] * cy / cz + m[17], H)):
                f = ((2 * p / size - 1) + 1) * size / 2 - 0.5
                near |= np.abs(f - np.floor(f) - 0.5) <= ulps * EPS * np.maximum(1, np.abs(f))
            ix = np.rint(((2 * (m[12] * cx / cz + m[13] * cy / cz + m[14]) / W - 1) + 1) * W / 2 - 0.5)
            iy = np.rint(((2 * (m[15] * cx / cz + m[16] * cy / cz + m[17]) / H - 1) + 1) * H / 2 - 0.5)
            ok = (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
            sd = np.where(ok, depth[b, 0].numpy()[np.clip(iy, 0, H - 1).astype(int), np.clip(ix, 0, W - 1).astype(int)], 0)
            near |= np.abs(sd - vd + trunc) <= ulps * EPS * np.maximum(1, np.abs(vd))
            near |= np.abs(vd) <= ulps * EPS
    return near


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_oracle_a_matches_reference(name):
    """from_aabb's fields and the fused values, weights and colours after the reference's batches are reproduced bit for bit."""
    z, _ = golden()
    aabb, dims = case(name)[:2]
    for k, t in zip(("voxel_coords", "values", "weights", "colors", "voxel_size", "origin"), ot.from_aabb(aabb, dims)):
        assert torch.equal(t, torch.from_numpy(z[f"{name}/init_{k}"])), k
    st = oracle_a(name)
    for k, t in (("values", st[1]), ("weights", st[2]), ("colors", st[3])):
        assert np.array_equal(t.numpy(), z[f"{name}/{k}"], equal_nan=True), k


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_oracle_b_against_a(name):
    """(b) takes (a)'s pixel and validity everywhere except voxels on a rounding or validity boundary, which are counted; values agree
    within VALUE_ATOL elsewhere."""
    z, _ = golden()
    v, w, c, _ = oracle_b(name)
    ref_v, ref_w, ref_c = z[f"{name}/values"].reshape(-1), z[f"{name}/weights"].reshape(-1), z[f"{name}/colors"].reshape(-1, 3)
    flips = np.nonzero((w != ref_w) | (c != ref_c).any(1))[0]
    assert near_boundary(name, flips).all(), flips[~near_boundary(name, flips)]
    assert len(flips) <= max(2, len(ref_v) // 1000), len(flips)
    same = np.ones(len(ref_v), bool)
    same[flips] = False
    assert np.abs(v[same] - ref_v[same]).max() <= VALUE_ATOL
    print(f"{name}: {len(flips)} boundary voxels, max |value - reference| = {np.abs(v[same] - ref_v[same]).max():.2e}")


def test_golden_covers_the_rules():
    """The golden cases reach every rule the kernel documents: out-of-bounds pixels, NaN / infinite / zero depths, voxels behind a
    camera that fuse, and weights clamped at 1 after several observations."""
    z, _ = golden()
    behind = 0
    for name in GOLDEN_CASES:
        aabb, dims, c2w, K, depth, color, _ = case(name)
        _, _, _, trace = oracle_b(name)
        vc = ot.from_aabb(aabb, dims)[0].reshape(3, -1).numpy()
        inv = torch.inverse(c2w).numpy()
        for b, (ix, iy, valid) in enumerate(trace):
            behind += int((((inv[b, 2, :3] @ vc) + inv[b, 2, 3] > 0) & valid).sum())   # camera z > 0 before the flip: behind it
    assert behind > 0
    d = np.concatenate([z[f"{n}/depth"].ravel() for n in GOLDEN_CASES])
    assert np.isnan(d).any() and np.isinf(d).any() and (d == 0).any()
    ix, iy, _ = oracle_b("outside_b10")[3][0]
    assert (ix < 0).any() and (ix >= 0).any() and (iy < 0).any()
    assert (z["outside_b10/weights"] == 1).any()


def test_get_mesh_gather_and_pymeshlab_matrices():
    """get_mesh after marching cubes: colours gathered at the vertices rounded half to even, world-space vertices, and the matrices the
    reference hands pymeshlab (float64, alpha 1)."""
    z, meta = golden()
    st = oracle_a("outside_b10")
    assert np.array_equal(st[1].clamp(-1, 1).numpy(), z["outside_b10/mc_volume"])
    assert meta["cases"]["outside_b10"]["mc_args"] == {"level": 0, "allow_degenerate": False}
    verts, faces, normals, colors = ot.mesh_from_marching_cubes(st[1], st[3], st[5], st[4], torch.from_numpy(z["mc_vertices"]),
                                                                torch.from_numpy(z["mc_faces"]), torch.from_numpy(z["mc_normals"]))
    assert torch.equal(verts, torch.from_numpy(z["outside_b10/mesh_vertices"]))
    assert torch.equal(colors, torch.from_numpy(z["outside_b10/mesh_colors"]))
    assert np.array_equal(z["outside_b10/pymeshlab_vertex_matrix"], verts.numpy().astype(np.float64))
    assert np.array_equal(z["outside_b10/pymeshlab_v_color_matrix"], np.concatenate([colors.numpy().astype(np.float64), np.ones((len(colors), 1))], 1))


def test_cameras_additions_match_reference_flow():
    """Cameras.rescale_output_resolution then get_intrinsics_matrices give the K and image size the reference's export flow hands
    integrate_tsdf, and the flow's homogeneous c2w is the cameras' with a [0, 0, 0, 1] row."""
    from sdfstudio_b200.cameras import Cameras

    z, meta = golden()
    fl = meta["flow"]
    c2w = torch.from_numpy(z["flow/c2w_in"])
    cams = Cameras(c2w, fl["f"], fl["f"] * 0.97, fl["width"] / 2 + 0.25, fl["height"] / 2 - 0.5, fl["width"], fl["height"])
    cams.rescale_output_resolution(1.0 / fl["downscale_factor"])
    assert [cams.height, cams.width] == fl["image_hw"] == [fl["rescaled_height"][0], fl["rescaled_width"][0]]
    assert torch.equal(cams.get_intrinsics_matrices(), torch.from_numpy(z["flow/K"]))
    hom = torch.cat([c2w, torch.tensor([0.0, 0, 0, 1]).expand(len(c2w), 1, 4)], dim=1)
    assert torch.equal(hom, torch.from_numpy(z["flow/c2w"]))
    assert fl["calls"] == [fl["batch_size"]] * (fl["n"] // fl["batch_size"]) + [fl["n"] % fl["batch_size"]]
    with pytest.raises(ValueError):
        cams.rescale_output_resolution(torch.ones(len(cams)))


def test_flow_matches_reference_restated():
    """The reference's whole export flow, restated: its images fused by (a) in one batch give the volume it handed skimage."""
    z, meta = golden()
    fl = meta["flow"]
    st = ot.from_aabb(torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), torch.tensor(fl["resolution"]))
    ot.integrate_batched(st[:4], ot.truncation(st[4]), torch.from_numpy(z["flow/c2w"]), torch.from_numpy(z["flow/K"]),
                         torch.from_numpy(z["flow/depth"]), torch.from_numpy(z["flow/color"]), fl["batch_size"])
    assert np.array_equal(st[1].clamp(-1, 1).numpy(), z["flow/mc_volume"])
    assert fl["file"] == os.path.join("out", "tsdf_mesh.ply")


def _params(fn):
    out = []
    for p in inspect.signature(fn).parameters.values():
        d = p.default
        if d is inspect.Parameter.empty:
            out.append([p.name, {"required": True}])
        elif isinstance(d, dataclasses.Field):
            out.append([p.name, {"field_default_factory": d.default_factory()}])
        else:
            out.append([p.name, {"default": list(d) if isinstance(d, tuple) else d}])
    return out


def test_signatures_and_defaults():
    from sdfstudio_b200 import tsdf

    sig = golden()[1]["signatures"]
    fields = []
    for f in dataclasses.fields(tsdf.TSDF):
        fields.append([f.name, {"required": True} if f.default is dataclasses.MISSING else {"default": f.default}])
    assert fields == sig["TSDF"]["fields"]
    assert set(sig["TSDF"]["members"]) <= set(k for k in vars(tsdf.TSDF) if not k.startswith("__"))
    assert isinstance(vars(tsdf.TSDF)["export_mesh"], classmethod) and isinstance(vars(tsdf.TSDF)["from_aabb"], staticmethod)
    assert _params(tsdf.TSDF.integrate_tsdf) == sig["TSDF"]["integrate_tsdf"]
    assert _params(tsdf.export_tsdf_mesh) == sig["export_tsdf_mesh"]
    # tsdf_mesh takes ExportTSDFMesh's defaults for every option it shares with it
    ours = {n: d for n, d in _params(tsdf.tsdf_mesh)}
    shared = 0
    for name, d in sig["ExportTSDFMesh"]:
        if name == "resolution":
            assert tsdf.volume_dims_of(ours[name]["default"]).tolist() == d["default"]
            shared += 1
        elif name in ours:
            assert ours[name] == d, name
            shared += 1
    assert shared == 12


def test_resolution_quirk_and_argument_errors(tmp_path):
    """The omitted resolution (a dataclasses.Field) and a tuple raise the reference's ValueError before anything is rendered; masks, CPU
    tensors and an unknown texture method raise."""
    from sdfstudio_b200 import tsdf

    meta = golden()[1]
    pipeline = types.SimpleNamespace(device=torch.device("cpu"), datamanager=types.SimpleNamespace(
        train_dataset=types.SimpleNamespace(_dataparser_outputs=types.SimpleNamespace(cameras=None, scene_box=None))))
    for label, kw in (("omitted", {}), ("tuple", dict(resolution=(8, 8, 8)))):
        with pytest.raises(ValueError) as e:
            tsdf.export_tsdf_mesh(pipeline, tmp_path, **kw)
        assert str(e.value) == meta["resolution_errors"][label]
    t = tsdf.TSDF.from_aabb(torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), torch.tensor([4, 4, 4]))
    c2w, K, depth = torch.eye(4)[None], torch.eye(3)[None], torch.ones(1, 1, 2, 2)
    with pytest.raises(NotImplementedError):
        t.integrate_tsdf(c2w, K, depth, mask_images=torch.ones(1, 1, 2, 2))
    with pytest.raises(RuntimeError, match="CUDA only"):
        t.integrate_tsdf(c2w, K, depth)
    with pytest.raises(ValueError):
        tsdf.tsdf_mesh(None, None, tmp_path, texture_method="poisson")


def test_c_abi_error_codes():
    """Invalid arguments return error codes before any device work."""
    from sdfstudio_b200 import _lib

    lib = _lib.load()
    p = 0x90000

    def call(coords=p, n=8, cams=p, B=2, depth=p, color=None, H=4, W=4, trunc=p, values=p, weights=p, colors=None):
        return lib.sdfb200_tsdf_integrate(coords, n, cams, B, depth, color, H, W, trunc, values, weights, colors, None)

    assert call(n=-1) == -1 and call(B=-1) == -1 and call(H=-1) == -1
    assert call(H=0) == -1 and call(W=0) == -1
    assert call(coords=None) == -1 and call(values=None) == -1 and call(weights=None) == -1 and call(trunc=None) == -1
    assert call(cams=None) == -1 and call(depth=None) == -1
    assert call(color=p, colors=None) == -1
    assert b"NULL pointer" in lib.sdfb200_last_error_string()
    assert call(B=0, H=0, W=0, cams=None, depth=None) == 0           # no images: nothing to do
    assert call(n=0, coords=None, values=None, weights=None) == 0    # no voxels: nothing to do
