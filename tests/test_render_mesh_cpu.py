"""CPU checks of the mesh renderer's host side: the camera paths, signatures, lighting constants and merge layout against the golden minted
from the unmodified reference (oracle/make_golden_render_mesh.py), the fp64 oracle rasterizer on hand-built cases with known answers, the
PNG encoder and the refusals that need no GPU."""
import inspect
import json
import sys
import zlib
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import render_mesh as orm
from oracle.make_golden_render_mesh import stub_frame
from sdfstudio_b200 import render_mesh, texturing
from sdfstudio_b200.cameras import FISHEYE, Cameras

GOLDEN = Path(__file__).parent / "golden"


@pytest.fixture(scope="module")
def golden():
    meta = json.loads((GOLDEN / "render_mesh.json").read_text())
    return meta, dict(np.load(GOLDEN / "render_mesh.npz"))


def _set(arrays, name):
    a = {k.split("/")[1]: v for k, v in arrays.items() if k.startswith(f"set_{name}/")}
    return Cameras(torch.from_numpy(a["c2w"]), float(a["fx"]), float(a["fy"]), float(a["cx"]), float(a["cy"]), int(a["W"]), int(a["H"]))


def _assert_path(cams, arrays, prefix):
    assert torch.equal(cams.camera_to_worlds, torch.from_numpy(arrays[f"{prefix}/c2w"]))
    for k in ("fx", "fy", "cx", "cy"):
        assert torch.equal(getattr(cams, k), torch.from_numpy(arrays[f"{prefix}/{k}"]).expand(len(cams))), (prefix, k)
    assert [cams.height, cams.width] == arrays[f"{prefix}/hw"].tolist(), prefix


def test_camera_paths_equal_the_reference(golden):
    meta, arrays = golden
    _assert_path(render_mesh.get_spiral_path(_set(arrays, "a"), steps=12, radius=1.0), arrays, "spiral_a")
    _assert_path(render_mesh.get_spiral_path(_set(arrays, "b"), steps=5, radiuses=(0.5, 0.7, 0.2), rots=1, zrate=0.25), arrays,
                 "spiral_b_radiuses")
    _assert_path(render_mesh.generate_ellipse_path(_set(arrays, "a"), n_frames=9, const_speed=False), arrays, "ellipse_a")
    _assert_path(render_mesh.generate_ellipse_path(_set(arrays, "b"), n_frames=6, const_speed=False, z_variation=0.5, z_phase=0.25), arrays,
                 "ellipse_b")
    _assert_path(render_mesh.interpolate_trajectory(_set(arrays, "a"), num_views=11), arrays, "interpolate_a")
    _assert_path(render_mesh.interpolate_trajectory(_set(arrays, "b"), num_views=7), arrays, "interpolate_b")
    _assert_path(render_mesh.get_path_from_json(meta["json_path"]), arrays, "json")
    with pytest.raises(NotImplementedError):
        render_mesh.generate_ellipse_path(_set(arrays, "a"), n_frames=9)
    with pytest.raises(ValueError):
        render_mesh.get_spiral_path(_set(arrays, "a"), radius=1.0, radiuses=(1.0, 1.0, 1.0))


def test_three_js_focal_length(golden):
    meta, _ = golden
    for fov, h, want in meta["three_js_focal"]:
        assert float(render_mesh.three_js_perspective_camera_focal_length(fov, h)) == want
    assert render_mesh.three_js_perspective_camera_focal_length(None, 100) == meta["three_js_focal_none"]


def _params(fn):
    return [[p.name, {"required": True} if p.default is inspect.Parameter.empty else {"default": p.default}]
            for p in inspect.signature(fn).parameters.values()]


def test_signatures_and_defaults(golden):
    meta, _ = golden
    sig = meta["signatures"]
    assert _params(render_mesh.render_trajectory_video) == sig["_render_trajectory_video"]
    assert _params(render_mesh.interpolate_trajectory) == sig["_interpolate_trajectory"]
    assert _params(render_mesh.get_spiral_path) == sig["get_spiral_path"]
    assert _params(render_mesh.generate_ellipse_path) == sig["generate_ellipse_path"]
    assert _params(render_mesh.get_path_from_json) == sig["get_path_from_json"]
    # RenderTrajectory's fields are render_mesh's parameters (the training cameras stand in for `data`)
    ours = {p.name: p.default for p in inspect.signature(render_mesh.render_mesh).parameters.values()}
    for name, d in meta["RenderTrajectory"]:
        if name == "data":
            assert ours["cameras"] is None
        elif name == "meshfile":
            assert d == {"required": True} and ours[name] is inspect.Parameter.empty
        elif name == "rendered_output_names":
            assert ours[name] is None and d == {"default": ["rgb", "normal"]}
        else:
            want = d["default"]
            got = str(ours[name]) if isinstance(ours[name], Path) else ours[name]
            assert got == want, name


def test_lighting_constants_are_render_json(golden):
    meta, _ = golden
    for k, v in render_mesh.RENDER_OPTIONS.items():
        assert meta["render_json"][k] == v, k
    assert meta["paint_uniform_color"] == [1, 1, 1] and meta["render_json"]["mesh_show_back_face"] is False
    p = render_mesh.light_params()
    assert p.dtype == np.float32 and p.shape == (27,)
    assert p[0:6].tolist() == np.float32([0.7, 0.7, 0.7, 0.66, 0.2, 10.0]).tolist()
    assert p[24:].tolist() == np.float32([0.3] * 3).tolist()


def test_merge_layout_equals_the_reference(golden):
    meta, arrays = golden
    for key, m in meta["merge"].items():
        merge_type = key.split("_")[0]
        want = arrays[f"merge/{key}"]
        assert m["fps"] == len(want) / 1.5
        for i in range(len(want)):
            images = [stub_frame(n, i)[:, :, ::-1] for n in m["names"]]
            assert np.array_equal(render_mesh.merge_frames(images, merge_type), want[i]), (key, i)
            assert np.array_equal(orm.merge(images, merge_type), want[i]), (key, i)
        # every output of every frame is written to <stem>/<name>/<index:05d>.png
        assert [c[0] for c in m["captures"]] == [f"renders/out/{n}/{i:05d}.png" for i in range(len(want)) for n in m["names"]]


def decode_png(data):
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    w, h = int.from_bytes(data[16:20], "big"), int.from_bytes(data[20:24], "big")
    n = int.from_bytes(data[33:37], "big")
    raw = np.frombuffer(zlib.decompress(data[41:41 + n]), np.uint8).reshape(h, 1 + 3 * w)
    return raw[:, 1:].reshape(h, w, 3)


def test_png_bytes_uint8_round_trip():
    img = np.random.default_rng(0).integers(0, 256, (13, 17, 3), dtype=np.uint8)
    assert np.array_equal(decode_png(texturing.png_bytes_u8(img)), img)
    f = np.random.default_rng(1).uniform(-0.1, 1.1, (5, 7, 3)).astype(np.float32)
    assert texturing.png_bytes(f) == texturing.png_bytes_u8(orm.quantise(f.astype(np.float64)))
    with pytest.raises(ValueError):
        texturing.png_bytes_u8(img.astype(np.float32))
    with pytest.raises(ValueError):
        texturing.png_bytes_u8(img[..., :2])


# ---------------------------------------------------------------------------------------------------------------------------------
# the oracle rasterizer on cases with known answers
# ---------------------------------------------------------------------------------------------------------------------------------
def cam_row(fx, fy, cx, cy, w2c=None):
    m = np.eye(4, dtype=np.float32)[:3] if w2c is None else np.asarray(w2c, np.float32)[:3]
    return np.concatenate([m.reshape(-1), [fx, 0, cx, 0, fy, cy]]).astype(np.float32)[None]


def test_one_triangle_exact_pixel_set():
    v = np.array([[-0.2, -0.2, -1], [0.2, -0.2, -1], [-0.2, 0.2, -1]], np.float32)
    keys = orm.rasterize(v, [[0, 1, 2]], cam_row(10, 10, 4, 4), 8, 8, 0.01)
    face, depth = orm.split(keys[0])
    want = np.zeros((8, 8), bool)
    for j in range(8):
        for i in range(8):
            want[j, i] = 2 <= i <= j <= 5       # x >= -0.2, y >= -0.2 and x + y <= 0, the hypotenuse through pixel centres included
    assert np.array_equal(face >= 0, want)
    assert np.allclose(depth[want], 1.0, rtol=1e-7)
    # clockwise on screen: culled
    assert (orm.rasterize(v, [[0, 2, 1]], cam_row(10, 10, 4, 4), 8, 8, 0.01) == orm.BACKGROUND).all()
    # the near plane: every hit is at depth 1
    assert (orm.rasterize(v, [[0, 1, 2]], cam_row(10, 10, 4, 4), 8, 8, 1.0001) == orm.BACKGROUND).all()


def oriented(vertices, faces, inward_to=None, outward_from=None):
    """Faces reordered so that each normal (v1 - v0) x (v2 - v0) points toward ``inward_to`` or away from ``outward_from``."""
    v = np.asarray(vertices, np.float64)
    f = np.array(faces, np.int64)
    n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    c = v[f[:, 0]] - (inward_to if inward_to is not None else outward_from)
    flip = (n * c).sum(1) > 0 if inward_to is not None else (n * c).sum(1) < 0
    f[flip] = f[flip][:, [0, 2, 1]]
    return f


def box_mesh(lo, hi, n=2):
    """The surface of the box [lo, hi]^3 as a grid of n x n quads per side, two triangles each (unoriented)."""
    verts, faces = [], []
    t = np.linspace(lo, hi, n + 1)
    for axis in range(3):
        for side in (lo, hi):
            base = len(verts)
            for a in t:
                for b in t:
                    p = [0.0, 0.0, 0.0]
                    p[axis], p[(axis + 1) % 3], p[(axis + 2) % 3] = side, a, b
                    verts.append(p)
            for i in range(n):
                for j in range(n):
                    q = base + i * (n + 1) + j
                    faces += [[q, q + 1, q + n + 1], [q + 1, q + n + 2, q + n + 1]]
    return np.array(verts, np.float32), np.array(faces)


def test_box_room_depths_are_the_plane_distances():
    v, f = box_mesh(-1.0, 1.0)
    f = oriented(v, f, inward_to=np.zeros(3))
    H, W = 15, 21
    keys = orm.rasterize(v, f, cam_row(6.0, 6.5, 10.5, 7.25), H, W, 0.01)
    face, depth = orm.split(keys[0])
    assert (face >= 0).all()
    dx = (np.arange(W) + 0.5 - 10.5) / 6.0
    dy = -(np.arange(H) + 0.5 - 7.25) / 6.5
    want = 1.0 / np.maximum(np.maximum(np.abs(dx)[None, :], np.abs(dy)[:, None]), 1.0)
    assert np.allclose(depth, want, rtol=1e-6)
    # the same room with outward-facing faces shows the camera only their backs: all culled
    assert (orm.rasterize(v, oriented(v, f, outward_from=np.zeros(3)), cam_row(6.0, 6.5, 10.5, 7.25), H, W, 0.01) == orm.BACKGROUND).all()


def plane_grid(n_lo, n_hi, z, jitter=0.0, seed=0):
    """A planar grid at view depth -z whose vertices lie on the rays through pixel centres of cam_row(8, 8, 4, 4) (plus jitter)."""
    k = np.arange(n_lo, n_hi + 1)
    xs = (2 * k - 7) / 16 * -z
    X, Y = np.meshgrid(xs, xs, indexing="xy")
    v = np.stack([X.ravel(), Y.ravel(), np.full(X.size, z)], 1)
    v[:, :2] += np.random.default_rng(seed).uniform(-jitter, jitter, (len(v), 2))
    n = len(k)
    faces = []
    for r in range(n - 1):
        for c in range(n - 1):
            q = r * n + c
            faces += [[q, q + 1, q + n], [q + 1, q + n + 1, q + n]]
    return v.astype(np.float32), oriented(v.astype(np.float32), faces, inward_to=np.zeros(3))


@pytest.mark.parametrize("jitter", [0.0, 0.03])
def test_watertight_grid_has_no_holes(jitter):
    v, f = plane_grid(-2, 9, -2.0, jitter)
    if jitter == 0.0:   # the vertices project exactly onto pixel centres
        assert np.array_equal(v[:, 0][:12] / 2 * 8 + 4, np.arange(-2, 10) + 0.5)
    keys = orm.rasterize(v, f, cam_row(8, 8, 4, 4), 8, 8, 0.01)
    face, depth = orm.split(keys[0])
    assert (face >= 0).all() and np.allclose(depth, 2.0, rtol=1e-6)


def test_coplanar_duplicates_resolve_to_the_smaller_id():
    v = np.array([[-0.2, -0.2, -1], [0.2, -0.2, -1], [-0.2, 0.2, -1], [0.3, 0.3, -1]], np.float32)
    f = [[1, 3, 2], [0, 1, 2], [1, 2, 0], [2, 0, 1], [0, 1, 2]]
    face, _ = orm.split(orm.rasterize(v, f, cam_row(10, 10, 4, 4), 8, 8, 0.01)[0])
    covered = face >= 0
    assert set(np.unique(face[covered]).tolist()) <= {0, 1}
    # faces 1..4 are the same triangle at the same depth: face 1 wins wherever face 0 does not cover
    only = orm.split(orm.rasterize(v, f[1:], cam_row(10, 10, 4, 4), 8, 8, 0.01)[0])[0]
    assert (only[only >= 0] == 0).all()


# ---------------------------------------------------------------------------------------------------------------------------------
# refusals that need no GPU
# ---------------------------------------------------------------------------------------------------------------------------------
def _cams(n=2, camera_type=1):
    return Cameras(torch.eye(4)[:3].expand(n, 3, 4), 10.0, 10.0, 4.0, 3.0, 8, 6, camera_type=camera_type)


def test_refusals(tmp_path):
    ply = tmp_path / "m.ply"
    rtv = render_mesh.render_trajectory_video
    with pytest.raises(ValueError, match="rendered outputs"):
        rtv(ply, _cams(), tmp_path / "o.mp4", ["rgb", "depth"], output_format="images", merge_type="concat")
    with pytest.raises(ValueError, match="half"):
        rtv(ply, _cams(), tmp_path / "o.mp4", ["rgb"], output_format="images")
    with pytest.raises(ValueError, match="mp4"):
        rtv(ply, _cams(), tmp_path / "o.avi", ["rgb", "normal"])
    with pytest.raises(ValueError, match="perspective"):
        rtv(ply, _cams(camera_type=FISHEYE), tmp_path / "o.mp4", ["rgb", "normal"], output_format="images")
    with pytest.raises(ValueError, match="perspective"):
        render_mesh.rasterize(torch.zeros(3, 3), torch.zeros(1, 3, dtype=torch.int64), _cams(camera_type=FISHEYE))
    with pytest.raises(ValueError, match="traj"):
        render_mesh.render_mesh(ply, _cams(), tmp_path / "o.mp4", traj="circle")
    with pytest.raises(ValueError, match="training cameras"):
        render_mesh.render_mesh(ply, None, tmp_path / "o.mp4", traj="spiral")
    assert not (tmp_path / "o").exists()


def test_video_needs_mediapy(tmp_path, monkeypatch):
    monkeypatch.setitem(sys.modules, "mediapy", None)
    with pytest.raises(ImportError, match='output_format="images"'):
        render_mesh.render_trajectory_video(tmp_path / "m.ply", _cams(), tmp_path / "o.mp4", ["rgb", "normal"])
    assert not (tmp_path / "o").exists()


# ---------------------------------------------------------------------------------------------------------------------------------
# the reference's Cameras, as RenderTrajectory.main passes them to _render_trajectory_video
# ---------------------------------------------------------------------------------------------------------------------------------
class RefShapedCameras:
    """The members of nerfstudio's Cameras that the reference's render_mesh.py reads: [N,3,4] poses, [N,1] intrinsics, per-camera
    width / height (int64) and camera_type, and rescale_output_resolution as the reference scales them (fp32 products, sizes truncated)."""

    def __init__(self, c2w, fx, fy, cx, cy, width, height, camera_type=1):
        n = len(c2w)

        def col(x, dtype=torch.float32):
            t = torch.as_tensor(x, dtype=dtype).reshape(-1, 1)
            return t.expand(n, 1).clone() if t.shape[0] == 1 else t

        self.camera_to_worlds = torch.as_tensor(c2w, dtype=torch.float32)
        self.fx, self.fy, self.cx, self.cy = col(fx), col(fy), col(cx), col(cy)
        self.width, self.height, self.camera_type = col(width, torch.int64), col(height, torch.int64), col(camera_type, torch.int64)

    def rescale_output_resolution(self, s):
        self.fx, self.fy, self.cx, self.cy = self.fx * s, self.fy * s, self.cx * s, self.cy * s
        self.height = (self.height * s).to(torch.int64)
        self.width = (self.width * s).to(torch.int64)


def test_the_reference_cameras_are_read():
    c2w = torch.eye(4)[:3].expand(3, 3, 4).clone()
    c2w[:, :, 3] = torch.tensor([[0.1, 0.2, 0.3], [0.0, -1.0, 2.0], [0.5, 0.5, 0.5]])
    ref = RefShapedCameras(c2w, [10.0, 11.0, 12.0], 9.0, 4.5, 3.25, 9, 7)
    cams = render_mesh.package_cameras(ref)
    assert isinstance(cams, Cameras) and (cams.width, cams.height) == (9, 7) and len(cams) == 3
    assert torch.equal(cams.camera_to_worlds, c2w) and torch.equal(cams.fx, torch.tensor([10.0, 11.0, 12.0]))
    assert torch.equal(cams.cy, torch.full((3,), 3.25)) and torch.equal(cams.camera_type, torch.ones(3, dtype=torch.int32))
    assert render_mesh.package_cameras(cams) is cams
    with pytest.raises(ValueError, match="one image size"):
        render_mesh.package_cameras(RefShapedCameras(c2w, 10.0, 9.0, 4.5, 3.25, [9, 9, 8], 7))
    with pytest.raises(ValueError, match="Cameras"):
        render_mesh.package_cameras(object())


def test_render_trajectory_video_takes_the_reference_cameras(tmp_path, monkeypatch):
    """The reference's Cameras get past the camera checks (the next step, mediapy, is made unimportable here), and a fisheye one is
    refused as the package's is."""
    ref = RefShapedCameras(torch.eye(4)[:3].expand(2, 3, 4), 10.0, 10.0, 4.0, 3.0, 8, 6)
    monkeypatch.setitem(sys.modules, "mediapy", None)
    with pytest.raises(ImportError, match='output_format="images"'):
        render_mesh.render_trajectory_video(tmp_path / "m.ply", ref, tmp_path / "o.mp4", ["rgb", "normal"])
    with pytest.raises(ValueError, match="perspective"):
        render_mesh.render_trajectory_video(tmp_path / "m.ply", RefShapedCameras(torch.eye(4)[:3].expand(2, 3, 4), 10.0, 10.0, 4.0, 3.0, 8, 6,
                                                                                 camera_type=2), tmp_path / "o.mp4", ["rgb", "normal"],
                                            output_format="images")
    assert torch.equal(ref.fx, torch.full((2, 1), 10.0)) and not (tmp_path / "o").exists()


def test_light_positions_equal_a_world_space_construction():
    """Light k of a frame at the box centre + extent (p.x right + p.y up + p.z front) in world space (the columns of c2w; front, the
    camera's +z, points toward the eye), moved to camera space with the camera's own world-to-camera rows."""
    from sdfstudio_b200.tsdf import pack_cams

    g = torch.Generator().manual_seed(0)
    q = torch.linalg.qr(torch.randn(4, 3, 3, generator=g, dtype=torch.float64))[0]
    c2w = torch.eye(4, dtype=torch.float64).repeat(4, 1, 1)
    c2w[:, :3, :3] = q * torch.sign(torch.linalg.det(q)).view(-1, 1, 1)
    c2w[:, :3, 3] = torch.randn(4, 3, generator=g, dtype=torch.float64) * 3
    K = torch.tensor([[20.0, 0, 8], [0, 20, 6], [0, 0, 1]]).expand(4, 3, 3)
    rows = pack_cams(c2w.float(), K)
    centre, extent = torch.tensor([0.3, -0.2, 0.7]), 2.5
    got = render_mesh.light_positions(rows, centre, extent)
    p = torch.tensor([render_mesh.RENDER_OPTIONS[f"light{k}_position"] for k in range(4)], dtype=torch.float64)
    world = centre.double().view(1, 1, 3) + extent * torch.einsum("bij,kj->bki", c2w[:, :3, :3], p)        # [B,4,3]
    want = torch.einsum("bij,bkj->bki", c2w[:, :3, :3].transpose(1, 2), world - c2w[:, None, :3, 3])
    assert torch.allclose(got.double(), want, atol=1e-5)
