"""GPU checks of the mesh renderer: sdfb200_mesh_rasterize's keys against the brute-force fp64 oracle (oracle/render_mesh.py) bit for bit
on meshes that stress an exact rasterizer (spheres from outside and inside, a room around the camera, faces across or behind the camera
plane, edge-on and degenerate faces, exact-edge grids, duplicates, both work paths and their threshold, sub-pixel faces, per-frame
intrinsics, odd frame sizes, empty meshes and zero frames), the depth against the package's rays, the shading against the oracle's,
marching-cubes orientation, determinism, a multi-million-face case against a torch-fp64 restatement, the refusals and the end-to-end
writers."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import render_mesh as orm
from oracle.make_golden_tsdf import look_at, on_sphere
from sdfstudio_b200 import _lib, meshing, render_mesh, texturing
from sdfstudio_b200.cameras import Cameras
from sdfstudio_b200.tsdf import pack_cams

pytestmark = pytest.mark.gpu

LARGE = 256          # SDFB200_MESH_LARGE_TRIANGLE_PIXELS
THREADS = 256        # the rasterizer's block size


@pytest.fixture(autouse=True)
def _keep_global_rng():
    """Every test here restores the global CPU and CUDA generators, so that the tests after this file draw what they would draw
    without it."""
    with torch.random.fork_rng(devices=range(torch.cuda.device_count())):
        yield


def uv_sphere(n_lat, n_lon, radius=1.0, centre=(0.0, 0.0, 0.0), outward=True):
    """A closed UV sphere, faces counter-clockwise seen from outside (outward=True) or from inside."""
    lat = np.linspace(0, np.pi, n_lat + 1)[1:-1]
    lon = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    v = [[0, 0, radius]] + [[radius * np.sin(a) * np.cos(b), radius * np.sin(a) * np.sin(b), radius * np.cos(a)] for a in lat for b in lon]
    v.append([0, 0, -radius])
    f = []
    ring = lambda r, k: 1 + r * n_lon + k % n_lon  # noqa: E731
    for k in range(n_lon):
        f.append([0, ring(0, k), ring(0, k + 1)])
        f.append([len(v) - 1, ring(n_lat - 2, k + 1), ring(n_lat - 2, k)])
    for r in range(n_lat - 2):
        for k in range(n_lon):
            f += [[ring(r, k), ring(r + 1, k), ring(r + 1, k + 1)], [ring(r, k), ring(r + 1, k + 1), ring(r, k + 1)]]
    v = np.array(v, np.float64) + np.array(centre)
    f = np.array(f, np.int64)
    n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    out = (n * (v[f[:, 0]] - np.array(centre))).sum(1) > 0
    flip = ~out if outward else out
    f[flip] = f[flip][:, [0, 2, 1]]
    return v.astype(np.float32), f


def box(lo, hi, n, inward):
    from test_render_mesh_cpu import box_mesh, oriented

    v, f = box_mesh(lo, hi, n)
    c = np.full(3, (lo + hi) / 2)
    return v, oriented(v, f, inward_to=c) if inward else oriented(v, f, outward_from=c)


def K(fx, fy, cx, cy):
    return torch.tensor([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], dtype=torch.float32)


def cams_rows(c2w, Ks):
    """[B,18] packed rows of c2w [B,4,4] and K [B,3,3] (tsdf.pack_cams), on the host."""
    return pack_cams(torch.as_tensor(c2w, dtype=torch.float32), torch.as_tensor(Ks, dtype=torch.float32)).numpy()


def gpu_keys(v, f, cams, H, W, z_near, large=None):
    """keys [B,H,W] uint64 through sdfb200_mesh_rasterize, or through the debug hook with the block path's threshold ``large``."""
    vt = torch.as_tensor(np.asarray(v, np.float32)).reshape(-1, 3).cuda().contiguous()
    ft = torch.as_tensor(np.asarray(f, np.int64)).reshape(-1, 3).cuda().contiguous()
    ct = torch.as_tensor(np.asarray(cams, np.float32)).reshape(-1, 18).cuda().contiguous()
    keys = torch.empty(ct.shape[0], H, W, dtype=torch.int64, device="cuda")
    args = (_lib.ptr(vt) if len(vt) else None, _lib.ptr(ft) if len(ft) else None, len(ft), _lib.ptr(ct) if len(ct) else None, ct.shape[0], H, W,
            float(z_near), _lib.ptr(keys) if keys.numel() else None)
    if large is None:
        _lib.check(_lib.load().sdfb200_mesh_rasterize(*args, _lib.stream_ptr()), "sdfb200_mesh_rasterize")
    else:
        _lib.check(_lib.load_debug().sdfb200_debug_mesh_rasterize(*args, large, _lib.stream_ptr()), "sdfb200_debug_mesh_rasterize")
    return keys.cpu().numpy().view(np.uint64)


def look(positions, target, Ks):
    c2w = look_at(torch.tensor(np.asarray(positions, np.float32)), target=target)
    return cams_rows(c2w, Ks)


def cases():
    out = {}
    v, f = uv_sphere(12, 20, 0.8, (0.1, -0.05, 0.02))
    out["sphere_outside"] = (v, f, look(on_sphere(3, 2.5, 1), (0.0, 0.0, 0.0), K(30.0, 28.0, 16.0, 12.5).expand(3, 3, 3)), 25, 32, 0.01)
    v2, f2 = uv_sphere(10, 14, 1.0, outward=True)
    c2w = look_at(torch.zeros(2, 3) + torch.tensor([[0.1, 0.0, 0.05]]), target=(1.0, 0.3, -0.2))
    out["inside_outward_sphere"] = (v2, f2, cams_rows(c2w, K(12.0, 12.0, 8.5, 6.5).expand(2, 3, 3)), 13, 17, 0.01)
    vb, fb = box(-1.0, 1.0, 3, inward=True)
    c2w = look_at(torch.tensor([[0.1, -0.2, 0.15], [0.0, 0.0, 0.0]]), target=(0.7, 0.4, -0.3))
    out["inside_inward_cube"] = (vb, fb, cams_rows(c2w, K(9.0, 9.0, 8.5, 6.5).expand(2, 3, 3)), 13, 17, 0.01)
    # the same room with the near plane among the walls: faces clipped at z_near / 2 for their pixel box, and the test at z_near
    out["inside_cube_near_walls"] = (vb, fb, cams_rows(c2w, K(9.0, 9.0, 8.5, 6.5).expand(2, 3, 3)), 13, 17, 0.95)
    # faces across the camera plane, wholly behind it, edge-on (their plane through the eye) and degenerate, around a camera at the origin
    rng = np.random.default_rng(5)
    tri = rng.uniform(-2, 2, (60, 3, 3))
    tri[:10, :, 2] = rng.uniform(0.1, 2, (10, 3))                       # behind
    tri[10:25, 0, 2], tri[10:25, 1:, 2] = 1.0, -1.5                     # across
    tri[25:30] = np.stack([tri[25:30, 0], 2 * tri[25:30, 0], tri[25:30, 2]], 1)   # v1 = 2 v0: edge-on
    tri[30:33, 2] = tri[30:33, 1]                                        # repeated vertex
    tri[33:36, 2] = 0.5 * (tri[33:36, 0] + tri[33:36, 1])                # collinear
    out["near_behind_edge_degenerate"] = (tri.reshape(-1, 3).astype(np.float32), np.arange(180).reshape(60, 3),
                                          cams_rows(torch.eye(4)[None], K(10.0, 10.0, 8.0, 8.0)[None]), 16, 16, 0.05)
    from test_render_mesh_cpu import plane_grid

    vg, fg = plane_grid(-2, 9, -2.0)
    out["exact_edge_grid"] = (vg, fg, cams_rows(torch.eye(4)[None], K(8.0, 8.0, 4.0, 4.0)[None]), 8, 8, 0.01)
    vd = np.array([[-0.2, -0.2, -1], [0.2, -0.2, -1], [-0.2, 0.2, -1], [0.3, 0.3, -1]], np.float32)
    out["duplicates"] = (vd, np.array([[1, 3, 2], [0, 1, 2], [1, 2, 0], [2, 0, 1], [0, 1, 2]]),
                         cams_rows(torch.eye(4)[None], K(10.0, 10.0, 4.0, 4.0)[None]), 8, 8, 0.01)
    # screen-space right triangles of legs 1 .. 40 pixels at depth 10 (boxes of 9 .. 1764 pixels), both sides of the block path's threshold
    sq = []
    for s in range(1, 41):
        x0, y0 = (s * 7) % 23 - 11.0, (s * 5) % 19 - 9.0
        sq.append([[x0, y0, -10.0], [x0 + s * 0.25, y0, -10.0], [x0, y0 + s * 0.25, -10.0]])
    out["sizes"] = (np.array(sq, np.float32).reshape(-1, 3), np.arange(120).reshape(40, 3), cams_rows(torch.eye(4)[None], K(40.0, 40.0, 32.0, 24.0)[None]),
                    48, 64, 0.01)
    # sub-pixel faces
    c = rng.uniform(-0.5, 0.5, (3000, 1, 3)) + np.array([0, 0, -3.0])
    small = c + rng.normal(0, 0.004, (3000, 3, 3))
    out["sub_pixel"] = (small.reshape(-1, 3).astype(np.float32), np.arange(9000).reshape(3000, 3),
                        cams_rows(torch.eye(4)[None].expand(2, 4, 4), torch.stack([K(60.0, 60.0, 20.0, 15.0), K(70.0, 65.0, 21.0, 14.0)])), 30, 40,
                        0.01)
    # per-frame intrinsics and frame sizes 1 x 1, 17 x 13 and one block + 1 pixels wide
    Ks = torch.stack([K(30.0, 28.0, 16.0, 12.5), K(20.0, 35.0, 10.0, 15.0), K(45.0, 40.0, 12.0, 9.0)])
    out["per_frame_intrinsics"] = (v, f, look(on_sphere(3, 2.2, 4), (0.1, 0.0, 0.0), Ks), 25, 32, 0.01)
    out["one_pixel"] = (v, f, look(on_sphere(2, 2.5, 6), (0.0, 0.0, 0.0), K(1.0, 1.0, 0.5, 0.5).expand(2, 3, 3)), 1, 1, 0.01)
    out["17x13"] = (v, f, look(on_sphere(2, 2.5, 7), (0.0, 0.0, 0.0), K(15.0, 15.0, 8.5, 6.5).expand(2, 3, 3)), 13, 17, 0.01)
    out["block_plus_one"] = (v, f, look(on_sphere(1, 2.5, 8), (0.0, 0.0, 0.0), K(200.0, 200.0, 128.5, 1.0).expand(1, 3, 3)), 2, THREADS + 1,
                             0.01)
    out["empty_mesh"] = (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64), look(on_sphere(2, 2.5, 9), (0.0, 0.0, 0.0),
                                                                                       K(10.0, 10.0, 4.0, 3.0).expand(2, 3, 3)), 6, 8, 0.01)
    out["zero_frames"] = (v, f, np.zeros((0, 18), np.float32), 6, 8, 0.01)
    return out


CASES = cases()


@pytest.mark.parametrize("name", list(CASES))
def test_keys_equal_the_oracle(name):
    v, f, cams, H, W, zn = CASES[name]
    want = orm.rasterize(v, f, cams, H, W, zn)
    got = gpu_keys(v, f, cams, H, W, zn)
    assert got.shape == want.shape and np.array_equal(got, want), f"{name}: {int((got != want).sum())} keys differ"
    face, _ = orm.split(want)
    if name in ("inside_outward_sphere", "empty_mesh"):
        assert (face < 0).all()
    if name in ("inside_inward_cube", "exact_edge_grid"):
        assert (face >= 0).all()
    if name in ("sphere_outside", "sizes", "sub_pixel"):
        assert (face >= 0).any()


@pytest.mark.parametrize("large", [0, 1, LARGE - 1, LARGE, LARGE + 1, 2**62])
@pytest.mark.parametrize("name", ["sizes", "inside_inward_cube", "inside_cube_near_walls", "near_behind_edge_degenerate", "sphere_outside"])
def test_both_paths_and_the_threshold_give_the_same_keys(name, large):
    v, f, cams, H, W, zn = CASES[name]
    assert np.array_equal(gpu_keys(v, f, cams, H, W, zn, large=large), gpu_keys(v, f, cams, H, W, zn))


def sphere_cameras(n, H, W, seed=1, dist=2.5):
    c2w = look_at(on_sphere(n, dist, seed), target=(0.0, 0.0, 0.0))
    return Cameras(c2w[:, :3, :], 0.9 * W, 0.9 * W, W / 2 - 0.3, H / 2 + 0.2, W, H, device=torch.device("cuda"))


def test_depth_agrees_with_the_package_rays():
    v, f = uv_sphere(24, 40, 0.8)
    cams = sphere_cameras(2, 40, 56)
    face, depth = render_mesh.rasterize(torch.from_numpy(v), torch.from_numpy(f), cams)
    vv = torch.from_numpy(v).double().cuda()
    ff = torch.from_numpy(f).cuda()
    for b in range(len(cams)):
        rays = cams.generate_rays(b)
        hit = face[b].reshape(-1) >= 0
        assert int(hit.sum()) > 300
        o, d = rays.origins[hit].double(), rays.directions[hit].double()
        tri = vv[ff[face[b].reshape(-1)[hit].long()]]
        e1, e2 = tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]
        p = torch.cross(d, e2, dim=-1)
        s = o - tri[:, 0]
        q = torch.cross(s, e1, dim=-1)
        det = (e1 * p).sum(-1)
        t = (e2 * q).sum(-1) / det
        u, w = (s * p).sum(-1) / det, (d * q).sum(-1) / det
        assert bool(((u > -1e-6) & (w > -1e-6) & (u + w < 1 + 1e-6)).all())
        view = t / rays.directions_norm[hit, 0].double()
        assert torch.allclose(depth[b].reshape(-1)[hit].double(), view, rtol=2e-6, atol=0)


def _shade_case(v, f, cams):
    vt, ft = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    frames = render_mesh.render_frames(vt, ft, cams)
    c2w = torch.cat([cams.camera_to_worlds, torch.tensor([0.0, 0, 0, 1], device="cuda").expand(len(cams), 1, 4)], 1)
    rows = pack_cams(c2w, cams.get_intrinsics_matrices())
    centre, ext = render_mesh._box(vt)
    lights = render_mesh.light_positions(rows, centre, ext).cpu().numpy()
    normals = texturing.vertex_normals_area_weighted(vt, ft).cpu().numpy()
    keys = orm.rasterize(v, f, rows.cpu().numpy(), cams.height, cams.width, 0.01 * ext)
    rgb, nrm = orm.shade(keys, v, normals, f, rows.cpu().numpy(), lights, render_mesh.light_params())
    return frames, orm.quantise(rgb), orm.quantise(nrm), keys


@pytest.mark.parametrize("where", ["outside", "inside"])
def test_shading_matches_the_oracle(where):
    if where == "outside":
        v, f = uv_sphere(16, 24, 0.8, (0.05, 0.0, -0.1))
        cams = sphere_cameras(2, 30, 40)
    else:
        v, f = box(-1.0, 1.0, 3, inward=True)
        c2w = look_at(torch.tensor([[0.2, -0.1, 0.1], [-0.3, 0.2, 0.0]]), target=(0.5, 0.5, -0.4))
        cams = Cameras(c2w[:, :3], 14.0, 14.0, 20.0, 15.0, 40, 30, device=torch.device("cuda"))
    frames, rgb, nrm, keys = _shade_case(v, f, cams)
    for name, want in (("rgb", rgb), ("normal", nrm)):
        got = frames[name].cpu().numpy()
        diff = np.abs(got.astype(np.int16) - want.astype(np.int16))
        frac = float((diff > 0).mean())
        print(f"{where} {name}: max |byte - oracle| = {int(diff.max())}, fraction off by one = {frac:.2e}")
        assert diff.max() <= 1 and frac < 0.01
        assert (got[orm.split(keys)[0] < 0] == 255).all()


def mc_sphere(n, radius_frac, device="cuda"):
    """A marching-cubes sphere of radius radius_frac (n - 1) cells centred in an n^3 lattice, in world units of 1 / (n - 1) around 0."""
    x = torch.arange(n, device=device, dtype=torch.float32)
    c = (n - 1) / 2
    g = torch.stack(torch.meshgrid(x, x, x, indexing="ij"), -1)
    vol = (g - c).norm(dim=-1) - radius_frac * (n - 1)
    verts, faces, _ = meshing.marching_cubes(vol, 0.0)
    return (verts - c) / (n - 1), faces.long()


def test_marching_cubes_sphere_orientation():
    v, f = mc_sphere(64, 0.35)
    H = W = 64
    cams = sphere_cameras(2, H, W, seed=3, dist=1.5)
    face, _ = render_mesh.rasterize(v, f, cams)
    frames = render_mesh.render_frames(v, f, cams, outputs=("normal",))
    h = 1 / 63
    for b in range(2):
        rays = cams.generate_rays(b)
        o, d = rays.origins[0].double(), rays.directions.double()
        to_c = -o / o.norm()
        ang = torch.acos((d @ to_c).clamp(-1, 1)).reshape(H, W)
        edge = math.asin(0.35 / float(o.norm()))
        disc = ang <= edge
        covered = face[b] >= 0
        assert int(covered.sum()) > 200
        wrong = covered != disc
        band = (1.5 * h) / (float(o.norm()) - 0.35)
        assert bool(((ang[wrong] - edge).abs() <= band).all()), "silhouette off the analytic disc by more than a cell"
        # the normals face the eye (a reversed winding would show the far side's inner faces, normals away from the eye), and inside
        # the inner half of the disc, where the surface faces the camera, their camera-space z is positive
        n = frames["normal"][b].double() / 255 * 2 - 1
        c2w = cams.camera_to_worlds[b].double()
        toward_eye = -(d.reshape(H, W, 3) @ c2w[:, :3])                   # the pixel rays in camera space, reversed
        facing = (n * toward_eye).sum(-1)[covered]
        assert float(facing.mean()) > 0.5 and float(facing.min()) > -0.1
        assert float(n[..., 2][covered & (ang < edge / 2)].min()) > 0.5


def test_determinism_shuffles_and_batching():
    v, f, cams, H, W, zn = CASES["sphere_outside"]
    a = gpu_keys(v, f, cams, H, W, zn)
    assert np.array_equal(a, gpu_keys(v, f, cams, H, W, zn))
    for b in range(len(cams)):   # one frame per call
        assert np.array_equal(a[b:b + 1], gpu_keys(v, f, cams[b:b + 1], H, W, zn))
    perm = np.random.default_rng(0).permutation(len(f))
    s = gpu_keys(v, f[perm], cams, H, W, zn)
    fa, da = orm.split(a)
    fs, ds = orm.split(s)
    assert np.array_equal(da.view(np.uint32), ds.view(np.uint32))
    remapped = np.where(fs >= 0, perm[np.maximum(fs, 0)], -1)
    differ = remapped != fa
    # where the faces differ, both cover the pixel at the same depth (a tie, which goes to the smaller id of each numbering)
    assert differ.mean() < 0.05
    for bb, j, i in list(zip(*np.nonzero(differ)))[:40]:
        for face_id in (fa[bb, j, i], remapped[bb, j, i]):
            one = orm.rasterize(v, f[[face_id]], cams[bb:bb + 1], H, W, zn)
            assert orm.split(one)[1][0, j, i] == da[bb, j, i]


def test_large_marching_cubes_mesh_against_torch_fp64():
    v, f = mc_sphere(768, 0.45)
    # a bumpy surface: every vertex moved along its radius
    v = (v * (1 + 0.03 * torch.sin(9 * v[:, :1]) * torch.cos(7 * v[:, 1:2]))).contiguous()
    assert len(f) > 2_000_000
    H, W = 1080, 1920
    cams = Cameras(look_at(on_sphere(3, 1.4, 11))[:, :3], 1400.0, 1400.0, 960.0, 540.0, W, H, device=torch.device("cuda"))
    face, depth = render_mesh.rasterize(v, f, cams)
    c2w = torch.cat([cams.camera_to_worlds, torch.tensor([0.0, 0, 0, 1], device="cuda").expand(3, 1, 4)], 1)
    rows = pack_cams(c2w, cams.get_intrinsics_matrices()).double()
    zn = float(torch.tensor(0.01 * render_mesh._box(v)[1], dtype=torch.float32))
    g = torch.Generator(device="cuda").manual_seed(0)
    for b in range(3):
        m = rows[b, :12].view(3, 4)
        p = v.double()[f]                                              # [F,3,3]
        cam = torch.stack([((m[r, 0] * p[..., 0] + m[r, 1] * p[..., 1]) + m[r, 2] * p[..., 2]) + m[r, 3] for r in range(3)], -1)

        def cross(a, c):
            return torch.stack([a[..., 1] * c[..., 2] - a[..., 2] * c[..., 1], a[..., 2] * c[..., 0] - a[..., 0] * c[..., 2],
                                a[..., 0] * c[..., 1] - a[..., 1] * c[..., 0]], -1)

        E = torch.stack([cross(cam[:, 1], cam[:, 2]), cross(cam[:, 2], cam[:, 0]), cross(cam[:, 0], cam[:, 1])], 1)
        det = (cam[:, 0, 0] * E[:, 0, 0] + cam[:, 0, 1] * E[:, 0, 1]) + cam[:, 0, 2] * E[:, 0, 2]
        e, num, front = -E, -det, det < 0
        del cam, p, E
        pix = torch.randint(0, H * W, (1024,), generator=g, device="cuda")
        # half the samples on covered pixels
        cov = torch.nonzero(face[b].reshape(-1) >= 0)[:, 0]
        pix[:512] = cov[torch.randint(0, len(cov), (512,), generator=g, device="cuda")]
        ii, jj = (pix % W).double(), (pix // W).double()
        k = rows[b, 12:]
        dx = ((ii + 0.5) - k[2]) / k[0]
        dy = -(((jj + 0.5) - k[5]) / k[4])
        none = torch.iinfo(torch.int64).max     # covered keys are < 2^63
        best = torch.full((len(pix),), none, dtype=torch.int64, device="cuda")
        for f0 in range(0, len(f), 1 << 17):
            ee = e[f0:f0 + (1 << 17)]
            w = (dx[:, None, None] * ee[None, :, :, 0] + dy[:, None, None] * ee[None, :, :, 1]) - ee[None, :, :, 2]
            S = (w[..., 0] + w[..., 1]) + w[..., 2]
            dep = num[None, f0:f0 + len(ee)] / S
            ok = front[None, f0:f0 + len(ee)] & (w >= 0).all(-1) & (S > 0) & (dep >= zn)
            del w
            key = (dep.float().view(torch.int32).long() << 32) | torch.arange(f0, f0 + len(ee), device="cuda")[None]
            best = torch.minimum(best, torch.where(ok, key, none).amin(1))
            del S, dep, ok, key
        want_face = torch.where(best == none, -1, best & 0xFFFFFFFF).to(torch.int32)
        assert torch.equal(face[b].reshape(-1)[pix], want_face), f"frame {b}: {int((face[b].reshape(-1)[pix] != want_face).sum())} faces differ"
        hit = best != none
        want_depth = (best[hit] >> 32).to(torch.int32).view(torch.float32)
        assert torch.equal(depth[b].reshape(-1)[pix][hit], want_depth)


def test_refusals_launch_nothing():
    v, f = uv_sphere(6, 8, 0.8)
    vt, ft = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    cams = sphere_cameras(1, 8, 8)
    bad_v = vt.clone()
    bad_v[3, 1] = float("nan")
    n0 = _lib.launch_count()
    for fn in (lambda: render_mesh.rasterize(bad_v, ft, cams), lambda: render_mesh.rasterize(vt, ft + len(v), cams),
               lambda: render_mesh.rasterize(vt, ft - 1, cams), lambda: render_mesh.render_frames(vt, ft, cams, outputs=("rgb", "depth")),
               lambda: render_mesh.rasterize(vt, ft, cams, z_near=0.0), lambda: render_mesh.rasterize(vt, ft, cams, z_near=float("inf")),
               lambda: render_mesh.render_frames(vt, ft, cams, outputs=())):
        with pytest.raises(ValueError):
            fn()
    assert _lib.launch_count() == n0
    # the C entry points refuse before any launch
    lib = _lib.load()
    rows = torch.zeros(1, 18, device="cuda")
    keys = torch.empty(1, 8, 8, dtype=torch.int64, device="cuda")
    base = dict(v=_lib.ptr(vt), f=_lib.ptr(ft), n=len(ft), c=_lib.ptr(rows), b=1, h=8, w=8, z=0.1, k=_lib.ptr(keys))
    for bad in (dict(h=0), dict(w=-1), dict(h=40000), dict(b=-1), dict(z=0.0), dict(z=float("nan")), dict(z=float("inf")), dict(n=-1),
                dict(n=2**31), dict(f=None), dict(c=None), dict(k=None), dict(k=_lib.ptr(keys) + 4), dict(f=_lib.ptr(ft) + 4),
                dict(v=_lib.ptr(vt) + 2)):
        a = dict(base, **bad)
        assert lib.sdfb200_mesh_rasterize(a["v"], a["f"], a["n"], a["c"], a["b"], a["h"], a["w"], a["z"], a["k"], _lib.stream_ptr()) == -1, bad
    params = render_mesh.light_params().ctypes.data_as(C.POINTER(C.c_float))
    assert lib.sdfb200_mesh_shade(_lib.ptr(keys), 1, 8, 8, _lib.ptr(vt), _lib.ptr(vt), _lib.ptr(ft), len(ft), _lib.ptr(rows), _lib.ptr(rows),
                                  params, None, None, _lib.stream_ptr()) == -1
    assert _lib.launch_count() == n0


def test_empty_mesh_renders_white_frames():
    cams = sphere_cameras(2, 6, 9)
    frames = render_mesh.render_frames(torch.zeros(0, 3), torch.zeros(0, 3, dtype=torch.int64), cams)
    assert all(bool((t == 255).all()) and t.shape == (2, 6, 9, 3) for t in frames.values())


def test_render_trajectory_video_writes_the_frames(tmp_path):
    v, f = mc_sphere(48, 0.3)
    ply = tmp_path / "mesh.ply"
    meshing.write_ply(str(ply), v.cpu().numpy(), f.cpu().numpy(), None)
    cams = sphere_cameras(3, 24, 33, seed=5, dist=1.2)
    want = render_mesh.render_frames(v, f, sphere_cameras(3, 24, 33, seed=5, dist=1.2))
    out = tmp_path / "renders" / "out.mp4"
    render_mesh.render_trajectory_video(ply, cams, out, ["normal", "rgb"], output_format="images", merge_type="concat")
    files = sorted(p.relative_to(tmp_path).as_posix() for p in tmp_path.rglob("*.png"))
    assert files == sorted(f"renders/out/{n}/{i:05d}.png" for n in ("normal", "rgb") for i in range(3))
    from test_render_mesh_cpu import decode_png

    for n in ("normal", "rgb"):
        for i in range(3):
            assert np.array_equal(decode_png((tmp_path / "renders" / "out" / n / f"{i:05d}.png").read_bytes()), want[n][i].cpu().numpy())
    # rescaling: half the resolution
    render_mesh.render_trajectory_video(ply, sphere_cameras(2, 24, 33), tmp_path / "half" / "o.mp4", ["rgb", "normal"], 0.5, output_format="images")
    assert decode_png((tmp_path / "half" / "o" / "rgb" / "00001.png").read_bytes()).shape == (12, 16, 3)


def test_render_trajectory_video_with_the_reference_cameras(tmp_path):
    """The reference's Cameras (as RenderTrajectory.main passes them) render the frames the package's Cameras render, and are rescaled
    in place as the reference rescales them."""
    from test_render_mesh_cpu import RefShapedCameras, decode_png

    v, f = mc_sphere(40, 0.3)
    ply = tmp_path / "mesh.ply"
    meshing.write_ply(str(ply), v.cpu().numpy(), f.cpu().numpy(), None)
    cams = sphere_cameras(2, 24, 32, seed=6, dist=1.2)
    ref = RefShapedCameras(cams.camera_to_worlds.cpu(), cams.fx.cpu(), cams.fy.cpu(), cams.cx.cpu(), cams.cy.cpu(), 32, 24)
    render_mesh.render_trajectory_video(ply, ref, tmp_path / "r" / "o.mp4", ["rgb", "normal"], 0.5, output_format="images")
    assert ref.width.view(-1).tolist() == [16, 16] and ref.height.view(-1).tolist() == [12, 12]
    cams.rescale_output_resolution(0.5)
    want = render_mesh.render_frames(v, f, cams)
    for n in ("rgb", "normal"):
        for i in range(2):
            assert np.array_equal(decode_png((tmp_path / "r" / "o" / n / f"{i:05d}.png").read_bytes()), want[n][i].cpu().numpy())


def test_render_mesh_on_a_spiral(tmp_path):
    v, f = mc_sphere(40, 0.3)
    ply = tmp_path / "mesh.ply"
    meshing.write_ply(str(ply), v.cpu().numpy(), f.cpu().numpy(), None)
    train = Cameras(look_at(on_sphere(4, 1.5, 2))[:, :3], 20.0, 20.0, 16.0, 12.0, 32, 24, device=torch.device("cuda"))
    render_mesh.render_mesh(ply, train, tmp_path / "r" / "spiral.mp4", traj="spiral", num_views=5, output_format="images")
    for n in ("rgb", "normal"):
        pngs = sorted((tmp_path / "r" / "spiral" / n).glob("*.png"))
        assert len(pngs) == 5
        from test_render_mesh_cpu import decode_png

        img = decode_png(pngs[0].read_bytes())
        assert img.shape == (24, 32, 3)
