"""GPU: sdfb200_tsdf_integrate against restatement (b) of oracle/tsdf.py (its documented op order, bit for bit) and against the golden
minted from the unmodified reference, batching and rerun identity, the edges (no images, one voxel, hand-built volumes, past 2^31
elements), 512^3 x 49 images against restatement (a) with the memory it takes, get_mesh, and tsdf_mesh on a SurfaceRenderer.

Against the golden (and against (a) on the GPU), the kernel differs from the reference's ATen ops in the summation order inside
``bmm`` and in the grid_sample backend's unnormalisation, so a voxel's depth moves by a few ulp; values then agree within
test_tsdf_cpu.VALUE_ATOL (derived there), and a pixel or validity decision flips only for voxels on a rounding or validity boundary,
which are counted and checked to lie there."""
import numpy as np
import pytest
import torch

from oracle import tsdf as ot
from test_tsdf_cpu import GOLDEN_CASES, VALUE_ATOL, case, golden, near_boundary

pytestmark = pytest.mark.gpu
MB = 1 << 20


def kernel_tsdf(name, batch_size=None, color=True):
    """The golden case fused by TSDF.integrate_tsdf on cuda, all images in one call or in batches of ``batch_size``."""
    from sdfstudio_b200 import tsdf

    aabb, dims, c2w, K, depth, col, _ = case(name)
    t = tsdf.TSDF.from_aabb(aabb, dims).to("cuda")
    B = len(c2w)
    bs = batch_size or B
    for i in range(0, B, bs):
        t.integrate_tsdf(c2w[i:i + bs].cuda(), K[i:i + bs].cuda(), depth[i:i + bs].cuda(), col[i:i + bs].cuda() if color else None)
    return t


def device_cams(c2w, K):
    """The camera rows the kernel receives (inverses computed on the device), for restatement (b)."""
    from sdfstudio_b200 import tsdf

    return tsdf.pack_cams(c2w.cuda(), K.cuda()).cpu().numpy()


def oracle_b(name):
    aabb, dims, c2w, K, depth, color, _ = case(name)
    vc, v, w, c, vs, _ = ot.from_aabb(aabb, dims)
    return ot.integrate_ops(vc.reshape(3, -1).numpy(), v.reshape(-1).numpy(), w.reshape(-1).numpy(), c.reshape(-1, 3).numpy(),
                            np.float32(ot.truncation(vs)), device_cams(c2w, K), depth[:, 0].numpy(), color.numpy())


def as_np(t):
    return t.values.reshape(-1).cpu().numpy(), t.weights.reshape(-1).cpu().numpy(), t.colors.reshape(-1, 3).cpu().numpy()


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_kernel_equals_op_order_restatement(name):
    v, w, c = as_np(kernel_tsdf(name))
    bv, bw, bc, _ = oracle_b(name)
    assert np.array_equal(v, bv) and np.array_equal(w, bw) and np.array_equal(c, bc)


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_kernel_against_reference_golden(name):
    z, _ = golden()
    v, w, c = as_np(kernel_tsdf(name))
    ref_v, ref_w, ref_c = z[f"{name}/values"].reshape(-1), z[f"{name}/weights"].reshape(-1), z[f"{name}/colors"].reshape(-1, 3)
    flips = np.nonzero((w != ref_w) | (c != ref_c).any(1))[0]
    assert near_boundary(name, flips).all() and len(flips) <= max(2, len(ref_v) // 1000)
    same = np.ones(len(v), bool)
    same[flips] = False
    assert np.abs(v[same] - ref_v[same]).max() <= VALUE_ATOL
    print(f"{name}: {len(flips)} boundary voxels, max |value - reference| = {np.abs(v[same] - ref_v[same]).max():.2e}")


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_batching_and_reruns_are_bit_identical(name):
    ref = as_np(kernel_tsdf(name))
    for bs in (1, 3, 10, None, None):
        got = as_np(kernel_tsdf(name, bs))
        assert all(np.array_equal(a, b) for a, b in zip(got, ref)), bs


def test_without_colour_images_colours_stay():
    t = kernel_tsdf("outside_b10", color=False)
    ref = kernel_tsdf("outside_b10")
    assert torch.equal(t.colors, torch.zeros_like(t.colors))
    assert torch.equal(t.values, ref.values) and torch.equal(t.weights, ref.weights)


def random_cameras(seed, B, H, W, radius=2.5):
    g = torch.Generator().manual_seed(seed)
    from oracle.make_golden_tsdf import look_at

    pos = torch.randn(B, 3, generator=g)
    pos = radius * pos / pos.norm(dim=-1, keepdim=True) * (0.3 + torch.rand(B, 1, generator=g))
    c2w = look_at(pos, target=tuple((0.3 * torch.randn(3, generator=g)).tolist()))
    K = torch.zeros(B, 3, 3)
    K[:, 0, 0], K[:, 1, 1] = 0.5 * W + W * torch.rand(B, generator=g), 0.5 * H + H * torch.rand(B, generator=g)
    K[:, 0, 1] = 0.05 * torch.randn(B, generator=g)
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = W / 2 + torch.randn(B, generator=g), H / 2 + torch.randn(B, generator=g), 1.0
    depth = 0.1 + 3 * torch.rand(B, 1, H, W, generator=g)
    depth[torch.rand(depth.shape, generator=g) < 0.05] = 0
    depth[torch.rand(depth.shape, generator=g) < 0.02] = float("nan")
    return c2w, K, depth, torch.rand(B, 3, H, W, generator=g)


def check_against_b(t, c2w, K, depth, color, v0, w0, c0):
    bv, bw, bc, _ = ot.integrate_ops(t.voxel_coords.reshape(3, -1).cpu().numpy(), v0.reshape(-1).numpy(), w0.reshape(-1).numpy(),
                                     c0.reshape(-1, 3).numpy(), np.float32(float(t.truncation)), device_cams(c2w, K),
                                     depth[:, 0].numpy(), None if color is None else color.numpy())
    v, w, c = as_np(t)
    assert np.array_equal(v, bv, equal_nan=True) and np.array_equal(w, bw, equal_nan=True) and np.array_equal(c, bc, equal_nan=True)


@pytest.mark.parametrize("seed,dims,hw,B", [(0, (24, 17, 30), (37, 53), 21), (1, (31, 31, 31), (64, 48), 150), (2, (5, 80, 9), (1, 90), 7)])
def test_seeded_random_cameras(seed, dims, hw, B):
    """More cameras than one shared-memory tile (150), skewed K, cameras inside and outside the volume."""
    from sdfstudio_b200 import tsdf

    c2w, K, depth, color = random_cameras(seed, B, *hw)
    t = tsdf.TSDF.from_aabb(torch.tensor([[-1.0, -1.2, -0.9], [1.1, 1.0, 1.3]]), torch.tensor(dims)).to("cuda")
    v0, w0, c0 = t.values.cpu(), t.weights.cpu(), t.colors.cpu()
    t.integrate_tsdf(c2w.cuda(), K.cuda(), depth.cuda(), color.cuda())
    check_against_b(t, c2w, K, depth, color, v0, w0, c0)
    assert float(t.weights.sum()) > 0


def test_hand_built_tsdf():
    """Arbitrary voxel coordinates, values, weights above 1 and colours: fused as the reference fuses them."""
    from sdfstudio_b200 import tsdf

    g = torch.Generator().manual_seed(7)
    dims = (6, 11, 13)
    coords = 2.4 * torch.rand(3, *dims, generator=g) - 1.2
    v0, w0, c0 = 2 * torch.rand(dims, generator=g) - 1, 3 * torch.rand(dims, generator=g), torch.rand(*dims, 3, generator=g)
    t = tsdf.TSDF(coords, v0.clone(), w0.clone(), c0.clone(), torch.tensor([0.05, 0.1, 0.2]), torch.tensor([-1.0, -1, -1]), 3.0).to("cuda")
    c2w, K, depth, color = random_cameras(8, 9, 20, 30)
    t.integrate_tsdf(c2w.cuda(), K.cuda(), depth.cuda(), color.cuda())
    check_against_b(t, c2w, K, depth, color, v0, w0, c0)


def test_no_cameras_and_one_voxel():
    from sdfstudio_b200 import tsdf

    t = tsdf.TSDF.from_aabb(torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), torch.tensor([3, 4, 5])).to("cuda")
    t.integrate_tsdf(torch.zeros(0, 4, 4, device="cuda"), torch.zeros(0, 3, 3, device="cuda"), torch.zeros(0, 1, 8, 8, device="cuda"))
    assert torch.equal(t.values, -torch.ones(3, 4, 5, device="cuda")) and not t.weights.any()
    c2w, K, depth, color = random_cameras(3, 4, 1, 1, radius=0.2)
    depth.fill_(1.0)
    t = tsdf.TSDF.from_aabb(torch.tensor([[-0.1, -0.1, -0.1], [0.1, 0.1, 0.1]]), torch.tensor([1, 1, 1])).to("cuda")
    v0, w0, c0 = t.values.cpu(), t.weights.cpu(), t.colors.cpu()
    t.integrate_tsdf(c2w.cuda(), K.cuda(), depth.cuda(), color.cuda())
    check_against_b(t, c2w, K, depth, color, v0, w0, c0)


def dtu_like(B=49, H=192, W=192, seed=0):
    """B cameras on a sphere of radius 2.5 around a sphere-shaped scene, with its depth and colour images (as rendered at downscale 2)."""
    from oracle.make_golden_tsdf import intrinsics, look_at, on_sphere, sphere_images

    c2w = look_at(on_sphere(B, 2.5, seed))
    K = intrinsics(B, 0.9 * W, H, W)
    depth, color = sphere_images(c2w, K, H, W, seed + 1)
    return c2w, K, depth, color


def test_512_cubed_49_images_against_reference_ops():
    """512^3 voxels x 49 images of 192^2 in one call, against restatement (a) on the GPU one image at a time; nothing per (voxel, image)
    is materialised: the peak beyond the TSDF and the images stays under 64 MB."""
    from sdfstudio_b200 import tsdf

    aabb, dims = torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), torch.tensor([512, 512, 512])
    c2w, K, depth, color = (x.cuda() for x in dtu_like())
    t = tsdf.TSDF.from_aabb(aabb, dims).to("cuda")
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t.integrate_tsdf(c2w, K, depth, color)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    assert extra < 64 * MB, extra
    v, w, c = t.values.reshape(-1), t.weights.reshape(-1), t.colors.reshape(-1, 3)
    t.voxel_coords = None
    st = list(ot.from_aabb(aabb, dims))
    st = [x.cuda() for x in st]
    for i in range(len(c2w)):
        ot.integrate(*st[:4], ot.truncation(st[4]), c2w[i:i + 1], K[i:i + 1], depth[i:i + 1], color[i:i + 1])
    rv, rw, rc = st[1].reshape(-1), st[2].reshape(-1), st[3].reshape(-1, 3)
    flips = (w != rw) | (c != rc).any(1)
    n_flips = int(flips.sum())
    assert n_flips <= v.numel() // 100000, n_flips
    # the truncation here is 5 voxels = 0.0195, so a few ulp of a depth up to 4 move a value by more than at the golden cases' scale
    atol = 16 * float(np.finfo(np.float32).eps) * 4.0 / float(ot.truncation(st[4]))
    assert float((v - rv)[~flips].abs().max()) <= atol
    assert int((w > 0).sum()) > v.numel() // 100
    print(f"512^3 x 49: {n_flips} boundary voxels of {v.numel()}, peak beyond the TSDF and images {extra / MB:.1f} MB")


def test_past_2_31_elements():
    """896^3: colors and the third plane of voxel_coords end past 2^31 elements; the voxels there fuse as (b) fuses them."""
    from sdfstudio_b200 import tsdf

    n = 896
    dims = torch.tensor([n, n, n])
    vs = torch.tensor([2.0 / n] * 3)
    origin = torch.tensor([-1.0, -1.0, -1.0])
    N = n**3
    coords = torch.empty(3, n, n, n, device="cuda")
    ar = torch.arange(n, device="cuda")
    coords[0] = (origin[0] + ar * vs[0]).view(n, 1, 1).cuda()
    coords[1] = (origin[1] + ar * vs[1]).view(1, n, 1).cuda()
    coords[2] = (origin[2] + ar * vs[2]).view(1, 1, n).cuda()
    t = tsdf.TSDF(coords, -torch.ones(n, n, n, device="cuda"), torch.zeros(n, n, n, device="cuda"), torch.zeros(n, n, n, 3, device="cuda"),
                  vs.cuda(), origin.cuda())
    c2w, K, depth, color = dtu_like(B=3, H=16, W=16, seed=5)
    t.integrate_tsdf(c2w.cuda(), K.cuda(), depth.cuda(), color.cuda())
    g = torch.Generator().manual_seed(0)
    idx = torch.cat([torch.arange(N - 4096, N), torch.randint(0, N, (8192,), generator=g)]).cuda()
    assert 3 * int(idx.max()) > 2**31
    xyz = coords.view(3, -1)[:, idx].cpu().numpy()
    N0 = len(idx)
    bv, bw, bc, _ = ot.integrate_ops(xyz, -np.ones(N0, np.float32), np.zeros(N0, np.float32), np.zeros((N0, 3), np.float32),
                                     np.float32(float(t.truncation)), device_cams(c2w, K), depth[:, 0].numpy(), color.numpy())
    assert np.array_equal(t.values.view(-1)[idx].cpu().numpy(), bv) and np.array_equal(t.weights.view(-1)[idx].cpu().numpy(), bw)
    assert np.array_equal(t.colors.view(-1, 3)[idx].cpu().numpy(), bc)
    assert (bw > 0).any()


def test_get_mesh():
    """get_mesh is meshing.marching_cubes on the clamped values plus the rounding gather; degenerate faces (two equal vertex positions)
    are removed on a volume with exact zeros."""
    from sdfstudio_b200 import meshing, tsdf

    t = kernel_tsdf("outside_b10")
    mesh = t.get_mesh()
    verts, faces, normals = meshing.marching_cubes(t.values.clamp(-1, 1), 0.0)
    ov, of, on, oc = ot.mesh_from_marching_cubes(t.values, t.colors, t.origin, t.voxel_size, verts, faces.long(), normals)
    assert len(faces) > 20 and torch.equal(mesh.vertices, ov) and torch.equal(mesh.colors, oc) and torch.equal(mesh.faces, of)

    g = torch.Generator().manual_seed(1)
    vol = torch.randint(-1, 2, (8, 8, 8), generator=g).float().cuda()     # exact zeros: cut edges meet at shared corners
    h = tsdf.TSDF(torch.zeros(3, 8, 8, 8, device="cuda"), vol, torch.ones_like(vol), torch.rand(8, 8, 8, 3, device="cuda"),
                  torch.ones(3, device="cuda"), torch.zeros(3, device="cuda"))
    mesh = h.get_mesh()
    verts, faces, _ = meshing.marching_cubes(vol.clamp(-1, 1), 0.0)
    p = verts[faces.long()]
    degenerate = (p[:, 0] == p[:, 1]).all(-1) | (p[:, 1] == p[:, 2]).all(-1) | (p[:, 0] == p[:, 2]).all(-1)
    assert degenerate.any() and torch.equal(mesh.faces, faces.long()[~degenerate])


def test_tsdf_mesh_on_surface_renderer(tmp_path):
    """tsdf_mesh end to end: render, fuse, mesh and write; the PLY reloads, and the NeRF texturing chain runs with the custom unwrap."""
    import sdfstudio_b200 as sb
    from sdfstudio_b200 import texturing, tsdf
    from sdfstudio_b200.cameras import Cameras
    from oracle.make_golden_tsdf import look_at, on_sphere
    from test_gpu_meshing import _field

    field = _field("fp32")
    renderer = sb.SurfaceRenderer(field, sb.NeuSSampler(num_samples=32, num_samples_importance=32).eval(),
                                  collider=sb.NearFarCollider(0.05, 4.0), kind="neus").eval()
    c2w = look_at(on_sphere(6, 2.2, 3))[:, :3, :]
    cams = Cameras(c2w, 40.0, 40.0, 24.0, 20.0, 48, 40, device=torch.device("cuda"))
    tsdf.tsdf_mesh(renderer, cams, tmp_path, resolution=48, texture_method="nerf", unwrap_method="custom", target_num_faces=None)
    assert (cams.width, cams.height) == (24, 20)
    mesh = texturing.get_mesh_from_filename(str(tmp_path / "tsdf_mesh.ply"))
    assert len(mesh.faces) > 100
    for f in ("mesh.obj", "material_0.mtl", "material_0.png"):
        assert (tmp_path / f).stat().st_size > 0
