"""GPU: the texture kernels (sdfb200_uv_rasterize, sdfb200_uv_unwrap_grid, sdfb200_uv_texel_rays) against the torch restatement of the
reference (oracle/texture.py) on the golden cases and on random chart layouts, and export_textured_mesh on a SurfaceRenderer."""
import numpy as np
import pytest
import torch

from oracle import texture as otex
from test_texture_cpu import GOLDEN_CASES, case_inputs, decode_png, golden, oracle_texels, parse_obj

pytestmark = pytest.mark.gpu

# directions and shifted origins: F.normalize's norm and the ray length's mean reduce in another order than the kernel's.  Directions
# are unit vectors (3e-7 absolute); a shifted origin o - 0.5 raylen d carries that last-bit difference scaled by its magnitude.
RAY_ATOL = 3e-7


def shifted_close(got, ref, raylen):
    return np.allclose(got, ref, rtol=0, atol=RAY_ATOL * (1 + np.abs(ref).max() + 0.5 * float(raylen)), equal_nan=True)


def kernel_texels(name):
    from sdfstudio_b200 import texturing

    vertices, faces, _, uvs, kw = case_inputs(name)
    if kw.get("unwrap_method") == "custom":
        return texturing.uv_unwrap_grid(len(faces), kw["px_per_uv_triangle"], "cuda")
    n = kw["num_pixels_per_side"]
    face, bary = texturing.uv_rasterize(uvs.cuda(), n, 10)
    return uvs.cuda(), face, bary, (n, n)


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_golden_cases(name):
    from sdfstudio_b200 import texturing

    vertices, faces, normals, _, kw = case_inputs(name)
    tc, face, bary, hw = kernel_texels(name)
    otc, oface, obary, ohw = oracle_texels(name)
    assert hw == ohw
    assert torch.equal(tc.cpu(), otc)
    assert torch.equal(face.cpu().long(), oface)
    assert np.array_equal(bary.cpu().numpy(), obary.numpy(), equal_nan=True)
    o, d, _ = texturing.uv_texel_rays(vertices.cuda(), faces.cuda(), normals.cuda(), face, bary)
    oo, od = otex.texel_rays(vertices, faces, normals, oface, obary)
    assert np.array_equal(o.cpu().numpy(), oo.numpy(), equal_nan=True)
    assert np.allclose(d.cpu().numpy(), od.numpy(), rtol=0, atol=RAY_ATOL, equal_nan=True)
    # with the ray-length shift, against the bundle the reference built
    z, _ = golden()
    if kw.get("raylen_method", "edge") == "edge":
        fv = vertices.cuda()[faces.cuda()]
        raylen = 2.0 * torch.mean(torch.norm(fv[:, 1, :] - fv[:, 0, :], dim=-1)).float()
    else:
        raylen = torch.zeros((), device="cuda")
    o, d, fars = texturing.uv_texel_rays(vertices.cuda(), faces.cuda(), normals.cuda(), face, bary, raylen)
    assert np.allclose(d.cpu().numpy().reshape(z[f"{name}/directions"].shape), z[f"{name}/directions"], rtol=0, atol=RAY_ATOL, equal_nan=True)
    for k, v in (("origins", o), ("fars", fars)):
        assert shifted_close(v.cpu().numpy().reshape(z[f"{name}/{k}"].shape), z[f"{name}/{k}"], raylen), k


def random_charts(n_faces, seed, device="cuda"):
    """[F,3,2] UVs: small triangles scattered over [0,1]^2 (xatlas-like charts with gaps between them), plus duplicates (ties), slivers
    and zero-area triangles, some of them along texel rows."""
    g = torch.Generator().manual_seed(seed)
    centre = torch.rand(n_faces, 1, 2, generator=g)
    uv = centre + (torch.rand(n_faces, 3, 2, generator=g) - 0.5) * 0.02
    k = n_faces // 50
    dup = torch.randint(0, n_faces, (2, k), generator=g)
    uv[dup[0]] = uv[dup[1]]
    flat = torch.randint(0, n_faces, (k,), generator=g)
    uv[flat, 2] = uv[flat, 0] + (uv[flat, 1] - uv[flat, 0]) * 0.5            # collinear corners
    row = torch.randint(0, n_faces, (k,), generator=g)
    uv[row, :, 1] = uv[row, 0:1, 1]                                           # horizontal zero-area triangles
    return uv.float().to(device)


@pytest.mark.parametrize("n_faces,n,chunk", [(20000, 512, 10), (5003, 256, 10), (3001, 128, 7), (700, 96, 1), (40, 200, 64)])
def test_random_charts(n_faces, n, chunk):
    from sdfstudio_b200 import texturing

    uv = random_charts(n_faces, n_faces + chunk)
    face, bary = texturing.uv_rasterize(uv, n, chunk)
    oface, obary = otex.rasterize(uv, n, chunk)
    assert torch.equal(face.long(), oface)
    assert np.array_equal(bary.cpu().numpy(), obary.cpu().numpy(), equal_nan=True)
    g = torch.Generator().manual_seed(1)
    nv = 2 * n_faces
    vertices = (torch.rand(nv, 3, generator=g) * 2 - 1).cuda()
    normals = torch.randn(nv, 3, generator=g).cuda()
    faces = torch.randint(0, nv, (n_faces, 3), generator=g).cuda()
    o, d, _ = texturing.uv_texel_rays(vertices, faces, normals, face, bary)
    oo, od = otex.texel_rays(vertices, faces, normals, oface, obary)
    assert np.array_equal(o.cpu().numpy(), oo.cpu().numpy(), equal_nan=True)
    assert np.allclose(d.cpu().numpy(), od.cpu().numpy(), rtol=0, atol=RAY_ATOL, equal_nan=True)


@pytest.mark.parametrize("n_faces,ppt", [(1, 1), (2, 4), (9999, 4), (20001, 2)])
def test_grid_unwrap_random_sizes(n_faces, ppt):
    from sdfstudio_b200 import texturing

    tc, face, bary, hw = texturing.uv_unwrap_grid(n_faces, ppt, "cuda")
    otc, oface, obary, ohw = otex.grid_unwrap(n_faces, ppt, "cuda")
    assert hw == ohw and torch.equal(tc, otc) and torch.equal(face.long(), oface)
    assert np.array_equal(bary.cpu().numpy(), obary.cpu().numpy(), equal_nan=True)


def test_two_runs_are_bit_identical():
    from sdfstudio_b200 import texturing

    uv = random_charts(20000, 3)
    a = texturing.uv_rasterize(uv, 512)
    b = texturing.uv_rasterize(uv, 512)
    assert torch.equal(a[0], b[0]) and np.array_equal(a[1].cpu().numpy(), b[1].cpu().numpy(), equal_nan=True)


def test_one_texel():
    from sdfstudio_b200 import texturing

    vertices, faces, normals, uvs, _ = case_inputs("xatlas_30")
    tc, o, d = texturing.rasterize_uv(uvs.cuda(), vertices.cuda(), faces.cuda(), normals.cuda(), num_pixels_per_side=1)
    oface, obary = otex.rasterize(uvs, 1, 10)
    oo, od = otex.texel_rays(vertices, faces, normals, oface, obary)
    assert o.shape == (1, 1, 3) and torch.equal(o.cpu().view(1, 3), oo)
    assert (d.cpu().view(1, 3) - od).abs().max() <= RAY_ATOL


def test_public_unwraps_match_oracle():
    from sdfstudio_b200 import texturing

    vertices, faces, normals, _, _ = case_inputs("custom_odd")
    tc, o, d = texturing.unwrap_mesh_per_uv_triangle(vertices.cuda(), faces.cuda(), normals.cuda(), 4)
    otc, oface, obary, hw = otex.grid_unwrap(len(faces), 4, "cpu")
    oo, od = otex.texel_rays(vertices, faces, normals, oface, obary)
    assert torch.equal(tc.cpu(), otc) and torch.equal(o.cpu(), oo.view(*hw, 3))
    assert (d.cpu() - od.view(*hw, 3)).abs().max() <= RAY_ATOL


# ---------------------------------------------------------------------------------------------------------------------------------
# export_textured_mesh on a SurfaceRenderer
# ---------------------------------------------------------------------------------------------------------------------------------
def test_export_on_surface_renderer(tmp_path):
    import sdfstudio_b200 as sb
    from sdfstudio_b200 import meshing, texturing
    from test_gpu_meshing import _field

    field = _field("fp32")                    # perturbed SDFField with a closed surface inside the box
    res = 48
    with torch.no_grad():
        vol = meshing.evaluate_sdf_grid(field, res)
    verts, faces, normals = meshing.marching_cubes(vol, 0.0, (2.0 / (res - 1),) * 3)
    assert len(faces) > 500
    mesh = meshing.Mesh(verts.double().cpu().numpy() - 1.0, faces.cpu().numpy(), normals.cpu().numpy())
    renderer = sb.SurfaceRenderer(field, sb.NeuSSampler(num_samples=32, num_samples_importance=32).eval(), kind="neus").eval()
    texturing.export_textured_mesh(mesh, renderer, tmp_path, px_per_uv_triangle=3, unwrap_method="custom")

    # the oracle's texel bundle, rendered by the same renderer and quantised as the PNG is
    v = torch.from_numpy(mesh.vertices).float().cuda()
    f = torch.from_numpy(mesh.faces).cuda()
    n = torch.from_numpy(mesh.vertex_normals).float().cuda()
    otc, oface, obary, hw = otex.grid_unwrap(len(f), 3, "cuda")
    oo, od = otex.texel_rays(v, f, n, oface, obary)
    b = otex.texel_bundle(oo.view(*hw, 3), od.view(*hw, 3), otex.ray_length(v, f))
    with torch.no_grad():
        rgb = renderer.get_outputs_for_camera_ray_bundle(sb.RayBundle(**b))["rgb"].view(*hw, 3).cpu().numpy()
    want = np.floor(np.clip(rgb, 0, 1) * 255 + 0.5).astype(np.int32)
    got = decode_png((tmp_path / "material_0.png").read_bytes()).astype(np.int32)
    assert got.shape == want.shape
    # the kernel's directions may differ from the oracle's in the last bit (normalize's reduction order): a colour on a rounding edge
    # can then land one level away; measured on the H100, see DESIGN.md section 3
    assert np.abs(got - want).max() <= 1 and (got == want).mean() >= 0.999

    obj = parse_obj((tmp_path / "mesh.obj").read_text())
    assert np.array_equal(obj["v"].astype(np.float32), mesh.vertices.astype(np.float32))
    assert np.array_equal(obj["vn"].astype(np.float32), mesh.vertex_normals.astype(np.float32))
    assert np.array_equal(obj["vt"][:, 0].astype(np.float32), otc.cpu().numpy().reshape(-1, 2)[:, 0])
    assert np.array_equal(obj["f"][:, :, 0] - 1, mesh.faces)
    assert (tmp_path / "material_0.mtl").read_text().endswith("map_Kd material_0.png\n")
