"""GPU checks of the Poisson reconstruction (csrc/poisson.cu) against the fp64 oracle (oracle/poisson.py) at depths 3 to 6 on sphere,
torus, open-plane and clustered clouds: the right-hand side, the screening diagonal and the operator within fp32 rounding of their
fp64 sums, chi within 1e-4 ||chi*||_inf with the reported residual meeting the stopping rule, the iso value, the densities and colours;
then the depth-8 geometry against the bounds of test_poisson_cpu, determinism, refusals that launch nothing, a depth-9 solve of 1 M
points, and the export flow on a SurfaceRenderer (its mesh follows the rendered cloud, and the default normal output is refused before
any point is rendered)."""
import numpy as np
import pytest
import torch

from oracle import poisson as op
from test_poisson_cpu import SPHERE_BOUND_H, outward_fraction, topology

pytestmark = pytest.mark.gpu
U32 = 2.0 ** -24
CASES = [("sphere", 3), ("sphere", 5), ("sphere", 6), ("torus", 4), ("torus", 6), ("plane", 5), ("clusters", 3), ("clusters", 6)]


@pytest.fixture(autouse=True)
def _keep_global_rng():
    """Every test here restores the global CPU and CUDA generators, as test_gpu_pointcloud does."""
    with torch.random.fork_rng(devices=range(torch.cuda.device_count())):
        yield


def _cuda(*arrays):
    return [torch.from_numpy(a).cuda() for a in arrays]


def _system(name, depth, n=20000):
    from sdfstudio_b200 import poisson

    p, nrm, c = op.CLOUDS[name](n)
    return poisson.build_system(*_cuda(p, nrm, c), depth=depth), op.assemble(p, nrm, depth), (p, nrm, c)


@pytest.mark.parametrize("name,depth", CASES)
def test_against_oracle(name, depth):
    from sdfstudio_b200 import poisson

    gs, os_, (p, nrm, c) = _system(name, depth)
    assert gs.origin == pytest.approx(os_["origin"], abs=0) and gs.h == os_["h"] and gs.alpha_a == os_["alpha_a"]
    # a b: double sums rounded to fp32 once, then scaled by a; bound c u sum |terms|
    cc, u = op.locate(os_["points"], os_["origin"], os_["h"], os_["n"])
    phi, grad = op.hats(u)
    ids = op.corner_nodes(cc, os_["n"])
    _, nn, _ = op.usable(p, nrm)
    absterm = np.bincount(ids.ravel(), weights=np.abs(np.einsum("pla,pa->pl", grad, nn) / os_["h"]).ravel(), minlength=len(os_["b"]))
    rhs = gs.rhs.cpu().numpy().astype(np.float64)
    assert (np.abs(rhs - os_["a"] * os_["b"]) <= 16 * U32 * os_["a"] * absterm + 1e-300).all()
    # S diagonal: the corner diagonal entries of the adjacent cells' blocks
    sdiag = poisson.node_gather(gs, depth, gs.mats[depth], 64, 9, 1)[:, 0].cpu().numpy()
    sd = os_["S"].diagonal()
    assert (np.abs(sdiag - sd) <= 16 * U32 * sd).all()
    # the operator on a random vector
    x = torch.randn(len(rhs), generator=torch.Generator().manual_seed(depth)).cuda()
    y = poisson.apply_operator(gs, depth, x).cpu().numpy()
    A = os_["L"] + os_["alpha_a"] * os_["S"]
    Aabs = abs(os_["L"]) + os_["alpha_a"] * os_["S"]
    xd = x.cpu().numpy().astype(np.float64)
    assert (np.abs(y - A @ xd) <= 32 * U32 * (Aabs @ np.abs(xd))).all()
    # the solve
    poisson.solve(gs)
    op.solve(os_)
    assert 1 <= gs.cycles <= poisson.MAX_CYCLES and gs.residual <= poisson.TOL
    chi = gs.chi.cpu().numpy()
    scale = np.abs(os_["chi"]).max()
    assert np.abs(chi - os_["chi"]).max() <= 1e-4 * scale
    assert abs(gs.iso - os_["iso"]) <= 1e-4 * scale
    # densities and colours at the GPU's vertices, against the oracle's splat at the same points
    mesh, dens = poisson.mesh_from_system(gs)
    _, _, col = op.usable(p, nrm, c)
    lvl, hl, nodes = op.splat(os_["points"], col, depth, os_["origin"], os_["h"])
    at = op.interpolate(mesh.vertices, os_["origin"], hl, 2 ** lvl, nodes)
    d = dens.cpu().numpy()
    np.testing.assert_allclose(d, at[:, 0], rtol=1e-5, atol=1e-6 * at[:, 0].max())
    ok = at[:, 0] > 1e-3 * at[:, 0].max()
    np.testing.assert_allclose(mesh.vertex_colors[ok], at[ok, 1:] / at[ok, :1], atol=1e-4)
    # the meshes: the oracle's mesh of its own chi, compared by nearest vertices both ways and by Euler characteristic
    _, ov, of, _, _, _ = op.reconstruct(p, nrm, c, depth)
    from scipy.spatial import cKDTree

    assert cKDTree(ov).query(mesh.vertices)[0].max() <= 0.05 * gs.h
    assert cKDTree(mesh.vertices).query(ov)[0].max() <= 0.05 * gs.h
    assert topology(mesh.vertices, mesh.faces)[1] == topology(ov, of)[1]


@pytest.mark.parametrize("name,euler", [("sphere", 2), ("torus", 0)])
def test_depth8_geometry(name, euler):
    import sdfstudio_b200 as sb
    from sdfstudio_b200 import poisson

    p, nrm, c = op.CLOUDS[name](400000)
    mesh, dens = poisson.create_from_point_cloud_poisson(sb.PointCloud(*_cuda(p, c, nrm)), depth=8)
    closed, e = topology(mesh.vertices, mesh.faces)
    assert closed and e == euler
    h = poisson.build_system(*_cuda(p, nrm, c), depth=8).h
    v = mesh.vertices
    if name == "sphere":
        dist = np.abs(np.linalg.norm(v, axis=1) - 0.6)
        centre = lambda x: 0 * x  # noqa: E731
    else:
        ring = np.linalg.norm(v[:, :2], axis=1)
        dist = np.abs(np.hypot(ring - 0.6, v[:, 2]) - 0.25)
        centre = lambda x: np.concatenate([0.6 * x[:, :2] / np.linalg.norm(x[:, :2], axis=1, keepdims=True), 0 * x[:, 2:]], 1)  # noqa: E731
    assert dist.max() <= SPHERE_BOUND_H * h
    # a sliver (a cut within rounding of a node) has no meaningful normal: every face of doubled area > 1e-4 h^2 points outward
    f = mesh.faces
    big = np.linalg.norm(np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]), axis=1) > 1e-4 * h * h
    assert big.mean() > 0.99 and outward_fraction(v, f[big], centre) == 1.0
    assert (dens > 0).all()


def test_plane_trimmed():
    import sdfstudio_b200 as sb
    from sdfstudio_b200 import poisson

    p, nrm, c = op.plane_cloud(300000)
    mesh, dens = poisson.create_from_point_cloud_poisson(sb.PointCloud(*_cuda(p, c, nrm)), depth=8)
    h = poisson.build_system(*_cuda(p, nrm, c), depth=8).h
    poisson.remove_vertices_by_mask(mesh, poisson.low_density_mask(dens))
    assert len(mesh.faces) > 0
    assert np.abs(mesh.vertices[:, 2] - 0.1).max() <= 2 * h


def test_deterministic():
    import sdfstudio_b200 as sb
    from sdfstudio_b200 import poisson

    p, nrm, c = op.clustered_cloud(50000)
    runs = [poisson.create_from_point_cloud_poisson(sb.PointCloud(*_cuda(p, c, nrm)), depth=7) for _ in range(2)]
    (m0, d0), (m1, d1) = runs
    np.testing.assert_array_equal(m0.vertices, m1.vertices)
    np.testing.assert_array_equal(m0.faces, m1.faces)
    np.testing.assert_array_equal(m0.vertex_colors, m1.vertex_colors)
    assert torch.equal(d0, d1)


def test_refusals_launch_nothing():
    import ctypes as C

    from sdfstudio_b200 import _lib, poisson

    p, nrm, c = _cuda(*op.sphere_cloud(1000))
    bad = [dict(depth=0), dict(depth=11), dict(points=p[:0], normals=nrm[:0], colors=c[:0]), dict(points=torch.zeros_like(p)),
           dict(normals=torch.zeros_like(nrm)), dict(points=torch.where(torch.arange(1000, device="cuda")[:, None] == 7, float("inf"), p))]
    before = _lib.launch_count()
    for kw in bad:
        args = dict(points=p, normals=nrm, colors=c, depth=5) | kw
        with pytest.raises(ValueError):
            poisson.build_system(**args)
    lib = _lib.load()
    o = (C.c_double * 3)(0, 0, 0)
    assert lib.sdfb200_poisson_cells(None, None, None, 1, None, None, 11, o, 1.0, None, None, None, None) != 0
    assert lib.sdfb200_poisson_sample(None, 1, 3, o, -1.0, None, 1, None, None) != 0
    assert lib.sdfb200_poisson_apply(3, 1.0, None, None, 1.0, None, None, None) != 0
    assert lib.sdfb200_poisson_workspace_bytes(0) == 0 and lib.sdfb200_poisson_workspace_bytes(11) == 0
    x = C.c_int32(0)
    r = C.c_double(0)
    assert lib.sdfb200_poisson_solve(0, 1.0, None, None, 1.0, None, None, 30, 1e-5, None, 0, C.byref(x), C.byref(r), None) != 0
    torch.cuda.synchronize()
    assert _lib.launch_count() == before


def test_depth9_million_points():
    from sdfstudio_b200 import poisson

    p, nrm, c = op.sphere_cloud(1000000)
    s = poisson.solve(poisson.build_system(*_cuda(p, nrm, c), depth=9))
    assert 1 <= s.cycles <= poisson.MAX_CYCLES and s.residual <= poisson.TOL


def _renderer():
    """An SDFField at its geometric initialisation (an SDF close to |x| - 0.5) with a sharp NeuS variance (beta_init 0.7: inv_s = e^7),
    so that the rendered depth lands on the sphere."""
    import sdfstudio_b200 as sb

    cfg = sb.SDFFieldConfig(use_grid_feature=True, num_layers=2, num_layers_color=2, inside_outside=False, bias=0.5, beta_init=0.7,
                            precision="fp32")
    torch.manual_seed(0)
    field = sb.SDFField(cfg, torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), num_images=49).cuda().eval()
    return sb.SurfaceRenderer(field, sb.NeuSSampler(num_samples=64, num_samples_importance=64).eval(),
                              collider=sb.NearFarCollider(0.05, 4.0), kind="neus").eval()


def test_poisson_mesh_flow(tmp_path):
    """80 cameras at distance 2.2 whose whole frame (half-diagonal 8.9 degrees) falls on the sphere (13.1 degrees): every ray hits it,
    and 400 k points give the depth-9 grid about 0.6 points per surface cell."""
    from oracle.make_golden_tsdf import look_at, on_sphere
    from sdfstudio_b200 import meshing, poisson
    from sdfstudio_b200.cameras import Cameras

    renderer = _renderer()
    cams = Cameras(look_at(on_sphere(80, 2.2, 3))[:, :3, :], 400.0, 400.0, 48.0, 40.0, 96, 80, device=torch.device("cuda"))
    kw = dict(num_points=400000, num_rays_per_batch=32768, normal_output_name="normal", seed=3)
    with pytest.raises(ValueError, match="Normal output 'normals' not found"):
        poisson.poisson_mesh(renderer, cams, tmp_path / "defaults")
    assert not (tmp_path / "defaults" / "poisson_mesh.ply").exists()
    mesh, dens = poisson.poisson_mesh(renderer, cams, tmp_path / "a", texture_method="point_cloud", save_point_cloud=True, **kw)
    v, f, _ = meshing.read_ply(str(tmp_path / "a" / "poisson_mesh.ply"))
    assert len(f) > 100 and len(v) == len(mesh.vertices) == len(dens)
    assert mesh.solve_residual <= poisson.TOL
    assert (tmp_path / "a" / "point_cloud.ply").exists()
    cloud, _, _ = meshing.read_ply(str(tmp_path / "a" / "point_cloud.ply"))
    h = 1.1 * float((cloud.max(0) - cloud.min(0)).max()) / 2 ** 9
    # Every trimmed vertex lies on the field's zero level set, up to the rendered depth's own offset (the expected depth of 64 + 64
    # NeuS samples sits a few h off the level set): measured on an H100, |sdf| / h is 2.5 at the median, 5.1 at the 99th percentile
    # and 7.1 at most.  The geometric initialisation puts that level set near, not on, the sphere of radius bias: the vertices' |r - 0.5|
    # is 0.04 at the median and 0.095 at most.
    sdf = meshing.sdf_fn(renderer.field)(torch.from_numpy(v).cuda()).abs().cpu().numpy()
    assert np.quantile(sdf, 0.99) <= 6 * h and sdf.max() <= 8 * h
    assert np.abs(np.linalg.norm(v, axis=1) - 0.5).max() <= 0.12
    poisson.poisson_mesh(renderer, cams, tmp_path / "b", texture_method="nerf", unwrap_method="custom", target_num_faces=None, **kw)
    assert (tmp_path / "b" / "mesh.obj").exists()
