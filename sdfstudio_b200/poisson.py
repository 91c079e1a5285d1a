"""Poisson surface reconstruction on the GPU: drop-ins for open3d's ``TriangleMesh.create_from_point_cloud_poisson`` and
``remove_vertices_by_mask`` as ``ns-export poisson`` (``scripts/exporter.py:173-303``, ExportPoissonMesh) calls them, and for that
exporter's ``main``.

open3d's solver is Kazhdan's adaptive-octree screened Poisson reconstruction with degree-2 B-splines; it is not a dependency and its
source is not pinned, so it is not reproduced.  Here the same inputs give a screened Poisson surface of the same cloud on a dense grid
with trilinear (Q1) elements, whose discretisation include/sdfb200.h states once: the mesh is not open3d's mesh.  The solve, the
sampling and the splats are CUDA (csrc/poisson.cu), the iso-surface is ``meshing.marching_cubes``.
"""
import ctypes as C
import math
import warnings
from dataclasses import dataclass
from pathlib import Path
from typing import List, Optional, Tuple

import numpy as np
import torch

from . import _lib, meshing, pointcloud, texturing

SCALE = 1.1
POINT_WEIGHT = 4.0
"""alpha, PoissonRecon's default point weight (SDFB200_POISSON_POINT_WEIGHT)."""
KERNEL_DEPTH_OFFSET = 2
"""Densities and colours are splatted at depth - 2 (PoissonRecon's kernel depth), at least 0."""
MAX_CYCLES = 30
TOL = 1e-5
MIN_DEPTH, MAX_DEPTH = 1, 10


@dataclass
class PoissonSystem:
    """The grid, the hierarchy and the solution of one reconstruction (device tensors)."""

    depth: int
    origin: Tuple[float, float, float]
    h: float
    alpha_a: float
    points: torch.Tensor          # [N,3] the points that take part, in bucket order
    colors: torch.Tensor          # [N,3]
    slots: List[Optional[torch.Tensor]]   # per level l = 0 .. depth: [n_l^3] int32 (None for l = 0)
    mats: List[Optional[torch.Tensor]]    # per level: [cells, 8, 8] fp32
    rhs: torch.Tensor             # [(n+1)^3] fp32, a b
    chi: Optional[torch.Tensor] = None    # [(n+1)^3] fp32
    cycles: int = 0
    residual: float = float("nan")
    iso: float = float("nan")


def _cells(level_coords: torch.Tensor, n: int):
    key = (level_coords[:, 0] * n + level_coords[:, 1]) * n + level_coords[:, 2]
    return key


def _slot_map(keys: torch.Tensor, n: int) -> torch.Tensor:
    slot = torch.full((n ** 3,), -1, dtype=torch.int32, device=keys.device)
    slot[keys] = torch.arange(keys.numel(), dtype=torch.int32, device=keys.device)
    return slot


def _bucket(points: torch.Tensor, keys: torch.Tensor):
    """Stable sort by cell key: (order, the occupied keys ascending, their start offsets [cells+1] int64)."""
    skey, order = torch.sort(keys, stable=True)
    occ, counts = torch.unique_consecutive(skey, return_counts=True)
    start = torch.zeros(occ.numel() + 1, dtype=torch.int64, device=keys.device)
    torch.cumsum(counts, 0, out=start[1:])
    return order, occ, start


def _host3(v):
    return (C.c_double * 3)(*[float(x) for x in v])


def cube(points: torch.Tensor, depth: int, scale: float = SCALE):
    """(origin, h) of the grid: centre c of the box, W = scale * largest extent, h = W / 2^depth, origin = c - W / 2, all in double.
    A box of zero extent raises ValueError."""
    box = torch.cat([points.amin(0), points.amax(0)]).double().cpu().tolist()
    extent = max(box[a + 3] - box[a] for a in range(3))
    if not extent > 0:
        raise ValueError("the point cloud's box has zero extent")
    w = scale * extent
    centre = [(box[a] + box[a + 3]) / 2 for a in range(3)]
    return tuple(c - w / 2 for c in centre), w / 2 ** depth


def _check(points, normals, colors, depth, scale):
    if not isinstance(depth, (int, np.integer)) or not MIN_DEPTH <= int(depth) <= MAX_DEPTH:
        raise ValueError(f"depth must be an integer in [{MIN_DEPTH}, {MAX_DEPTH}], got {depth!r}")
    if not (math.isfinite(scale) and scale >= 1.0):
        raise ValueError(f"scale must be finite and >= 1, got {scale}")
    if points.dim() != 2 or points.shape[1] != 3 or normals is None or tuple(normals.shape) != tuple(points.shape):
        raise ValueError("expected points [N,3] and normals [N,3]")
    if colors is not None and tuple(colors.shape) != tuple(points.shape):
        raise ValueError("expected colors [N,3]")
    if points.shape[0] == 0:
        raise ValueError("the point cloud is empty")
    if not bool(torch.isfinite(points).all()):
        raise ValueError("the point cloud holds a non-finite coordinate")


def build_system(points: torch.Tensor, normals: torch.Tensor, colors: Optional[torch.Tensor] = None, depth: int = 8,
                 scale: float = SCALE) -> PoissonSystem:
    """Everything before the solve: the points that take part (finite, non-zero normal), the cube, the buckets, the screening blocks of
    every level (fine ones from the points, coarse ones by sdfb200_poisson_coarsen) and a b.  Refusals raise ValueError before any
    launch."""
    _check(points, normals, colors, depth, scale)
    depth = int(depth)
    pts, nrm = _lib.f32c(points), _lib.f32c(normals)
    col = _lib.f32c(colors) if colors is not None else torch.zeros_like(pts)
    valid = torch.isfinite(nrm).all(1) & (nrm != 0).any(1)
    pts, nrm, col = pts[valid], nrm[valid], col[valid]
    n_pts = pts.shape[0]
    if n_pts == 0:
        raise ValueError("no point has a finite, non-zero normal")
    origin, h = cube(pts, depth, scale)
    _lib.require_cuda(pts.device, "poisson")
    lib, st = _lib.load(), _lib.stream_ptr()
    n = 2 ** depth
    o_t = torch.tensor(origin, dtype=torch.float64, device=pts.device)
    cell = torch.floor((pts.double() - o_t) / h).clamp_(0, n - 1).long()
    order, occ, start = _bucket(pts, _cells(cell, n))
    pts, nrm, col, cell = pts[order].contiguous(), nrm[order].contiguous(), col[order].contiguous(), cell[order]
    a = h * h * occ.numel() / n_pts
    slots: List[Optional[torch.Tensor]] = [None] * (depth + 1)
    mats: List[Optional[torch.Tensor]] = [None] * (depth + 1)
    slots[depth] = _slot_map(occ, n)
    mats[depth] = torch.empty(occ.numel(), 8, 8, device=pts.device)
    rhs_cells = torch.empty(occ.numel(), 8, device=pts.device)
    _lib.check(lib.sdfb200_poisson_cells(_lib.ptr(pts), _lib.ptr(nrm), None, occ.numel(), _lib.ptr(occ), _lib.ptr(start), depth,
                                         _host3(origin), h, _lib.ptr(mats[depth]), _lib.ptr(rhs_cells), None, st), "sdfb200_poisson_cells")
    coords = torch.stack([occ // (n * n), (occ // n) % n, occ % n], 1)
    for lvl in range(depth - 1, 0, -1):
        nl = 2 ** lvl
        coords = torch.unique(coords >> 1, dim=0)      # rows sorted lexicographically: keys ascending
        keys = _cells(coords, nl)
        slots[lvl] = _slot_map(keys, nl)
        mats[lvl] = torch.empty(keys.numel(), 8, 8, device=pts.device)
        _lib.check(lib.sdfb200_poisson_coarsen(lvl, _lib.ptr(slots[lvl + 1]), _lib.ptr(mats[lvl + 1]), keys.numel(), _lib.ptr(keys),
                                               _lib.ptr(mats[lvl]), st), "sdfb200_poisson_coarsen")
    b = torch.empty((n + 1) ** 3, device=pts.device)
    _lib.check(lib.sdfb200_poisson_gather(depth, _lib.ptr(slots[depth]), _lib.ptr(rhs_cells), 8, 1, 1, _lib.ptr(b), st),
               "sdfb200_poisson_gather")
    b.mul_(a)   # in place: at depth 10 the node vector alone is 4.3 GB
    return PoissonSystem(depth, origin, h, POINT_WEIGHT * a, pts, col, slots, mats, b)


def node_gather(system: PoissonSystem, level: int, cell_vals: torch.Tensor, cell_stride: int, corner_stride: int, channels: int,
                slot: Optional[torch.Tensor] = None) -> torch.Tensor:
    """sdfb200_poisson_gather at ``level`` (the level's slot map unless ``slot`` is given): [(n+1)^3, channels] fp32."""
    out = torch.empty((2 ** level + 1) ** 3, channels, device=cell_vals.device)
    slot = system.slots[level] if slot is None else slot
    _lib.check(_lib.load().sdfb200_poisson_gather(level, _lib.ptr(slot), _lib.ptr(cell_vals.contiguous()), cell_stride, corner_stride,
                                                  channels, _lib.ptr(out), _lib.stream_ptr()), "sdfb200_poisson_gather")
    return out


def apply_operator(system: PoissonSystem, level: int, x: torch.Tensor) -> torch.Tensor:
    """(L + alpha a S) x at ``level`` (sdfb200_poisson_apply)."""
    y = torch.empty_like(x)
    h = system.h * 2 ** (system.depth - level)
    _lib.check(_lib.load().sdfb200_poisson_apply(level, h, _lib.ptr(system.slots[level]), _lib.ptr(system.mats[level]), system.alpha_a,
                                                 _lib.ptr(_lib.f32c(x)), _lib.ptr(y), _lib.stream_ptr()), "sdfb200_poisson_apply")
    return y


def sample(points: torch.Tensor, level: int, origin, h: float, node_vals: torch.Tensor, channels: int) -> torch.Tensor:
    """Trilinear interpolation of node values [(n+1)^3, channels] at points [P,3] on the grid of ``level``: [P, channels] double."""
    out = torch.empty(points.shape[0], channels, dtype=torch.float64, device=points.device)
    if points.shape[0]:
        _lib.check(_lib.load().sdfb200_poisson_sample(_lib.ptr(_lib.f32c(points)), points.shape[0], level, _host3(origin), h,
                                                      _lib.ptr(node_vals.contiguous()), channels, _lib.ptr(out), _lib.stream_ptr()),
                   "sdfb200_poisson_sample")
    return out


def solve(system: PoissonSystem, max_cycles: int = MAX_CYCLES, tol: float = TOL) -> PoissonSystem:
    """sdfb200_poisson_solve, then the iso value (the mean of chi at the points, summed by sdfb200_poisson_sum)."""
    lib, st = _lib.load(), _lib.stream_ptr()
    d = system.depth
    dev = system.rhs.device
    ws = torch.empty(lib.sdfb200_poisson_workspace_bytes(d), dtype=torch.uint8, device=dev)
    slot_ptrs = (C.c_void_p * (d + 1))(*[_lib.ptr(s) if s is not None else None for s in system.slots])
    mat_ptrs = (C.c_void_p * (d + 1))(*[_lib.ptr(m) if m is not None else None for m in system.mats])
    x = torch.empty_like(system.rhs)
    cycles, res = C.c_int32(0), C.c_double(0.0)
    _lib.check(lib.sdfb200_poisson_solve(d, system.h, slot_ptrs, mat_ptrs, system.alpha_a, _lib.ptr(system.rhs), _lib.ptr(x), max_cycles,
                                         tol, _lib.ptr(ws), ws.numel(), C.byref(cycles), C.byref(res), st), "sdfb200_poisson_solve")
    system.chi, system.cycles, system.residual = x, int(cycles.value), float(res.value)
    chi_p = sample(system.points, d, system.origin, system.h, x, 1)
    partial = torch.empty(1024, dtype=torch.float64, device=dev)
    total = torch.empty(1, dtype=torch.float64, device=dev)
    _lib.check(lib.sdfb200_poisson_sum(_lib.ptr(chi_p), chi_p.numel(), _lib.ptr(partial), _lib.ptr(total), st), "sdfb200_poisson_sum")
    system.iso = float(total.item()) / system.points.shape[0]
    return system


def splat(system: PoissonSystem) -> Tuple[int, torch.Tensor]:
    """(level, node values [(n+1)^3, 4]): per node of the grid at depth - 2 the sums sum phi and sum phi rgb over the points."""
    lvl = max(system.depth - KERNEL_DEPTH_OFFSET, 0)
    n = 2 ** lvl
    h = system.h * 2 ** (system.depth - lvl)
    pts = system.points
    o_t = torch.tensor(system.origin, dtype=torch.float64, device=pts.device)
    cell = torch.floor((pts.double() - o_t) / h).clamp_(0, n - 1).long()
    order, occ, start = _bucket(pts, _cells(cell, n))
    sp, sc = pts[order].contiguous(), system.colors[order].contiguous()
    cells = torch.empty(occ.numel(), 8, 4, device=pts.device)
    _lib.check(_lib.load().sdfb200_poisson_cells(_lib.ptr(sp), None, _lib.ptr(sc), occ.numel(), _lib.ptr(occ), _lib.ptr(start), lvl,
                                                 _host3(system.origin), h, None, None, _lib.ptr(cells), _lib.stream_ptr()),
               "sdfb200_poisson_cells")
    return lvl, node_gather(system, lvl, cells, 32, 4, 4, slot=_slot_map(occ, n))


def create_from_point_cloud_poisson(pcd: "pointcloud.PointCloud", depth: int = 8, scale: float = SCALE):
    """open3d's ``TriangleMesh.create_from_point_cloud_poisson(pcd, depth, scale=scale)`` on a :class:`pointcloud.PointCloud` with normals.
    Returns (mesh, densities): a ``meshing.Mesh`` (vertices, faces, vertex normals, and ``vertex_colors`` [V,3] in [0, 1]) and the
    densities [V] fp64 on the device.  The mesh also carries ``solve_cycles`` and ``solve_residual`` (the relative residual of the
    solve); a solve that stops at the cycle cap above the tolerance warns with RuntimeWarning.

    Restated from open3d / PoissonRecon: the cube (centre of the box, ``scale`` times the largest extent, 2^depth cells per side), the
    normalised normals without confidence, the point weight alpha = 4, the iso value as the mean of chi over the points, the density as
    the points' splat at depth - 2 interpolated at the vertices, and colours as the splatted colours over that density.
    Not pinned: the solver (a dense Q1 grid here, an adaptive B-spline octree in open3d), so vertex positions, counts and densities
    differ from open3d's; whether open3d's wrapper passes alpha = 4 could not be checked.  Faces are wound so that their normals point
    along the input normals.  Deterministic: reruns give bit-identical results.  ``depth`` outside [1, 10], an empty cloud, a cloud
    without a finite, non-zero normal, a box of zero extent or a non-finite point raise ValueError before any launch."""
    if pcd.normals is None:
        raise ValueError("create_from_point_cloud_poisson needs a point cloud with normals")
    system = solve(build_system(pcd.points, pcd.normals, pcd.colors, depth, scale))
    if not system.residual <= TOL:
        warnings.warn(f"create_from_point_cloud_poisson: the solve stopped after {system.cycles} cycles at a relative residual of "
                      f"{system.residual:.3g}, above {TOL:g}; the surface comes from an unconverged chi", RuntimeWarning, stacklevel=2)
    mesh, densities = mesh_from_system(system)
    mesh.solve_cycles, mesh.solve_residual = system.cycles, system.residual
    return mesh, densities


def mesh_from_system(system: PoissonSystem):
    """(mesh, densities) of a solved system: marching cubes of -chi at -iso, then the density and colour at the vertices."""
    m = 2 ** system.depth + 1
    verts, faces, normals = meshing.marching_cubes((-system.chi).view(m, m, m), level=-system.iso, spacing=(system.h,) * 3)
    verts = verts + torch.tensor(system.origin, dtype=torch.float32, device=verts.device)
    lvl, nodes = splat(system)
    at = sample(verts, lvl, system.origin, system.h * 2 ** (system.depth - lvl), nodes, 4)
    dens = at[:, 0]
    colors = torch.where(dens[:, None] > 0, at[:, 1:] / torch.where(dens > 0, dens, 1.0)[:, None], 0.0)
    mesh = meshing.Mesh(verts.cpu().numpy(), faces.cpu().numpy(), normals.cpu().numpy())
    mesh.vertex_colors = colors.cpu().numpy()
    return mesh, dens


def remove_vertices_by_mask(mesh, mask):
    """open3d's ``TriangleMesh.remove_vertices_by_mask``: drops the vertices where ``mask`` [V] is set and every face that touches one,
    keeps the other vertices (with their normals and colours) in order and reindexes the faces.  Modifies ``mesh`` and returns it."""
    mask = np.asarray(mask.cpu() if isinstance(mask, torch.Tensor) else mask, dtype=bool).reshape(-1)
    if mask.shape[0] != len(mesh.vertices):
        raise ValueError(f"mask has {mask.shape[0]} entries for {len(mesh.vertices)} vertices")
    keep = ~mask
    new_index = np.cumsum(keep) - 1
    faces = np.asarray(mesh.faces, dtype=np.int64).reshape(-1, 3)
    faces = faces[keep[faces].all(1)] if len(faces) else faces
    mesh.faces = new_index[faces].astype(np.int64).reshape(-1, 3)
    mesh.vertices = mesh.vertices[keep]
    mesh.vertex_normals = mesh.vertex_normals[keep]
    if getattr(mesh, "vertex_colors", None) is not None:
        mesh.vertex_colors = mesh.vertex_colors[keep]
    return mesh


def low_density_mask(densities, q: float = 0.1) -> np.ndarray:
    """``densities < np.quantile(densities, q)`` (numpy's linear interpolation) on the host; strict, so equal densities keep all."""
    d = np.asarray(densities.cpu() if isinstance(densities, torch.Tensor) else densities, dtype=np.float64).reshape(-1)
    if d.size == 0:
        return np.zeros(0, dtype=bool)
    return d < np.quantile(d, q)


def _normal_check_message(name, outputs) -> str:
    return (f"Warning: Normal output '{name}' not found in pipeline outputs.\nAvailable outputs: {list(outputs.keys())}\n"
            "Warning: Please train a model with normals (e.g., nerfacto with predicted normals turned on).\n"
            "Warning: Or change --normal-method\nExiting early.")


def validate_pipeline(model, normal_method: str, normal_output_name: str) -> None:
    """ExportPoissonMesh.validate_pipeline (:213-235): with ``normal_method="model_output"``, render one ray (origin 0, direction
    (1, 1, 1)) and raise ValueError with the reference's messages if ``normal_output_name`` is not an output."""
    if normal_method != "model_output":
        return
    model, device = texturing.model_and_device(model)
    origins = torch.zeros((1, 3), device=device)
    one = torch.ones_like(origins[..., :1])
    bundle = texturing._ray_bundle_class(model)(origins=origins, directions=torch.ones_like(origins), pixel_area=one,
                                                camera_indices=torch.zeros_like(one), directions_norm=one)
    with torch.no_grad():
        outputs = model(bundle)
    if normal_output_name not in outputs:
        raise ValueError(_normal_check_message(normal_output_name, outputs))


def poisson_mesh(renderer, cameras, output_dir, num_points: int = 1000000, remove_outliers: bool = True, depth_output_name: str = "depth",
                 rgb_output_name: str = "rgb", normal_method: str = "model_output", normal_output_name: str = "normals",
                 save_point_cloud: bool = False, use_bounding_box: bool = True,
                 bounding_box_min: Tuple[float, float, float] = (-1, -1, -1), bounding_box_max: Tuple[float, float, float] = (1, 1, 1),
                 num_rays_per_batch: int = 32768, texture_method: str = "nerf", px_per_uv_triangle: int = 4,
                 unwrap_method: str = "xatlas", num_pixels_per_side: int = 2048, target_num_faces: Optional[int] = 50000,
                 std_ratio: float = 10.0, seed: int = 0):
    """ExportPoissonMesh.main (scripts/exporter.py:237-303) on a renderer (a SurfaceRenderer) and the package's :class:`Cameras`.  The
    normal check first (:func:`validate_pipeline`), then ``pointcloud.generate_point_cloud`` with rays from a seeded restatement of the
    reference's pixel sampler (``seed``), the depth-9 reconstruction, the trim ``densities < quantile(densities, 0.1)``, optionally
    ``point_cloud.ply``, then ``poisson_mesh.ply`` and, with ``texture_method="nerf"``, the textured mesh through ``texturing``.
    With ``normal_method="open3d"`` the normals are ``pointcloud.estimate_normals`` and, as in the reference, not oriented.  Returns
    (the trimmed mesh, its densities)."""
    if normal_method not in ("open3d", "model_output"):
        raise ValueError(f"normal_method must be 'open3d' or 'model_output', got {normal_method!r}")
    if texture_method not in ("point_cloud", "nerf"):
        raise ValueError(f"texture_method must be 'point_cloud' or 'nerf', got {texture_method!r}")
    output_dir = Path(output_dir)
    output_dir.mkdir(parents=True, exist_ok=True)
    validate_pipeline(renderer, normal_method, normal_output_name)
    model, _ = texturing.model_and_device(renderer)
    pipeline = pointcloud._RendererPipeline(model, pointcloud._PixelRays(cameras, num_rays_per_batch, seed))
    pcd = pointcloud.generate_point_cloud(
        pipeline, num_points=num_points, remove_outliers=remove_outliers, estimate_normals=normal_method == "open3d",
        rgb_output_name=rgb_output_name, depth_output_name=depth_output_name,
        normal_output_name=normal_output_name if normal_method == "model_output" else None, use_bounding_box=use_bounding_box,
        bounding_box_min=bounding_box_min, bounding_box_max=bounding_box_max, std_ratio=std_ratio)
    if save_point_cloud:
        pcd.export(output_dir / "point_cloud.ply")
    mesh, densities = create_from_point_cloud_poisson(pcd, depth=9)
    keep = ~low_density_mask(densities)
    remove_vertices_by_mask(mesh, ~keep)
    densities = densities[torch.from_numpy(keep).to(densities.device)]
    mesh.export(output_dir / "poisson_mesh.ply", mesh.vertex_colors)
    if texture_method == "nerf":
        tmesh = texturing.get_mesh_from_filename(str(output_dir / "poisson_mesh.ply"), target_num_faces=target_num_faces)
        texturing.export_textured_mesh(tmesh, renderer, output_dir,
                                       px_per_uv_triangle=px_per_uv_triangle if unwrap_method == "custom" else None,
                                       unwrap_method=unwrap_method, num_pixels_per_side=num_pixels_per_side)
    return mesh, densities
