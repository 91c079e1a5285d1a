"""Mesh extraction on the GPU (SURVEY.md section 8f row 2): drop-ins for the three functions of ``nerfstudio/utils/marching_cubes.py``
and for ``scripts/extract_mesh.py``.

The reference's ``scripts/extract_mesh.py:95-133`` hands ``lambda x: field.forward_geonetwork(x)[:, 0]`` to
``utils/marching_cubes.py`` (:15-341), which materialises 512^3-point lattices on the host, evaluates them in 100 000-point chunks,
copies each block's volume to the host for ``skimage.measure.marching_cubes`` and welds the blocks with ``trimesh``.  Here the lattice
is generated on the device (sdfb200_lattice_points), only the SDF head is evaluated (the fused kernel's sdf-only mode when
``precision != "fp32"``), the pyramid and masks stay torch ops on the device, and marching cubes is the library's two-pass kernel
(sdfb200_marching_cubes): the volume never goes to the host, only the mesh does.  ``Mesh`` stands in for the few ``trimesh.Trimesh``
members the reference uses.  ``write_ply`` and ``read_ply`` are the package's one PLY writer and reader, for every exporter.

Kept from the reference, quirks included: ``level`` is overwritten with 0 in both sliding variants, ``coarse_mask`` is permuted in
get_surface_sliding only, ``merge_vertices`` runs on the file path of get_surface_sliding and always in the contraction variant.
get_surface_occupancy also returns its mesh when ``return_mesh`` is set (the reference ignores the flag; it still writes the file).
"""
import ctypes as C
import importlib
from pathlib import Path
from typing import Callable, Sequence

import numpy as np
import torch

from . import _lib

EVAL_CHUNK = 100000          # points per sdf call, as the reference's evaluate() splits them
CROP_N = 512                 # lattice points per block side of the sliding variants

avg_pool_3d = torch.nn.AvgPool3d(2, stride=2)
upsample = torch.nn.Upsample(scale_factor=2, mode="nearest")
max_pool_3d = torch.nn.MaxPool3d(3, stride=1, padding=1)


def work_device() -> torch.device:
    """Where host-side mesh work (welding, normals) runs as torch ops: the GPU when there is one."""
    return torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu")


def sdf_fn(field, level: float = 0.0) -> Callable[[torch.Tensor], torch.Tensor]:
    """Drop-in for the ``sdf=`` callable of get_surface_sliding / get_surface_sliding_with_contraction: [N,3] -> [N]."""

    def fn(x: torch.Tensor) -> torch.Tensor:
        with torch.no_grad():
            pts = _lib.f32c(x.reshape(-1, 3))
            s = field._run(pts, None, None, 1, ("sdf",), apply_contraction=False)["sdf"]
        return s - level if level != 0.0 else s

    return fn


def lattice_points(bbox_min: Sequence[float], bbox_max: Sequence[float], resolution, start: int, n: int, device) -> torch.Tensor:
    """[n,3] slice of the 'ij'-ordered np.linspace lattice (marching_cubes.py:49-56)."""
    lib = _lib.load()
    res = (resolution,) * 3 if isinstance(resolution, int) else tuple(int(r) for r in resolution)
    out = torch.empty(n, 3, device=device, dtype=torch.float32)
    mn = (C.c_double * 3)(*[float(v) for v in bbox_min])
    mx = (C.c_double * 3)(*[float(v) for v in bbox_max])
    rs = (C.c_int32 * 3)(*res)
    _lib.check(lib.sdfb200_lattice_points(mn, mx, rs, int(start), int(n), _lib.ptr(out), _lib.stream_ptr()), "sdfb200_lattice_points")
    return out


def _lattice_values(fn, bbox_min, bbox_max, res, chunk: int, device) -> torch.Tensor:
    """``fn`` on the lattice of ``res`` = (rx, ry, rz) points, called on ``chunk`` points at a time -> float32 [rx * ry * rz]."""
    total = res[0] * res[1] * res[2]
    out = torch.empty(total, device=device, dtype=torch.float32)
    for start in range(0, total, chunk):
        n = min(chunk, total - start)
        out[start:start + n] = fn(lattice_points(bbox_min, bbox_max, res, start, n, device))
    return out


@torch.no_grad()
def evaluate_sdf_grid(field, resolution, bbox_min=(-1.0, -1.0, -1.0), bbox_max=(1.0, 1.0, 1.0), chunk: int = 1 << 22) -> torch.Tensor:
    """SDF on the dense lattice -> float32 tensor [rx, ry, rz] (what ``evaluate(points).reshape(N, N, N)`` is in the reference)."""
    res = (resolution,) * 3 if isinstance(resolution, int) else tuple(int(r) for r in resolution)
    return _lattice_values(sdf_fn(field), bbox_min, bbox_max, res, chunk, field.aabb.device).view(*res)


# ---------------------------------------------------------------------------------------------------------------------------------
# marching cubes, the mesh and its files
# ---------------------------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def marching_cubes(volume: torch.Tensor, level: float = 0.0, spacing=(1.0, 1.0, 1.0), mask: torch.Tensor = None):
    """skimage.measure.marching_cubes on a CUDA volume [nx, ny, nz] -> (verts [V,3] fp32, faces [F,3] int32, normals [V,3] fp32), device
    tensors.  ``verts`` are in lattice units times ``spacing``.  ``mask`` [nx, ny, nz] (bool / uint8): cube (i, j, k) is meshed when
    mask[i, j, k] is set.  Ordering, the face rule and the arithmetic: include/sdfb200.h.  Non-finite volumes raise ValueError."""
    _lib.require_cuda(volume.device, "marching_cubes")
    if volume.dim() != 3:
        raise ValueError(f"marching_cubes needs a 3-D volume, got shape {tuple(volume.shape)}")
    vol = _lib.f32c(volume)
    dev = vol.device
    empty = (torch.zeros(0, 3, device=dev), torch.zeros(0, 3, device=dev, dtype=torch.int32), torch.zeros(0, 3, device=dev))
    if min(vol.shape) < 2:
        return empty
    if not bool(torch.isfinite(vol).all()):
        raise ValueError("marching_cubes: the volume holds non-finite values")
    m = None
    if mask is not None:
        if tuple(mask.shape) != tuple(vol.shape):
            raise ValueError(f"mask shape {tuple(mask.shape)} != volume shape {tuple(vol.shape)}")
        m = mask.to(device=dev, dtype=torch.uint8).contiguous()
    lib = _lib.load()
    dims = (C.c_int64 * 3)(*vol.shape)
    org = (C.c_float * 3)(0.0, 0.0, 0.0)
    sp = (C.c_float * 3)(*[float(s) for s in spacing])
    lvl = float(level)
    U = vol.shape[0] * vol.shape[1]
    counts = torch.empty(2, U, device=dev, dtype=torch.int32)
    assert counts.numel() * 4 == lib.sdfb200_marching_cubes_workspace_bytes(dims)
    _lib.check(lib.sdfb200_marching_cubes(_lib.ptr(vol), dims, lvl, _lib.ptr(m), org, sp, None, _lib.ptr(counts), None, None, None,
                                          _lib.stream_ptr()), "sdfb200_marching_cubes")
    offsets = torch.zeros(2, U + 1, device=dev, dtype=torch.int64)
    torch.cumsum(counts, 1, out=offsets[:, 1:])
    n_verts, n_faces = (int(v) for v in offsets[:, -1].cpu())          # the one host read
    if n_faces == 0:
        return empty
    verts = torch.empty(n_verts, 3, device=dev)
    normals = torch.empty(n_verts, 3, device=dev)
    faces = torch.empty(n_faces, 3, device=dev, dtype=torch.int32)
    _lib.check(lib.sdfb200_marching_cubes(_lib.ptr(vol), dims, lvl, _lib.ptr(m), org, sp, _lib.ptr(offsets[:, :-1].contiguous()),
                                          _lib.ptr(counts), _lib.ptr(verts), _lib.ptr(normals), _lib.ptr(faces), _lib.stream_ptr()),
               "sdfb200_marching_cubes")
    return verts, faces, normals


class Mesh:
    """The members of ``trimesh.Trimesh`` that the reference's mesh extraction uses: numpy ``vertices`` [V,3] float64, ``faces`` [F,3]
    int64 and ``vertex_normals`` [V,3] float64."""

    def __init__(self, vertices, faces, vertex_normals=None):
        self.vertices = np.asarray(vertices, dtype=np.float64).reshape(-1, 3)
        self.faces = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
        self.vertex_normals = (np.zeros_like(self.vertices) if vertex_normals is None
                               else np.asarray(vertex_normals, dtype=np.float64).reshape(-1, 3))

    @staticmethod
    def concatenate(meshes):
        """trimesh.util.concatenate: one mesh, faces re-indexed."""
        meshes = list(meshes)
        if not meshes:
            return Mesh(np.zeros((0, 3)), np.zeros((0, 3), np.int64))
        starts = np.cumsum([0] + [len(m.vertices) for m in meshes[:-1]])
        return Mesh(np.concatenate([m.vertices for m in meshes]), np.concatenate([m.faces + s for m, s in zip(meshes, starts)]),
                    np.concatenate([m.vertex_normals for m in meshes]))

    @torch.no_grad()
    def merge_vertices(self, digits_vertex: int = 6):
        """Welds vertices equal after rounding to ``digits_vertex`` decimals, keeping each group's first vertex (and normal) in order of
        first occurrence, and re-indexes the faces.  torch ops, on the GPU when there is one."""
        if len(self.vertices) == 0:
            return
        dev = work_device()
        v = torch.from_numpy(self.vertices).to(dev)
        key = torch.round(v * (10.0 ** digits_vertex)).to(torch.int64)
        _, inverse = torch.unique(key, dim=0, return_inverse=True)
        n = v.shape[0]
        idx = torch.arange(n, device=dev)
        first = torch.full((int(inverse.max()) + 1,), n, device=dev, dtype=torch.int64).scatter_reduce_(0, inverse, idx, "amin")
        order = torch.argsort(first)
        rank = torch.empty_like(order)
        rank[order] = torch.arange(order.numel(), device=dev)
        keep = first[order]
        self.faces = rank[inverse][torch.from_numpy(self.faces).to(dev)].cpu().numpy()
        self.vertices = v[keep].cpu().numpy()
        self.vertex_normals = self.vertex_normals[keep.cpu().numpy()]

    def export(self, path, vertex_colors=None):
        """:func:`write_ply` of the mesh."""
        write_ply(path, self.vertices, self.faces, self.vertex_normals, vertex_colors)


def write_ply(path, vertices, faces, normals, vertex_colors=None):
    """binary little-endian PLY of numpy ``vertices`` [V,3], ``faces`` [F,3] and ``normals`` [V,3]: float x, y, z, nx, ny, nz per vertex,
    uchar-counted int lists per face.  With ``vertex_colors`` [V,3] in [0, 1], each vertex also carries uchar red, green, blue =
    floor(clip(c, 0, 1) * 255 + 0.5) (in fp32) and alpha = 255.  ``normals`` None leaves out nx, ny, nz; ``faces`` None leaves out the
    face element (a point cloud)."""
    props = [(n, "<f4") for n in ("x", "y", "z")]
    if normals is not None:
        props += [(n, "<f4") for n in ("nx", "ny", "nz")]
    if vertex_colors is not None:
        props += [(n, "u1") for n in ("red", "green", "blue", "alpha")]
    v = np.empty(len(vertices), dtype=props)
    for a, n in enumerate("xyz"):
        v[n] = vertices[:, a]
        if normals is not None:
            v["n" + n] = normals[:, a]
    if vertex_colors is not None:
        c = np.asarray(vertex_colors, dtype=np.float32).reshape(len(v), 3)
        q = np.floor(np.clip(c, 0.0, 1.0) * np.float32(255.0) + np.float32(0.5)).astype(np.uint8)
        v["red"], v["green"], v["blue"], v["alpha"] = q[:, 0], q[:, 1], q[:, 2], 255
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {len(v)}\n" + "".join(f"property {'float' if t == '<f4' else 'uchar'} {n}\n" for n, t in props))
    if faces is not None:
        f = np.empty(len(faces), dtype=[("n", "u1"), ("i", "<i4", (3,))])
        f["n"] = 3
        f["i"] = faces
        header += f"element face {len(f)}\nproperty list uchar int vertex_indices\n"
    with open(path, "wb") as fh:
        fh.write((header + "end_header\n").encode("ascii"))
        fh.write(v.tobytes())
        if faces is not None:
            fh.write(f.tobytes())


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "<i2", "int16": "<i2", "ushort": "<u2", "uint16": "<u2",
              "int": "<i4", "int32": "<i4", "uint": "<u4", "uint32": "<u4", "float": "<f4", "float32": "<f4", "double": "<f8",
              "float64": "<f8"}


def read_ply(filename):
    """(vertices [V,3] fp32, faces [F,3] int64, normals [V,3] fp32 or None) of a binary little-endian PLY of triangles, such as
    :func:`write_ply` writes.  A file without a face element (a point cloud) gives no faces."""
    with open(filename, "rb") as fh:
        data = fh.read()
    end = data.find(b"end_header\n")
    if not data.startswith(b"ply\n") or end < 0:
        raise ValueError(f"{filename}: not a PLY file")
    elements, fmt = [], None
    for line in data[:end].decode("ascii").splitlines()[1:]:
        tok = line.split()
        if not tok or tok[0] in ("comment", "obj_info"):
            continue
        if tok[0] == "format":
            fmt = tok[1]
        elif tok[0] == "element":
            elements.append((tok[1], int(tok[2]), []))
        elif tok[0] == "property":
            elements[-1][2].append(tok[1:])
    if fmt != "binary_little_endian":
        raise ValueError(f"{filename}: only binary_little_endian PLY is read, not {fmt}")
    pos, out = end + len(b"end_header\n"), {}
    for name, count, props in elements:
        if any(p[0] == "list" for p in props):
            if name != "face" or len(props) != 1:
                raise ValueError(f"{filename}: unsupported list element {name}")
            _, ct, it, _ = props[0]
            dt = np.dtype([("n", _PLY_TYPES[ct]), ("i", _PLY_TYPES[it], (3,))])
            rec = np.frombuffer(data, dtype=dt, count=count, offset=pos)
            if count and (rec["n"] != 3).any():
                raise ValueError(f"{filename}: only triangle faces are read")
            out[name] = rec["i"].astype(np.int64)
        else:
            dt = np.dtype([(p[1], _PLY_TYPES[p[0]]) for p in props])
            out[name] = np.frombuffer(data, dtype=dt, count=count, offset=pos)
        pos += count * dt.itemsize
    v = out["vertex"]
    vertices = np.stack([v[c] for c in "xyz"], axis=1).astype(np.float32)
    normals = np.stack([v[c] for c in ("nx", "ny", "nz")], axis=1).astype(np.float32) if "nx" in v.dtype.names else None
    return vertices, out.get("face", np.zeros((0, 3), np.int64)), normals


def import_optional(name: str, message: str):
    """The module ``name``, or an ImportError with ``message`` (what needed it and what to do instead) when it is not installed."""
    try:
        return importlib.import_module(name)
    except ImportError as e:
        raise ImportError(message) from e


def decimate(filename, target_num_faces: int, message: str):
    """pymeshlab's quadric edge collapse of the mesh file ``filename`` to ``target_num_faces`` faces: the MeshSet holding the result.
    ``message``: the ImportError's text when pymeshlab is not installed."""
    ms = import_optional("pymeshlab", message).MeshSet()
    ms.load_new_mesh(str(filename))
    ms.meshing_decimation_quadric_edge_collapse(targetfacenum=target_num_faces)
    return ms


def _block_mesh(volume, level, spacing, mask, offset) -> Mesh:
    verts, faces, normals = marching_cubes(volume, level=level, spacing=spacing, mask=mask)
    verts = verts.double() + torch.tensor(offset, dtype=torch.float64, device=verts.device)
    return Mesh(verts.cpu().numpy(), faces.cpu().numpy(), normals.cpu().numpy())


def _write(combined: Mesh, output_path, simplify_mesh: bool):
    filename = str(output_path)
    filename_simplify = str(output_path).replace(".ply", "-simplify.ply")
    combined.export(filename)
    if simplify_mesh:
        ms = decimate(filename, 2000000, f"simplify_mesh=True needs pymeshlab, which is not installed; the unsimplified mesh is at {filename}")
        ms.save_current_mesh(filename_simplify, save_face_color=False)


def _evaluate(fn, points):
    return torch.cat([fn(p) for p in torch.split(points, EVAL_CHUNK, dim=0)], dim=0)


def _outside(z, level) -> bool:
    """np.min(z) > level or np.max(z) < level, with one host read."""
    lo, hi = (float(v) for v in torch.stack(torch.aminmax(z)).cpu())
    return lo > level or hi < level


def _blocks(bounding_box_min, bounding_box_max, resolution, device):
    """The sliding variants' CROP_N^3-point blocks, i then j then k: (lower corner, upper corner, the block's lattice points [CROP_N^3, 3])
    for each, the corners from np.linspace over the box in float64."""
    N = resolution // CROP_N
    xs, ys, zs = [np.linspace(bounding_box_min[a], bounding_box_max[a], N + 1) for a in range(3)]
    for i in range(N):
        for j in range(N):
            for k in range(N):
                lo, hi = (xs[i], ys[j], zs[k]), (xs[i + 1], ys[j + 1], zs[k + 1])
                yield lo, hi, lattice_points(lo, hi, CROP_N, 0, CROP_N**3, device)


def _crossing_block_mesh(z, level, mask, lo, hi):
    """The mesh of block ``z`` [CROP_N]^3 between corners ``lo`` and ``hi``, or None unless ``level`` crosses both the values under
    ``mask`` (when there is one) and the whole block."""
    if mask is not None:
        valid_z = z[mask]
        if valid_z.shape[0] <= 0 or _outside(valid_z, level):
            return None
    if _outside(z, level):
        return None
    spacing = tuple((hi[a] - lo[a]) / (CROP_N - 1) for a in range(3))
    return _block_mesh(z, level, spacing, mask, lo)


@torch.no_grad()
def get_surface_sliding(
    sdf,
    resolution=512,
    bounding_box_min=(-1.0, -1.0, -1.0),
    bounding_box_max=(1.0, 1.0, 1.0),
    return_mesh=False,
    level=0,
    coarse_mask=None,
    output_path: Path = Path("test.ply"),
    simplify_mesh=True,
):
    """utils/marching_cubes.py:14-167: 512^3 blocks, each evaluated coarse to fine (64^3 -> 512^3) near the surface only."""
    assert resolution % 512 == 0
    dev = torch.device("cuda")
    if coarse_mask is not None:
        # grid_sample reads (z, y, x)
        coarse_mask = coarse_mask.permute(2, 1, 0)[None, None].to(dev).float()
    cropN = CROP_N
    level = 0
    meshes = []
    for lo, hi, points in _blocks(bounding_box_min, bounding_box_max, resolution, dev):
        points = points.reshape(cropN, cropN, cropN, 3).permute(3, 0, 1, 2)
        if coarse_mask is not None:
            current_mask = torch.nn.functional.grid_sample(coarse_mask, points.permute(1, 2, 3, 0)[None])
            current_mask = (current_mask > 0.0)[0, 0]
        else:
            current_mask = None

        points_pyramid = [points]
        for _ in range(3):
            points = avg_pool_3d(points[None])[0]
            points_pyramid.append(points)
        points_pyramid = points_pyramid[::-1]

        mask = None
        threshold = 2 * (hi[0] - lo[0]) / cropN * 8
        for pid, pts in enumerate(points_pyramid):
            coarse_N = pts.shape[-1]
            pts = pts.reshape(3, -1).permute(1, 0).contiguous()
            if mask is None:
                if coarse_mask is not None:
                    pts_sdf = torch.ones_like(pts[:, 1])
                    valid_mask = torch.nn.functional.grid_sample(coarse_mask, pts[None, None, None])[0, 0, 0, 0] > 0
                    if valid_mask.any():
                        pts_sdf[valid_mask] = _evaluate(sdf, pts[valid_mask].contiguous())
                else:
                    pts_sdf = _evaluate(sdf, pts)
            else:
                mask = mask.reshape(-1)
                pts_to_eval = pts[mask]
                if pts_to_eval.shape[0] > 0:
                    pts_sdf[mask] = _evaluate(sdf, pts_to_eval.contiguous())
            if pid < 3:
                mask = torch.abs(pts_sdf) < threshold
                mask = upsample(mask.reshape(coarse_N, coarse_N, coarse_N)[None, None].float()).bool()
                pts_sdf = upsample(pts_sdf.reshape(coarse_N, coarse_N, coarse_N)[None, None]).reshape(-1)
            threshold /= 2.0

        mesh = _crossing_block_mesh(pts_sdf.reshape(cropN, cropN, cropN), level, current_mask, lo, hi)
        if mesh is not None:
            meshes.append(mesh)

    combined = Mesh.concatenate(meshes)
    if return_mesh:
        return combined
    combined.merge_vertices(digits_vertex=6)
    _write(combined, output_path, simplify_mesh)


@torch.no_grad()
def get_surface_occupancy(
    occupancy_fn,
    resolution=512,
    bounding_box_min=(-1.0, -1.0, -1.0),
    bounding_box_max=(1.0, 1.0, 1.0),
    return_mesh=False,
    level=0.5,
    device=None,
    output_path: Path = Path("test.ply"),
):
    """utils/marching_cubes.py:170-215: one dense volume of resolution^3 points, meshed at ``level``."""
    grid_min, grid_max = bounding_box_min, bounding_box_max
    N = resolution
    dev = torch.device("cuda") if device is None else torch.device(device)
    z = _lattice_values(occupancy_fn, grid_min, grid_max, (N, N, N), EVAL_CHUNK, dev)
    if _outside(z, level):
        print("=================================================no surface skip")
        return None
    spacing = tuple((grid_max[a] - grid_min[a]) / (N - 1) for a in range(3))
    mesh = _block_mesh(z.reshape(N, N, N), level, spacing, None, tuple(float(v) for v in grid_min))
    Path(output_path).parent.mkdir(parents=True, exist_ok=True)
    mesh.export(str(output_path))
    return mesh if return_mesh else None


@torch.no_grad()
def get_surface_sliding_with_contraction(
    sdf,
    resolution=512,
    bounding_box_min=(-1.0, -1.0, -1.0),
    bounding_box_max=(1.0, 1.0, 1.0),
    return_mesh=False,
    level=0,
    coarse_mask=None,
    output_path: Path = Path("test.ply"),
    simplify_mesh=True,
    inv_contraction=None,
    max_range=32.0,
):
    """utils/marching_cubes.py:218-341: 512^3 blocks of the contracted space, evaluated where the visibility grid ``coarse_mask``
    ([1, 1, R, R, R], sampled at the points / 2) is set, 100 elsewhere, min-pooled across the mask border."""
    assert resolution % 512 == 0
    dev = torch.device("cuda")
    coarse_mask = coarse_mask.to(dev)
    cropN = CROP_N
    level = 0
    meshes = []
    for lo, hi, points in _blocks(bounding_box_min, bounding_box_max, resolution, dev):
        points = points.reshape(cropN, cropN, cropN, 3)
        current_mask = torch.nn.functional.grid_sample(coarse_mask, points[None] * 0.5)   # [-2, 2] -> [-1, 1]
        points = points.reshape(-1, 3)
        valid_mask = current_mask.reshape(-1) > 0
        pts_to_eval = points[valid_mask]
        pts_sdf = torch.ones_like(points[..., 0]) * 100.0
        if pts_to_eval.shape[0] > 0:
            pts_sdf[valid_mask.reshape(-1)] = _evaluate(sdf, pts_to_eval.contiguous())
        # min-pooling removes the artefacts of masked marching cubes
        min_sdf = max_pool_3d(pts_sdf.reshape(1, 1, cropN, cropN, cropN) * -1.0) * -1.0
        min_mask = (current_mask > 0.0).float()
        pts_sdf = pts_sdf.reshape(1, 1, cropN, cropN, cropN) * min_mask + min_sdf * (1.0 - min_mask)

        mesh = _crossing_block_mesh(pts_sdf.reshape(cropN, cropN, cropN), level, (current_mask > 0.0)[0, 0], lo, hi)
        if mesh is not None:
            meshes.append(mesh)

    combined = Mesh.concatenate(meshes)
    combined.merge_vertices(digits_vertex=6)
    if inv_contraction is not None:
        combined.vertices = inv_contraction(torch.from_numpy(combined.vertices)).numpy()
        combined.vertices = np.clip(combined.vertices, -max_range, max_range)
    if return_mesh:
        return combined
    _write(combined, output_path, simplify_mesh)


def extract_mesh(field, resolution: int = 1024, output_path: Path = Path("output.ply"), bounding_box_min=(-1.0, -1.0, -1.0),
                 bounding_box_max=(1.0, 1.0, 1.0), marching_cube_threshold: float = 0.0, is_occupancy: bool = False, coarse_mask=None,
                 inv_contraction=None, simplify_mesh: bool = False):
    """scripts/extract_mesh.py:62-133 (ExtractMesh.main) on a loaded field: the contraction variant when ``inv_contraction`` is given
    (with the visibility grid ``coarse_mask`` computed by the caller), the occupancy variant (unisurf) when ``is_occupancy``, the sliding
    variant otherwise.  As in the script, ``marching_cube_threshold`` only shifts the contraction variant."""
    assert str(output_path)[-4:] == ".ply"
    output_path = Path(output_path)
    output_path.parent.mkdir(parents=True, exist_ok=True)
    if inv_contraction is not None:
        assert resolution % 512 == 0
        return get_surface_sliding_with_contraction(sdf=sdf_fn(field, marching_cube_threshold), resolution=resolution,
                                                    bounding_box_min=bounding_box_min, bounding_box_max=bounding_box_max,
                                                    coarse_mask=coarse_mask, output_path=output_path, simplify_mesh=simplify_mesh,
                                                    inv_contraction=inv_contraction)
    if is_occupancy:
        f = sdf_fn(field)
        return get_surface_occupancy(occupancy_fn=lambda x: torch.sigmoid(10 * f(x)), resolution=resolution,
                                     bounding_box_min=bounding_box_min, bounding_box_max=bounding_box_max, level=0.5,
                                     device=field.aabb.device, output_path=output_path)
    assert resolution % 512 == 0
    return get_surface_sliding(sdf=sdf_fn(field), resolution=resolution, bounding_box_min=bounding_box_min,
                               bounding_box_max=bounding_box_max, coarse_mask=coarse_mask, output_path=output_path,
                               simplify_mesh=simplify_mesh)
