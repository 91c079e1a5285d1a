"""Textured-mesh export on the GPU: drop-ins for ``nerfstudio/exporter/texture_utils.py`` and for ``scripts/texture.py``.

The reference colours a mesh from the trained field by giving every texel of a UV texture a ray: the texel's face and barycentric
weights interpolate the face's vertices (the ray's midpoint) and vertex normals (its direction, reversed).  Its xatlas path finds each
texel's face by a brute-force ATen loop over chunks of 10 faces (texture_utils.py:263-301), ~30 kernels per chunk over every texel.
Here that search is one kernel (sdfb200_uv_rasterize), the custom grid unwrap another (sdfb200_uv_unwrap_grid), and the ray
construction a third (sdfb200_uv_texel_rays); faces and weights are bit-identical to the reference's.  The rays are rendered with the
renderer's large-chunk ``get_outputs_for_camera_ray_bundle`` and the OBJ / MTL / PNG files are written in bulk.

UV unwrapping itself stays with ``xatlas`` (``unwrap_method="xatlas"``, imported only when used), and decimation with ``pymeshlab``.
"""
import dataclasses
import math
import struct
import zlib
from pathlib import Path
from typing import Optional

import numpy as np
import torch

from . import _lib, meshing

MTL_LINES = ("# Generated with nerfstudio", "newmtl material_0", "Ka 1.000 1.000 1.000", "Kd 1.000 1.000 1.000", "Ks 0.000 0.000 0.000",
             "d 1.0", "illum 2", "Ns 1.00000000", "map_Kd material_0.png")


@dataclasses.dataclass
class Mesh:
    """nerfstudio.exporter.exporter_utils.Mesh: vertices [V,3] fp32, faces [F,3] int64, normals [V,3] fp32 (CPU tensors)."""

    vertices: torch.Tensor
    faces: torch.Tensor
    normals: torch.Tensor
    colors: Optional[torch.Tensor] = None


# ---------------------------------------------------------------------------------------------------------------------------------
# texels: face + barycentric weights, then rays
# ---------------------------------------------------------------------------------------------------------------------------------
def texel_linspaces(width: int, height: int, device):
    """The texel centres of get_texture_image (texture_utils.py:59-75) along u and v, built with torch.linspace as there."""
    px_w, px_h = 1.0 / width, 1.0 / height
    return torch.linspace(px_w / 2, 1 - px_w / 2, width, device=device), torch.linspace(px_h / 2, 1 - px_h / 2, height, device=device)


def uv_rasterize(texture_coordinates: torch.Tensor, num_pixels_per_side: int, num_faces_per_barycentric_chunk: int = 10):
    """Face [P] int32 and barycentric weights [P,3] of every texel of a square texture (P = num_pixels_per_side**2, row-major), as
    unwrap_mesh_with_xatlas' chunked search (texture_utils.py:263-301) finds them."""
    tc = _lib.f32c(texture_coordinates)
    _lib.require_cuda(tc.device, "texturing.uv_rasterize")
    if tc.dim() != 3 or tc.shape[1:] != (3, 2):
        raise ValueError(f"texture_coordinates must be [F, 3, 2], got {tuple(tc.shape)}")
    if num_faces_per_barycentric_chunk < 1:
        raise ValueError("num_faces_per_barycentric_chunk must be >= 1")
    n = int(num_pixels_per_side)
    lin_w, lin_h = texel_linspaces(n, n, tc.device)
    face = torch.empty(n * n, dtype=torch.int32, device=tc.device)
    bary = torch.empty(n * n, 3, dtype=torch.float32, device=tc.device)
    _lib.check(_lib.load().sdfb200_uv_rasterize(_lib.ptr(tc), tc.shape[0], int(num_faces_per_barycentric_chunk), _lib.ptr(lin_w), n,
                                                _lib.ptr(lin_h), n, _lib.ptr(face), _lib.ptr(bary), _lib.stream_ptr()), "sdfb200_uv_rasterize")
    return face, bary


def grid_layout(num_faces: int, px_per_uv_triangle: int):
    """Rectangles per row and column, and texture width and height, of the custom unwrap (texture_utils.py:100-108)."""
    num_squares = math.ceil(num_faces / 2)
    sw = math.ceil(math.sqrt(num_squares))
    sh = math.ceil(num_squares / sw)
    return sw, sh, sw * (px_per_uv_triangle + 3), sh * px_per_uv_triangle


def uv_unwrap_grid(num_faces: int, px_per_uv_triangle: int, device):
    """The custom unwrap (texture_utils.py:100-192): texture_coordinates [F,3,2], each texel's face [P] int32 (clamped to F - 1) and
    weights [P,3], and the texture's (height, width)."""
    ppt = int(px_per_uv_triangle)
    if num_faces < 1 or ppt < 1:
        raise ValueError("the custom unwrap needs at least one face and px_per_uv_triangle >= 1")
    sw, _, W, H = grid_layout(num_faces, ppt)
    # the first rectangle's two triangles, with the reference's fp32 ops (:119-149); the kernel adds each rectangle's offset
    lr_w, lr_h = (ppt + 3) / W, ppt / H
    lr = torch.tensor([lr_w, lr_h], device=device)
    px = torch.tensor([1.0 / W, 1.0 / H], device=device)
    scalar = (ppt - 1) / ppt
    upper_left = torch.tensor([[0, 0], [ppt / W, 0], [0, ppt / H]], device=device) * scalar + px / 2
    corner = torch.tensor([lr_w, lr_h], device=device)
    lower_right = (torch.tensor([[lr_w, lr_h], [3 * (1.0 / W), lr_h], [lr_w, 0]], device=device) - corner) * scalar + corner - px / 2
    square = torch.stack([upper_left, lower_right]).reshape(6, 2).contiguous()
    lin_w, lin_h = texel_linspaces(W, H, device)
    tc = torch.empty(num_faces, 3, 2, dtype=torch.float32, device=device)
    face = torch.empty(W * H, dtype=torch.int32, device=device)
    bary = torch.empty(W * H, 3, dtype=torch.float32, device=device)
    _lib.check(_lib.load().sdfb200_uv_unwrap_grid(_lib.ptr(square), _lib.ptr(lr), num_faces, sw, ppt, _lib.ptr(lin_w), W, _lib.ptr(lin_h), H,
                                                  _lib.ptr(tc), _lib.ptr(face), _lib.ptr(bary), _lib.stream_ptr()), "sdfb200_uv_unwrap_grid")
    return tc, face, bary, (H, W)


def uv_texel_rays(vertices, faces, vertex_normals, face, bary, raylen: Optional[torch.Tensor] = None):
    """Per texel, origin = the weights' blend of its face's vertices and direction = -normalize(the blend of its vertex normals)
    (texture_utils.py:194-205, :303-321).  With ``raylen`` (a device scalar) the origins move back by half of it and ``fars`` [P]
    = raylen is returned as well (:391-395); otherwise fars is None."""
    v, n = _lib.f32c(vertices), _lib.f32c(vertex_normals)
    f = faces.to(torch.int64).contiguous()
    P = face.shape[0]
    origins = torch.empty(P, 3, dtype=torch.float32, device=v.device)
    directions = torch.empty_like(origins)
    fars = None
    if raylen is not None:
        raylen = _lib.f32c(raylen.reshape(1))
        fars = torch.empty(P, dtype=torch.float32, device=v.device)
    _lib.check(_lib.load().sdfb200_uv_texel_rays(_lib.ptr(v), _lib.ptr(n), _lib.ptr(f), _lib.ptr(face.contiguous()), _lib.ptr(bary.contiguous()),
                                                 _lib.ptr(raylen), P, _lib.ptr(origins), _lib.ptr(directions), _lib.ptr(fars), _lib.stream_ptr()),
               "sdfb200_uv_texel_rays")
    return origins, directions, fars


# ---------------------------------------------------------------------------------------------------------------------------------
# drop-ins for texture_utils.py
# ---------------------------------------------------------------------------------------------------------------------------------
def _check_mesh(vertices, faces, vertex_normals):
    _lib.require_cuda(vertices.device, "texturing")
    if len(vertices) != len(vertex_normals):
        raise ValueError("Number of vertices and vertex normals must be equal")
    if faces.dim() != 2 or faces.shape[1] != 3 or len(faces) == 0:
        raise ValueError(f"faces must be a non-empty [F, 3] tensor, got {tuple(faces.shape)}")


def unwrap_mesh_per_uv_triangle(vertices, faces, vertex_normals, px_per_uv_triangle: int):
    """texture_utils.py:78-207: (texture_coordinates [F,3,2], origins [H,W,3], directions [H,W,3]) of the grid unwrap, two triangles per
    (px_per_uv_triangle + 3) x px_per_uv_triangle rectangle."""
    _check_mesh(vertices, faces, vertex_normals)
    tc, face, bary, hw = uv_unwrap_grid(len(faces), px_per_uv_triangle, vertices.device)
    origins, directions, _ = uv_texel_rays(vertices, faces, vertex_normals, face, bary)
    return tc, origins.view(*hw, 3), directions.view(*hw, 3)


def _import_xatlas():
    return meshing.import_optional("xatlas", 'unwrap_method="xatlas" needs the xatlas package, which is not installed; '
                                             'install it or use unwrap_method="custom"')


def _xatlas_texture_coordinates(vertices, faces, vertex_normals):
    _, indices, uvs = _import_xatlas().parametrize(vertices.cpu().numpy(), faces.cpu().numpy(), vertex_normals.cpu().numpy())
    return torch.from_numpy(np.asarray(uvs, dtype=np.float32)[indices]).to(vertices.device)


def rasterize_uv(texture_coordinates, vertices, faces, vertex_normals, num_pixels_per_side=1024, num_faces_per_barycentric_chunk=10):
    """The part of unwrap_mesh_with_xatlas after ``xatlas.parametrize`` (texture_utils.py:261-323), for meshes that already carry
    per-face-corner UVs ``texture_coordinates`` [F,3,2]: (texture_coordinates, origins [N,N,3], directions [N,N,3])."""
    _check_mesh(vertices, faces, vertex_normals)
    face, bary = uv_rasterize(texture_coordinates, num_pixels_per_side, num_faces_per_barycentric_chunk)
    origins, directions, _ = uv_texel_rays(vertices, faces, vertex_normals, face, bary)
    n = int(num_pixels_per_side)
    return texture_coordinates, origins.view(n, n, 3), directions.view(n, n, 3)


def unwrap_mesh_with_xatlas(vertices, faces, vertex_normals, num_pixels_per_side=1024, num_faces_per_barycentric_chunk=10):
    """texture_utils.py:210-323: UVs from ``xatlas.parametrize``, then :func:`rasterize_uv`."""
    _import_xatlas()
    _check_mesh(vertices, faces, vertex_normals)
    tc = _xatlas_texture_coordinates(vertices, faces, vertex_normals)
    return rasterize_uv(tc, vertices, faces, vertex_normals, num_pixels_per_side, num_faces_per_barycentric_chunk)


# ---------------------------------------------------------------------------------------------------------------------------------
# writers
# ---------------------------------------------------------------------------------------------------------------------------------
def obj_text(vertices: np.ndarray, faces: np.ndarray, vertex_normals: np.ndarray, texture_coordinates: np.ndarray) -> str:
    """mesh.obj as export_textured_mesh writes it (texture_utils.py:433-484): ``v``, then ``vt u 1-v`` per face corner, ``vn``, and
    ``f v/vt/vn`` with 1-based indices.  Numbers print as Python prints the fp32 values it formats (repr of their double)."""
    v = np.asarray(vertices, dtype=np.float32).reshape(-1, 3)
    tc = np.asarray(texture_coordinates, dtype=np.float32).reshape(-1, 2)
    vn = np.asarray(vertex_normals, dtype=np.float32).reshape(-1, 3)
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3) + 1
    vt = np.stack([tc[:, 0], np.float32(1.0) - tc[:, 1]], axis=1)   # 1.0 - uv[1] is an fp32 subtraction there
    fl = np.empty((len(f), 9), dtype=np.int64)
    fl[:, 0::3] = f
    fl[:, 1::3] = np.arange(1, 3 * len(f) + 1, dtype=np.int64).reshape(-1, 3)
    fl[:, 2::3] = f
    return ("# Generated with nerfstudio\nmtllib material_0.mtl\nusemtl material_0\n"
            + "v %r %r %r\n" * len(v) % tuple(v.astype(np.float64).ravel().tolist())
            + "vt %r %r\n" * len(vt) % tuple(vt.astype(np.float64).ravel().tolist())
            + "vn %r %r %r\n" * len(vn) % tuple(vn.astype(np.float64).ravel().tolist())
            + "f %d/%d/%d %d/%d/%d %d/%d/%d\n" * len(fl) % tuple(fl.ravel().tolist()))


def png_bytes(image: np.ndarray) -> bytes:
    """8-bit RGB PNG of an [H,W,3] float image in [0,1]: floor(clip(x, 0, 1) * 255 + 0.5), unfiltered rows, one zlib stream."""
    return png_bytes_u8(np.floor(np.clip(np.asarray(image, dtype=np.float32), 0.0, 1.0) * 255.0 + 0.5).astype(np.uint8))


def png_bytes_u8(img: np.ndarray) -> bytes:
    """8-bit RGB PNG of an [H,W,3] uint8 image: unfiltered rows, one zlib stream (zlib releases the GIL, so threads encode in parallel)."""
    img = np.ascontiguousarray(img)
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
        raise ValueError(f"expected an [H, W, 3] uint8 image, got {img.dtype} {img.shape}")
    h, w = img.shape[:2]
    raw = np.concatenate([np.zeros((h, 1), np.uint8), img.reshape(h, w * 3)], axis=1).tobytes()

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)

    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0)) + chunk(b"IDAT", zlib.compress(raw, 6))
            + chunk(b"IEND", b""))


def write_textured_mesh(output_dir, image, vertices, faces, vertex_normals, texture_coordinates):
    """material_0.png, material_0.mtl and mesh.obj in ``output_dir``."""
    output_dir = Path(output_dir)
    (output_dir / "material_0.png").write_bytes(png_bytes(image))
    (output_dir / "material_0.mtl").write_text("".join(line + "\n" for line in MTL_LINES), encoding="utf-8")
    (output_dir / "mesh.obj").write_text(obj_text(vertices, faces, vertex_normals, texture_coordinates), encoding="utf-8")


# ---------------------------------------------------------------------------------------------------------------------------------
# export
# ---------------------------------------------------------------------------------------------------------------------------------
def _mesh_tensors(mesh, device):
    normals = mesh.normals if hasattr(mesh, "normals") else mesh.vertex_normals       # exporter Mesh or meshing.Mesh
    return (torch.as_tensor(mesh.vertices).to(device, torch.float32), torch.as_tensor(mesh.faces).to(device, torch.int64),
            torch.as_tensor(normals).to(device, torch.float32))


def model_and_device(pipeline):
    """(model, device) of the reference's Pipeline (its ``.model`` and ``.device``) or of a renderer (itself, where its parameters are)."""
    model = getattr(pipeline, "model", pipeline)
    return model, (pipeline.device if hasattr(pipeline, "device") else next(model.parameters()).device)


def _ray_bundle_class(model):
    from .surface_model import SurfaceRenderer

    if isinstance(model, SurfaceRenderer):
        from .rays import RayBundle
    else:
        from nerfstudio.cameras.rays import RayBundle   # a reference model takes the reference's bundle
    return RayBundle


def export_textured_mesh(mesh, pipeline, output_dir: Path, px_per_uv_triangle: Optional[int] = None, unwrap_method: str = "xatlas",
                         raylen_method: str = "edge", num_pixels_per_side=1024):
    """texture_utils.py:326-496.  ``pipeline``: the reference's Pipeline (``.device``, ``.model.get_outputs_for_camera_ray_bundle``) or a
    SurfaceRenderer; ``mesh``: the reference's exporter Mesh, :class:`Mesh` or ``meshing.Mesh``.  Writes mesh.obj, material_0.mtl and
    material_0.png (8-bit, rounded to nearest) to ``output_dir``."""
    if unwrap_method not in ("xatlas", "custom"):
        raise ValueError(f"Unwrap method {unwrap_method} not supported.")
    if raylen_method not in ("edge", "none"):
        raise ValueError(f"Ray length method {raylen_method} not supported.")
    if unwrap_method == "custom" and px_per_uv_triangle is None:
        raise ValueError('unwrap_method="custom" needs px_per_uv_triangle')
    if unwrap_method == "xatlas":
        _import_xatlas()
    model, device = model_and_device(pipeline)
    vertices, faces, vertex_normals = _mesh_tensors(mesh, device)
    _check_mesh(vertices, faces, vertex_normals)
    if unwrap_method == "xatlas":
        tc = _xatlas_texture_coordinates(vertices, faces, vertex_normals)
        face, bary = uv_rasterize(tc, num_pixels_per_side)
        hw = (int(num_pixels_per_side),) * 2
    else:
        tc, face, bary, hw = uv_unwrap_grid(len(faces), px_per_uv_triangle, device)
    if raylen_method == "edge":
        fv = vertices[faces]
        raylen = 2.0 * torch.mean(torch.norm(fv[:, 1, :] - fv[:, 0, :], dim=-1)).float()
    else:
        raylen = torch.zeros((), dtype=torch.float32, device=device)
    origins, directions, fars = uv_texel_rays(vertices, faces, vertex_normals, face, bary, raylen)
    one = torch.ones(*hw, 1, device=device)
    bundle = _ray_bundle_class(model)(origins=origins.view(*hw, 3), directions=directions.view(*hw, 3), pixel_area=one,
                                      camera_indices=torch.zeros_like(one), directions_norm=one, nears=torch.zeros_like(one),
                                      fars=fars.view(*hw, 1))
    with torch.no_grad():
        outputs = model.get_outputs_for_camera_ray_bundle(bundle)
    write_textured_mesh(output_dir, outputs["rgb"].reshape(*hw, 3).cpu().numpy(), vertices.cpu().numpy(), faces.cpu().numpy(),
                        vertex_normals.cpu().numpy(), tc.cpu().numpy())


# ---------------------------------------------------------------------------------------------------------------------------------
# mesh input and scripts/texture.py
# ---------------------------------------------------------------------------------------------------------------------------------
def vertex_normals_area_weighted(vertices: torch.Tensor, faces: torch.Tensor) -> torch.Tensor:
    """Unit vertex normals: the sum of the adjacent faces' cross products (each twice the face's area), normalised."""
    fv = vertices[faces]
    fn = torch.cross(fv[:, 1] - fv[:, 0], fv[:, 2] - fv[:, 0], dim=-1)
    n = torch.zeros_like(vertices).index_add_(0, faces.reshape(-1), fn.repeat_interleave(3, dim=0))
    return torch.nn.functional.normalize(n, dim=-1)


def get_mesh_from_filename(filename, target_num_faces: Optional[int] = None) -> Mesh:
    """exporter_utils.py:75-83.  Reads a binary little-endian PLY; without normals in the file, area-weighted vertex normals are computed
    (on the GPU when there is one).  Decimating to ``target_num_faces`` needs pymeshlab, as in the reference."""
    vertices, faces, normals = meshing.read_ply(filename)
    if target_num_faces is not None and target_num_faces < len(faces):
        m = meshing.decimate(filename, target_num_faces,
                             f"reducing {filename} from {len(faces)} to {target_num_faces} faces needs pymeshlab, which is not installed; "
                             "pass target_num_faces=None to texture the mesh as it is").current_mesh()
        return Mesh(torch.from_numpy(m.vertex_matrix()).float(), torch.from_numpy(m.face_matrix()).long(),
                    torch.from_numpy(np.copy(m.vertex_normal_matrix())).float())
    v, f = torch.from_numpy(vertices), torch.from_numpy(faces)
    if normals is None:
        dev = meshing.work_device()
        n = vertex_normals_area_weighted(v.to(dev), f.to(dev)).cpu()
    else:
        n = torch.from_numpy(normals)
    return Mesh(v, f, n)


def texture_mesh(renderer, input_mesh_filename, output_dir, px_per_uv_triangle: int = 4, unwrap_method: str = "xatlas",
                 num_pixels_per_side: int = 2048, target_num_faces: Optional[int] = 50000):
    """scripts/texture.py:45-67 (TextureMesh.main) on a loaded renderer (a SurfaceRenderer or the reference's Pipeline)."""
    output_dir = Path(output_dir)
    output_dir.mkdir(parents=True, exist_ok=True)
    mesh = get_mesh_from_filename(str(input_mesh_filename), target_num_faces=target_num_faces)
    export_textured_mesh(mesh, renderer, px_per_uv_triangle=px_per_uv_triangle, output_dir=output_dir, unwrap_method=unwrap_method,
                         num_pixels_per_side=num_pixels_per_side)
