"""TSDF mesh export on the GPU: drop-ins for ``nerfstudio/exporter/tsdf_utils.py`` and for ``ns-export tsdf``
(``scripts/exporter.py:99-169``, ExportTSDFMesh).

The reference fuses depth images into a truncated signed distance volume with whole-batch ATen temporaries (a [batch, 4, N] fp32 camera
transform alone is 21.5 GB at 512^3 and a batch of 10) and then a masked gather and scatter per image; it meshes the volume with
skimage on the host and writes it with pymeshlab.  Here the fusion of every image is one kernel over the voxels
(sdfb200_tsdf_integrate: the images in order, the update in registers, the volume read and written once), the mesh comes from the
package's marching-cubes kernel (``meshing.marching_cubes``), and the PLY from ``meshing.write_ply``.  Depth and rgb images stay on
the device.

Kept from the reference, quirks included: the weight stored after an update is clamped to 1, colours mix with the old weight, voxels
behind a camera fuse through the mirrored point, the rendered depth is compared with the Euclidean distance to the camera, and
``export_tsdf_mesh``'s default ``resolution`` is a ``dataclasses.Field``, so omitting it raises the reference's ValueError.
``mask_images`` is not supported, as in the reference.
"""
from dataclasses import dataclass, field
from pathlib import Path
from typing import List, Optional, Tuple, Union

import torch

from . import _lib, meshing, texturing
from .cameras import Cameras


@dataclass
class TSDF:
    """tsdf_utils.TSDF: voxel_coords [3,X,Y,Z], values / weights [X,Y,Z], colors [X,Y,Z,3], voxel_size [3], origin [3]."""

    voxel_coords: torch.Tensor
    """Coordinates of each voxel in the TSDF."""
    values: torch.Tensor
    """TSDF values for each voxel."""
    weights: torch.Tensor
    """TSDF weights for each voxel."""
    colors: torch.Tensor
    """TSDF colors for each voxel."""
    voxel_size: torch.Tensor
    """Size of each voxel in the TSDF. [x, y, z] size."""
    origin: torch.Tensor
    """Origin of the TSDF [xmin, ymin, zmin]."""
    truncation_margin: float = 5.0
    """Margin for truncation."""

    def to(self, device: str):
        """Moves every tensor to ``device``."""
        for name in ("voxel_coords", "values", "weights", "colors", "voxel_size", "origin"):
            setattr(self, name, getattr(self, name).to(device))
        return self

    @property
    def device(self):
        """The device of voxel_coords."""
        return self.voxel_coords.device

    @property
    def truncation(self):
        """The truncation distance: voxel_size[0] * truncation_margin (a tensor on the TSDF's device)."""
        return self.voxel_size[0] * self.truncation_margin

    @staticmethod
    def from_aabb(aabb: torch.Tensor, volume_dims: torch.Tensor):
        """A TSDF over ``aabb`` [[xmin, ymin, zmin], [xmax, ymax, zmax]] with ``volume_dims`` [3] voxels, on the CPU as in the
        reference: values -1, weights and colors 0."""
        origin = aabb[0]
        voxel_size = (aabb[1] - aabb[0]) / volume_dims
        axes = [torch.arange(d) for d in volume_dims]
        grid = torch.stack(torch.meshgrid(axes, indexing="ij"), dim=0)
        voxel_coords = origin.view(3, 1, 1, 1) + grid * voxel_size.view(3, 1, 1, 1)
        dims = volume_dims.tolist()
        return TSDF(voxel_coords, -torch.ones(dims), torch.zeros(dims), torch.zeros(dims + [3]), voxel_size, origin)

    def get_mesh(self) -> texturing.Mesh:
        """Marching cubes at level 0 on values clamped to [-1, 1] (``meshing.marching_cubes``), without degenerate faces (faces with two
        equal vertex positions are removed; skimage's own rule for ``allow_degenerate=False`` is not pinned).  Colours are gathered at the
        vertices rounded half to even, as np.round rounds them, and the vertices are moved to world space.  Device tensors."""
        _lib.require_cuda(self.values.device, "tsdf.TSDF.get_mesh")
        verts, faces, normals = meshing.marching_cubes(self.values.clamp(-1, 1), level=0.0)
        faces = faces.long()
        p = verts[faces]
        keep = ~((p[:, 0] == p[:, 1]).all(-1) | (p[:, 1] == p[:, 2]).all(-1) | (p[:, 0] == p[:, 2]).all(-1))
        faces = faces[keep]
        idx = torch.round(verts).long()
        colors = self.colors[idx[:, 0], idx[:, 1], idx[:, 2]]
        vertices = self.origin.view(1, 3) + verts * self.voxel_size.view(1, 3)
        return texturing.Mesh(vertices=vertices, faces=faces, normals=normals, colors=colors)

    @classmethod
    def export_mesh(cls, mesh, filename: str):
        """Binary PLY with per-vertex normals and colours (uchar red, green, blue, alpha = 255; each channel
        floor(clip(c, 0, 1) * 255 + 0.5)), written by ``meshing.write_ply``."""
        colors = None if mesh.colors is None else mesh.colors.cpu().numpy()
        meshing.write_ply(filename, mesh.vertices.cpu().numpy(), mesh.faces.cpu().numpy(), mesh.normals.cpu().numpy(), colors)

    def integrate_tsdf(self, c2w: torch.Tensor, K: torch.Tensor, depth_images: torch.Tensor, color_images: Optional[torch.Tensor] = None,
                       mask_images: Optional[torch.Tensor] = None):
        """Fuses c2w [B,4,4], K [B,3,3], depth_images [B,1,H,W] and color_images [B,3,H,W] (or None: colours untouched), in order, with
        one sdfb200_tsdf_integrate call.  The result depends only on the order of the images, not on how they are split into calls.
        Images that are not fp32 are converted (``_lib.f32c``).  CUDA only."""
        if mask_images is not None:
            raise NotImplementedError("Mask images are not supported yet.")
        for name, t in (("the TSDF", self.voxel_coords), ("c2w", c2w), ("K", K), ("depth_images", depth_images),
                        ("color_images", color_images)):
            if t is not None and t.device.type != "cuda":
                raise RuntimeError(f"sdfstudio_b200.tsdf.TSDF.integrate_tsdf runs on CUDA only (there is no CPU path): {name} is on {t.device}")
        B = c2w.shape[0]
        if c2w.shape != (B, 4, 4) or K.shape != (B, 3, 3) or depth_images.dim() != 4 or depth_images.shape[:2] != (B, 1):
            raise ValueError(f"expected c2w [B,4,4], K [B,3,3] and depth_images [B,1,H,W], got {tuple(c2w.shape)}, {tuple(K.shape)} and "
                             f"{tuple(depth_images.shape)}")
        H, W = depth_images.shape[-2:]
        if color_images is not None and color_images.shape != (B, 3, H, W):
            raise ValueError(f"expected color_images [{B},3,{H},{W}], got {tuple(color_images.shape)}")
        n = self.values.numel()
        if self.voxel_coords.shape != (3, *self.values.shape) or self.weights.shape != self.values.shape or self.colors.shape != (*self.values.shape, 3):
            raise ValueError("voxel_coords [3,X,Y,Z], values and weights [X,Y,Z] and colors [X,Y,Z,3] disagree")
        for name in ("values", "weights", "colors"):
            setattr(self, name, _lib.f32c(getattr(self, name)))
        cams = pack_cams(c2w, K)
        coords = _lib.f32c(self.voxel_coords)
        depth = _lib.f32c(depth_images)
        color = None if color_images is None else _lib.f32c(color_images)
        trunc = _lib.f32c(torch.as_tensor(self.truncation, device=self.device).reshape(1))
        _lib.check(_lib.load().sdfb200_tsdf_integrate(_lib.ptr(coords), n, _lib.ptr(cams), B, _lib.ptr(depth), _lib.ptr(color), H, W,
                                                      _lib.ptr(trunc), _lib.ptr(self.values), _lib.ptr(self.weights), _lib.ptr(self.colors),
                                                      _lib.stream_ptr()), "sdfb200_tsdf_integrate")


def pack_cams(c2w: torch.Tensor, K: torch.Tensor) -> torch.Tensor:
    """[B,18] fp32 camera rows of sdfb200_tsdf_integrate: rows 0-2 of torch.inverse(c2w), then rows 0-1 of K.  Each camera is inverted
    on its own, so that its inverse, and hence the fused volume, does not depend on how the images are batched (the batched inverse
    may take another algorithm).  ``inv_ex`` is torch.inverse without its error check, which would read back to the host per camera."""
    inv = torch.cat([torch.linalg.inv_ex(c2w[i:i + 1]).inverse for i in range(c2w.shape[0])]) if c2w.shape[0] else c2w
    return torch.cat([inv[:, :3, :].reshape(-1, 12), K[:, :2, :].reshape(-1, 6)], dim=1).float().contiguous()


# ---------------------------------------------------------------------------------------------------------------------------------
# export
# ---------------------------------------------------------------------------------------------------------------------------------
def _hw(cameras, i):
    if isinstance(cameras, Cameras):
        return cameras.height, cameras.width
    return int(cameras.height.view(-1)[i]), int(cameras.width.view(-1)[i])


@torch.no_grad()
def render_images(model, cameras, rgb_output_name: str, depth_output_name: str, device, rendered_resolution_scaling_factor: float = 1.0):
    """exporter_utils.render_trajectory (:212-259) with the images kept on the device: the cameras are rescaled in place, then each is
    rendered through ``model.get_outputs_for_camera_ray_bundle``.  Returns colour [C,3,H,W] and depth [C,1,H,W].  ``cameras``: the
    package's :class:`Cameras` or the reference's (rendered without distortion)."""
    cameras.rescale_output_resolution(rendered_resolution_scaling_factor)
    rgbs, depths = [], []
    for i in range(len(cameras)):
        if isinstance(cameras, Cameras):
            bundle = cameras.generate_rays(i)
        else:
            bundle = cameras.generate_rays(camera_indices=i, disable_distortion=True).to(device)
        outputs = model.get_outputs_for_camera_ray_bundle(bundle)
        for name in (rgb_output_name, depth_output_name):
            if name not in outputs:
                raise ValueError(f"Could not find {name} in the model outputs; choose one of: {list(outputs.keys())}")
        H, W = _hw(cameras, i)
        rgbs.append(outputs[rgb_output_name].reshape(H, W, -1))
        depths.append(outputs[depth_output_name].reshape(H, W, -1))
    return torch.stack(rgbs).permute(0, 3, 1, 2), torch.stack(depths).permute(0, 3, 1, 2)


def volume_dims_of(resolution) -> torch.Tensor:
    if isinstance(resolution, int):
        return torch.tensor([resolution] * 3)
    if isinstance(resolution, List):
        return torch.tensor(resolution)
    raise ValueError("Resolution must be an int or a list.")


def _export(model, device, cameras, aabb, output_dir, downscale_factor, depth_output_name, rgb_output_name, volume_dims):
    tsdf = TSDF.from_aabb(aabb, volume_dims=volume_dims).to(device)
    color_images, depth_images = render_images(model, cameras, rgb_output_name, depth_output_name, device, 1.0 / downscale_factor)
    c2w = cameras.camera_to_worlds.to(device)
    c2w = torch.cat([c2w, torch.zeros(c2w.shape[0], 1, 4, device=device)], dim=1)
    c2w[:, 3, 3] = 1
    K = cameras.get_intrinsics_matrices().to(device)
    tsdf.integrate_tsdf(c2w, K, depth_images, color_images=color_images)
    mesh = tsdf.get_mesh()
    TSDF.export_mesh(mesh, filename=str(Path(output_dir) / "tsdf_mesh.ply"))


def export_tsdf_mesh(
    pipeline,
    output_dir: Path,
    downscale_factor: int = 2,
    depth_output_name: str = "depth",
    rgb_output_name: str = "rgb",
    resolution: Union[int, List[int]] = field(default_factory=lambda: [256, 256, 256]),
    batch_size: int = 10,
    use_bounding_box: bool = True,
    bounding_box_min: Tuple[float, float, float] = (-1.0, -1.0, -1.0),
    bounding_box_max: Tuple[float, float, float] = (1.0, 1.0, 1.0),
):
    """tsdf_utils.export_tsdf_mesh (:273-351) on the reference's Pipeline: renders the datamanager's training cameras at
    1 / downscale_factor, fuses every image in one call (equal to the reference's batches of ``batch_size``, which is therefore only
    accepted), and writes ``output_dir / "tsdf_mesh.ply"``.  As in the reference, ``resolution`` must be an int or a list: the default
    (a dataclasses.Field) and tuples raise ValueError."""
    device = pipeline.device
    dataparser_outputs = pipeline.datamanager.train_dataset._dataparser_outputs  # pylint: disable=protected-access
    aabb = dataparser_outputs.scene_box.aabb if not use_bounding_box else torch.tensor([bounding_box_min, bounding_box_max])
    volume_dims = volume_dims_of(resolution)
    _export(pipeline.model, device, dataparser_outputs.cameras, aabb, output_dir, downscale_factor, depth_output_name, rgb_output_name,
            volume_dims)


def tsdf_mesh(renderer, cameras: Cameras, output_dir, downscale_factor: int = 2, depth_output_name: str = "depth", rgb_output_name: str = "rgb",
              resolution: Union[int, List[int]] = 128, bounding_box_min: Tuple[float, float, float] = (-1.0, -1.0, -1.0),
              bounding_box_max: Tuple[float, float, float] = (1.0, 1.0, 1.0), texture_method: str = "nerf", px_per_uv_triangle: int = 4,
              unwrap_method: str = "xatlas", num_pixels_per_side: int = 2048, target_num_faces: Optional[int] = 50000):
    """ExportTSDFMesh.main (scripts/exporter.py:144-169) on a renderer (a SurfaceRenderer) and the package's :class:`Cameras` (rescaled in
    place), over the bounding box: writes tsdf_mesh.ply to ``output_dir`` and, with ``texture_method="nerf"``, textures it with
    ``texturing.export_textured_mesh`` (mesh.obj, material_0.mtl, material_0.png).  Reducing the mesh to ``target_num_faces`` needs
    pymeshlab, as in ``texturing.texture_mesh``."""
    if texture_method not in ("tsdf", "nerf"):
        raise ValueError(f"texture_method must be 'tsdf' or 'nerf', not {texture_method!r}")
    output_dir = Path(output_dir)
    output_dir.mkdir(parents=True, exist_ok=True)
    model, device = texturing.model_and_device(renderer)
    _export(model, device, cameras, torch.tensor([bounding_box_min, bounding_box_max]), output_dir, downscale_factor, depth_output_name,
            rgb_output_name, volume_dims_of(resolution))
    if texture_method == "nerf":
        mesh = texturing.get_mesh_from_filename(str(output_dir / "tsdf_mesh.ply"), target_num_faces=target_num_faces)
        texturing.export_textured_mesh(mesh, renderer, output_dir, px_per_uv_triangle=px_per_uv_triangle if unwrap_method == "custom" else None,
                                       unwrap_method=unwrap_method, num_pixels_per_side=num_pixels_per_side)
