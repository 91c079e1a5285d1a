"""Point-cloud export on the GPU: drop-ins for ``exporter_utils.generate_point_cloud`` (nerfstudio/exporter/exporter_utils.py:86-205)
and for ``ns-export pointcloud`` (``scripts/exporter.py:42-96``, ExportPointCloud).

The reference renders training rays, keeps the points inside a box, and hands the cloud to open3d on the host, whose
``remove_statistical_outlier`` and ``estimate_normals`` each run a CPU KD-tree k-nearest-neighbour search over every point.  Here the
cloud stays on the device: the neighbours come from an exact grid search (sdfb200_knn), the normals from a PCA over them
(sdfb200_point_normals), and the PLY from ``meshing.write_ply``.

open3d is not a dependency, so its rules are restated, not pinned; each function lists the ones it follows.
"""
import math
from dataclasses import dataclass
from pathlib import Path
from typing import Optional, Tuple

import torch

from . import _lib, meshing, texturing

MAX_K = 32
CELLS_PER_POINT = 4
"""The grid of sdfb200_knn has the finest power-of-two cell size with at most CELLS_PER_POINT * N cells over the cloud's box (DESIGN
section 3, "Point clouds")."""


def _grid(box, log2_cell: int):
    """(cell_min [3], dims [3]) as Python ints: cell_min = floor(box_min 2^-e), dims = floor(box_max 2^-e) - cell_min + 1 (exact)."""
    cmin = [math.floor(math.ldexp(float(box[a]), -log2_cell)) for a in range(3)]
    dims = [math.floor(math.ldexp(float(box[a + 3]), -log2_cell)) - cmin[a] + 1 for a in range(3)]
    return cmin, dims


def cell_log2(n: int, box) -> int:
    """The grid policy: the smallest e (the finest cell 2^e) such that the box holds at most max(1, CELLS_PER_POINT * n) cells.  On a
    cloud that lies on a surface most cells are empty and the occupied ones hold more points than the average; DESIGN section 3 reports
    what this gives on the benchmark's clouds."""
    budget = max(1, CELLS_PER_POINT * n)
    extent = max(float(box[a + 3]) - float(box[a]) for a in range(3))
    e = math.frexp(extent)[1] + 1 if extent > 0 else 0
    if extent == 0:
        return e
    while e > -150:
        cells = math.prod(_grid(box, e - 1)[1])
        if cells > budget:
            break
        e -= 1
    return e


def nearest_neighbours(points: torch.Tensor, k: int, mean_distances: bool = True, neighbours: bool = True):
    """Exact k nearest neighbours of every point of ``points`` [N,3] (CUDA; converted to fp32) among all of them, each point included at
    distance 0, by sdfb200_knn.  Returns (mean distances [N] fp64 or None, neighbour indices [N,k] int32 or None): the neighbours in
    ascending (squared distance, index) order, the mean the average of the square roots of the k_eff = min(k, N) smallest squared
    distances, added in ascending order.  The distances are computed in double from the fp32 coordinates; include/sdfb200.h has the
    op order.  Entries k_eff..k-1 of a list (only when N < k) are -1.

    The cloud's box is read back to the host once (it sets the grid); points are bucketed with a stable sort by cell.  A non-finite
    point raises ValueError before the search runs; ``k`` must lie in [1, 32]."""
    if not 1 <= k <= MAX_K:
        raise ValueError(f"k must lie in [1, {MAX_K}], got {k}")
    if not (mean_distances or neighbours):
        raise ValueError("ask for the mean distances, the neighbours or both")
    _lib.require_cuda(points.device, "pointcloud.nearest_neighbours")
    pts = _lib.f32c(points)
    if pts.dim() != 2 or pts.shape[1] != 3:
        raise ValueError(f"expected points [N,3], got {tuple(pts.shape)}")
    n = pts.shape[0]
    dev = pts.device
    mean = torch.empty(n, dtype=torch.float64, device=dev) if mean_distances else None
    idx = torch.empty(n, k, dtype=torch.int32, device=dev) if neighbours else None
    if n == 0:
        return mean, idx
    if n >= 2**31:
        raise ValueError(f"at most 2^31 - 1 points, got {n}")
    box = torch.cat([pts.amin(0), pts.amax(0)]).cpu()   # amin / amax propagate NaN
    if not torch.isfinite(box).all():
        raise ValueError("the point cloud holds a non-finite coordinate")
    e = cell_log2(n, box)
    cmin, dims = _grid(box, e)
    cells = math.prod(dims)
    c = (torch.floor(pts.double() * math.ldexp(1.0, -e)) - torch.tensor(cmin, dtype=torch.float64, device=dev)).long()
    key = (c[:, 2] * dims[1] + c[:, 1]) * dims[0] + c[:, 0]
    skey, order = torch.sort(key, stable=True)
    cell_start = torch.zeros(cells + 1, dtype=torch.int32, device=dev)
    cell_start[1:] = torch.bincount(skey, minlength=cells).cumsum(0)
    sorted_pts = pts[order].contiguous()
    host_box = (_lib.C.c_float * 6)(*box.tolist())
    _lib.check(_lib.load().sdfb200_knn(_lib.ptr(sorted_pts), _lib.ptr(order.int()), n, _lib.ptr(cell_start), host_box, e, k, _lib.ptr(mean),
                                       _lib.ptr(idx), _lib.stream_ptr()), "sdfb200_knn")
    return mean, idx


def remove_statistical_outlier(points: torch.Tensor, nb_neighbors: int, std_ratio: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """open3d's ``PointCloud::RemoveStatisticalOutliers`` (open3d >= 0.16) on a CUDA cloud [N,3].  Returns (the kept indices [M] int64 in
    ascending order, the mean distances [N] fp64 of :func:`nearest_neighbours` with k = ``nb_neighbors``).  Restated, not pinned (open3d is absent):

    - the mean distance of a point averages its distances to its k_eff = min(nb_neighbors, N) nearest points, itself included;
    - a point is valid when its mean distance is > 0, so a point whose k_eff neighbours all coincide with it is dropped;
    - the cloud mean is taken over the valid points, and the standard deviation over them with Bessel's correction (n - 1);
    - threshold = mean + std_ratio * std; a point is kept when it is valid and its mean distance is strictly below the threshold;
    - an empty cloud, or one with no valid point, keeps nothing; with one valid point the deviation is 0 / 0 and nothing is kept.

    ``nb_neighbors < 1`` or ``std_ratio <= 0`` raise ValueError, as does ``nb_neighbors > 32`` (the kernel's limit).  The reductions
    are deterministic torch sums in double: they round differently from open3d's sequential ``std::accumulate``, so a point whose mean
    distance lies within a few ulps of the threshold may be decided the other way."""
    if nb_neighbors < 1 or std_ratio <= 0:
        raise ValueError(f"Illegal input parameters, number of neighbors and standard deviation ratio must be positive "
                         f"(nb_neighbors={nb_neighbors}, std_ratio={std_ratio})")
    _lib.require_cuda(points.device, "pointcloud.remove_statistical_outlier")
    if points.shape[0] == 0:
        return torch.empty(0, dtype=torch.int64, device=points.device), torch.empty(0, dtype=torch.float64, device=points.device)
    mean, _ = nearest_neighbours(points, nb_neighbors, neighbours=False)
    valid = mean > 0
    count = valid.sum()
    cloud_mean = torch.where(valid, mean, 0.0).sum() / count
    sq_sum = torch.where(valid, (mean - cloud_mean) * (mean - cloud_mean), 0.0).sum()
    threshold = cloud_mean + std_ratio * torch.sqrt(sq_sum / (count - 1))
    return torch.nonzero(valid & (mean < threshold)).squeeze(1), mean


def estimate_normals(points: torch.Tensor, knn: int = 30) -> torch.Tensor:
    """open3d's ``estimate_normals()`` with its default ``KDTreeSearchParamKNN(30)`` on a CUDA cloud [N,3], without an orientation step:
    the :func:`nearest_neighbours` lists, then the eigenvector of the smallest eigenvalue of each list's covariance (sdfb200_point_normals).  Returns
    [N,3] fp32.  Not pinned (open3d is absent): the sign (the fp32 component of largest magnitude is positive, the first axis on ties) and a
    zero covariance, which gives (0, 0, 1).

    Accuracy: the covariance is open3d's cumulant form in double, and the Jacobi solver is backward stable, so the vector is an exact
    eigenvector of a matrix within c u ||C|| of the computed covariance C (u = 2^-53, c a small constant).  By the Davis-Kahan theorem
    its angle to the true one is at most c u ||C|| / gap, gap being the distance from the smallest eigenvalue to the next; writing it as
    fp32 adds at most 2^-24 per component."""
    return _normals(points, knn)


def _normals(points: torch.Tensor, k: int) -> torch.Tensor:
    _, idx = nearest_neighbours(points, k, mean_distances=False)
    pts = _lib.f32c(points)
    normals = torch.empty_like(pts)
    _lib.check(_lib.load().sdfb200_point_normals(_lib.ptr(pts), pts.shape[0], _lib.ptr(idx), k, _lib.ptr(normals), _lib.stream_ptr()),
               "sdfb200_point_normals")
    return normals


@dataclass
class PointCloud:
    """The cloud of :func:`generate_point_cloud`: fp32 device tensors."""

    points: torch.Tensor
    """[N,3] positions."""
    colors: torch.Tensor
    """[N,3] rgb in [0, 1]."""
    normals: Optional[torch.Tensor] = None
    """[N,3] normals, or None."""

    def __len__(self):
        return self.points.shape[0]

    def export(self, path) -> None:
        """Binary little-endian PLY of the vertices (float x y z, float nx ny nz when there are normals, uchar red green blue alpha with
        each channel floor(clip(c, 0, 1) * 255 + 0.5) and alpha 255) and no face element, by ``meshing.write_ply``."""
        normals = None if self.normals is None else self.normals.float().cpu().numpy()
        meshing.write_ply(str(path), self.points.float().cpu().numpy(), None, normals, self.colors.float().cpu().numpy())


def generate_point_cloud(
    pipeline,
    num_points: int = 1000000,
    remove_outliers: bool = True,
    estimate_normals: bool = False,
    rgb_output_name: str = "rgb",
    depth_output_name: str = "depth",
    normal_output_name: Optional[str] = None,
    use_bounding_box: bool = True,
    bounding_box_min: Tuple[float, float, float] = (-1.0, -1.0, -1.0),
    bounding_box_max: Tuple[float, float, float] = (1.0, 1.0, 1.0),
    std_ratio: float = 10.0,
) -> PointCloud:
    """exporter_utils.generate_point_cloud (:86-205) on the reference's Pipeline, with the cloud kept on the device.  Batches come from
    ``pipeline.datamanager.next_train(0)`` and ``pipeline.model(ray_bundle)`` under no_grad, until the points kept reach ``num_points``
    (at least one batch; the last batch is not truncated).  A point is origin + direction * depth with the model's depth; with
    ``use_bounding_box`` it is kept when strictly inside the box (which must have min < max, as the reference asserts).  Then outliers
    are removed (:func:`remove_statistical_outlier` with 20 neighbours) and either normals are estimated (:func:`estimate_normals`) or
    the ``normal_output_name`` output is masked by the kept indices.  A missing output, or ``estimate_normals`` together with
    ``normal_output_name`` (checked where the reference checks it, after the cloud is cleaned), raises ValueError with the reference's
    message instead of exiting."""
    points, rgbs, normals = [], [], []
    kept = 0
    while True:
        with torch.no_grad():
            ray_bundle, _ = pipeline.datamanager.next_train(0)
            outputs = pipeline.model(ray_bundle)
        for name, flag in ((rgb_output_name, "rgb_output_name"), (depth_output_name, "depth_output_name"),
                           (normal_output_name, "normal_output_name")):
            if name is not None and name not in outputs:
                raise ValueError(f"Could not find {name} in the model outputs. Please set --{flag} to one of: {outputs.keys()}")
        rgb = outputs[rgb_output_name]
        depth = outputs[depth_output_name]
        normal = outputs[normal_output_name] if normal_output_name is not None else None
        point = ray_bundle.origins + ray_bundle.directions * depth
        if use_bounding_box:
            comp_l = torch.tensor(bounding_box_min, device=point.device)
            comp_m = torch.tensor(bounding_box_max, device=point.device)
            assert torch.all(comp_l < comp_m), f"Bounding box min {bounding_box_min} must be smaller than max {bounding_box_max}"
            mask = torch.all(torch.concat([point > comp_l, point < comp_m], dim=-1), dim=-1)
            point = point[mask]
            rgb = rgb[mask]
            if normal is not None:
                normal = normal[mask]
        points.append(point)
        rgbs.append(rgb)
        if normal is not None:
            normals.append(normal)
        kept += point.shape[0]
        if kept >= num_points:
            break
    cloud = PointCloud(torch.cat(points, dim=0).float(), torch.cat(rgbs, dim=0).float())
    ind = None
    if remove_outliers:
        ind, _ = remove_statistical_outlier(cloud.points, nb_neighbors=20, std_ratio=std_ratio)
        cloud.points, cloud.colors = cloud.points[ind], cloud.colors[ind]
    if estimate_normals:
        if normal_output_name is not None:
            raise ValueError("Cannot estimate normals and use normal_output_name at the same time")
        cloud.normals = _normals(cloud.points, 30)
    elif normal_output_name is not None:
        n = torch.cat(normals, dim=0)
        if ind is not None:
            n = n[ind]
        cloud.normals = n.float()
    return cloud


class _PixelRays:
    """A stand-in for the reference's datamanager over the package's :class:`Cameras`: ``next_train`` draws ``num_rays_per_batch``
    pixels as the reference's PixelSampler does (``floor(rand(n, 3) * [C, H, W]).long()``, from a seeded device generator) and returns
    the rays through their centres."""

    def __init__(self, cameras, num_rays_per_batch: int, seed: int):
        self.cameras = cameras
        self.num_rays_per_batch = num_rays_per_batch
        self.generator = torch.Generator(device=cameras.device).manual_seed(seed)

    def next_train(self, step: int):
        cams, dev = self.cameras, self.cameras.device
        scale = torch.tensor([len(cams), cams.height, cams.width], device=dev)
        indices = torch.floor(torch.rand((self.num_rays_per_batch, 3), generator=self.generator, device=dev) * scale).long()
        coords = indices[:, 1:].float() + 0.5
        return cams.generate_rays(indices[:, 0], coords), {"indices": indices}


class _RendererPipeline:
    def __init__(self, model, datamanager):
        self.model, self.datamanager = model, datamanager


def point_cloud(renderer, cameras, output_dir, num_points: int = 1000000, remove_outliers: bool = True, estimate_normals: bool = False,
                depth_output_name: str = "depth", rgb_output_name: str = "rgb", use_bounding_box: bool = True,
                bounding_box_min: Tuple[float, float, float] = (-1, -1, -1), bounding_box_max: Tuple[float, float, float] = (1, 1, 1),
                num_rays_per_batch: int = 32768, std_ratio: float = 10.0, seed: int = 0) -> PointCloud:
    """ExportPointCloud.main (scripts/exporter.py:68-96) on a renderer (a SurfaceRenderer) and the package's :class:`Cameras`: writes
    ``output_dir / "point_cloud.ply"`` and returns the cloud.  Rays are drawn by a seeded restatement of the reference's PixelSampler
    (``seed``).  A reference Pipeline passed as ``renderer`` uses its own datamanager, with its pixel sampler set to
    ``num_rays_per_batch`` as the reference does, and ``cameras`` is ignored."""
    output_dir = Path(output_dir)
    output_dir.mkdir(parents=True, exist_ok=True)
    if hasattr(renderer, "datamanager"):
        renderer.datamanager.train_pixel_sampler.num_rays_per_batch = num_rays_per_batch
        pipeline = renderer
    else:
        model, _ = texturing.model_and_device(renderer)
        pipeline = _RendererPipeline(model, _PixelRays(cameras, num_rays_per_batch, seed))
    cloud = generate_point_cloud(pipeline, num_points=num_points, remove_outliers=remove_outliers, estimate_normals=estimate_normals,
                                 rgb_output_name=rgb_output_name, depth_output_name=depth_output_name, normal_output_name=None,
                                 use_bounding_box=use_bounding_box, bounding_box_min=bounding_box_min,
                                 bounding_box_max=bounding_box_max, std_ratio=std_ratio)
    cloud.export(output_dir / "point_cloud.ply")
    return cloud
