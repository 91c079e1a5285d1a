"""Restatements for the point-cloud exporter (sdfstudio_b200/pointcloud.py):

(a) ``reference_flow``: exporter_utils.generate_point_cloud (nerfstudio/exporter/exporter_utils.py:86-205) on torch-CPU, up to the
    calls into open3d, which are handed to the given callables.  It returns what the reference hands to open3d.
(b) ``knn`` and ``covariances``: the kNN, mean distances and covariances in numpy float64, in sdfb200_knn's and
    sdfb200_point_normals's documented op order and tie rule (include/sdfb200.h), by brute force.
(c) ``statistical_outliers``: open3d's RemoveStatisticalOutliers rules (open3d >= 0.16), restated in numpy.

``FakePipeline`` is the seeded pipeline that both the golden bundle and the GPU tests run: its datamanager draws rays around an
analytic sphere (some batches miss it entirely) and its model returns the sphere's rgb, depth and normal.
"""
from typing import Callable, Optional

import numpy as np
import torch

SPHERE_CENTRE, SPHERE_RADIUS = (0.1, -0.05, 0.0), 0.55


class SimpleBundle:
    def __init__(self, origins, directions):
        self.origins, self.directions = origins, directions


class FakeDataManager:
    """``next_train(step)`` returns (bundle, {}) of ``n`` seeded rays from a sphere of radius 2.2 towards the origin; every
    ``miss_every``-th call (when > 0) aims every ray away from the scene, so that the batch keeps no point."""

    def __init__(self, n: int, seed: int, bundle_cls=SimpleBundle, device="cpu", miss_every: int = 0):
        self.n, self.bundle_cls, self.device, self.miss_every = n, bundle_cls, device, miss_every
        self.generator = torch.Generator().manual_seed(seed)
        self.calls = 0

    def next_train(self, step: int):
        self.calls += 1
        g = self.generator
        o = torch.randn(self.n, 3, generator=g)
        o = 2.2 * o / o.norm(dim=-1, keepdim=True)
        d = -o + 0.45 * torch.randn(self.n, 3, generator=g)
        if self.miss_every and self.calls % self.miss_every == 0:
            d = o.clone()
        d = d / d.norm(dim=-1, keepdim=True)
        return self.bundle_cls(origins=o.to(self.device), directions=d.to(self.device)), {}


class FakeModel:
    """rgb = 0.5 + 0.5 n, depth = the distance to the sphere along the ray (0 on a miss, so the point is the ray's origin, outside
    the unit box), normal = n, on the bundle's device.  ``outputs`` limits the names returned."""

    def __init__(self, outputs=("rgb", "depth", "normal")):
        self.outputs = outputs

    def __call__(self, bundle):
        o, d = bundle.origins.cpu().float(), bundle.directions.cpu().float()
        c = torch.tensor(SPHERE_CENTRE)
        oc = o - c
        b = (oc * d).sum(-1)
        disc = b * b - ((oc * oc).sum(-1) - SPHERE_RADIUS**2)
        t = -b - torch.sqrt(disc.clamp(min=0))
        hit = (disc > 0) & (t > 0)
        depth = torch.where(hit, t, torch.zeros_like(t))[:, None]
        n = (o + depth * d - c) / SPHERE_RADIUS
        out = {"rgb": 0.5 + 0.5 * n, "depth": depth, "normal": n}
        return {k: v.to(bundle.origins.device) for k, v in out.items() if k in self.outputs}


class FakePipeline:
    def __init__(self, n: int = 1000, seed: int = 0, bundle_cls=SimpleBundle, device="cpu", miss_every: int = 0,
                 outputs=("rgb", "depth", "normal")):
        self.datamanager = FakeDataManager(n, seed, bundle_cls, device, miss_every)
        self.model = FakeModel(outputs)
        self.device = device


# ---------------------------------------------------------------------------------------------------------------------------------
# (a)
# ---------------------------------------------------------------------------------------------------------------------------------
def reference_flow(pipeline, remove: Callable, estimate: Callable, num_points: int = 1000000, remove_outliers: bool = True,
                   estimate_normals: bool = False, rgb_output_name: str = "rgb", depth_output_name: str = "depth",
                   normal_output_name: Optional[str] = None, use_bounding_box: bool = True, bounding_box_min=(-1.0, -1.0, -1.0),
                   bounding_box_max=(1.0, 1.0, 1.0), std_ratio: float = 10.0):
    """The reference's flow on torch-CPU.  ``remove(points [N,3] fp32 numpy, nb_neighbors, std_ratio)`` -> kept indices stands for
    open3d's remove_statistical_outlier, ``estimate(points)`` -> normals for estimate_normals.  Returns {"points", "colors", "normals"
    (or None), "outlier_args" (or None), "estimated" (bool), "batches"}; the error cases raise ValueError with the reference's message."""
    points, rgbs, normals = [], [], []
    kept, batches = 0, 0
    while True:
        with torch.no_grad():
            ray_bundle, _ = pipeline.datamanager.next_train(0)
            outputs = pipeline.model(ray_bundle)
        batches += 1
        for name, flag in ((rgb_output_name, "rgb_output_name"), (depth_output_name, "depth_output_name"),
                           (normal_output_name, "normal_output_name")):
            if name is not None and name not in outputs:
                raise ValueError(f"Could not find {name} in the model outputs. Please set --{flag} to one of: {outputs.keys()}")
        rgb, depth = outputs[rgb_output_name].cpu(), outputs[depth_output_name].cpu()
        normal = outputs[normal_output_name].cpu() if normal_output_name is not None else None
        point = ray_bundle.origins.cpu() + ray_bundle.directions.cpu() * depth
        if use_bounding_box:
            comp_l, comp_m = torch.tensor(bounding_box_min), torch.tensor(bounding_box_max)
            assert torch.all(comp_l < comp_m), f"Bounding box min {bounding_box_min} must be smaller than max {bounding_box_max}"
            mask = torch.all(torch.concat([point > comp_l, point < comp_m], dim=-1), dim=-1)
            point, rgb = point[mask], rgb[mask]
            if normal is not None:
                normal = normal[mask]
        points.append(point)
        rgbs.append(rgb)
        if normal is not None:
            normals.append(normal)
        kept += point.shape[0]
        if kept >= num_points:
            break
    out = {"points": torch.cat(points).float().numpy(), "colors": torch.cat(rgbs).float().numpy(), "normals": None, "outlier_args": None,
           "estimated": False, "batches": batches}
    ind = None
    if remove_outliers:
        out["outlier_args"] = (20, std_ratio)
        ind = np.asarray(remove(out["points"], 20, std_ratio), dtype=np.int64)
        out["points"], out["colors"] = out["points"][ind], out["colors"][ind]
    if estimate_normals:
        if normal_output_name is not None:
            raise ValueError("Cannot estimate normals and use normal_output_name at the same time")
        out["normals"], out["estimated"] = estimate(out["points"]), True
    elif normal_output_name is not None:
        n = torch.cat(normals)
        if ind is not None:
            n = n[torch.from_numpy(ind)]
        out["normals"] = n.float().numpy()
    return out


# ---------------------------------------------------------------------------------------------------------------------------------
# (b)
# ---------------------------------------------------------------------------------------------------------------------------------
def knn(points: np.ndarray, k: int, chunk: int = 512):
    """(mean distances [N] float64, neighbour indices [N,k] int32 with -1 past k_eff) of sdfb200_knn, by brute force:
    d2 = (dx dx + dy dy) + dz dz with dx = double(a) - double(b), the k_eff = min(k, N) smallest (d2, index) pairs (a stable sort
    breaks ties by index), and the square roots added in ascending order, divided by k_eff."""
    p = np.asarray(points, dtype=np.float32).astype(np.float64)
    n = len(p)
    k_eff = min(k, n)
    mean = np.empty(n, np.float64)
    idx = np.full((n, k), -1, np.int32)
    for i0 in range(0, n, chunk):
        q = p[i0:i0 + chunk]
        dx, dy, dz = (p[None, :, a] - q[:, None, a] for a in range(3))
        d2 = (dx * dx + dy * dy) + dz * dz
        order = np.argsort(d2, axis=1, kind="stable")[:, :k_eff]
        ds = np.take_along_axis(d2, order, axis=1)
        s = np.zeros(len(q))
        for j in range(k_eff):
            s = s + np.sqrt(ds[:, j])
        mean[i0:i0 + chunk] = s / k_eff
        idx[i0:i0 + chunk, :k_eff] = order
    return mean, idx


def covariances(points: np.ndarray, idx: np.ndarray):
    """[N,3,3] float64 covariances of sdfb200_point_normals: the cumulants x, y, z, xx, xy, xz, yy, yz, zz summed in list order over
    the entries >= 0, divided by their count, then E[ab] - E[a] E[b]."""
    p = np.asarray(points, dtype=np.float32).astype(np.float64)
    n, k = idx.shape
    m = np.zeros((n, 9))
    cnt = np.zeros(n)
    for j in range(k):
        ok = idx[:, j] >= 0
        x, y, z = (np.where(ok, p[np.maximum(idx[:, j], 0), a], 0.0) for a in range(3))
        for t, v in enumerate((x, y, z, x * x, x * y, x * z, y * y, y * z, z * z)):
            m[:, t] = np.where(ok, m[:, t] + v, m[:, t])
        cnt += ok
    m = m / np.maximum(cnt, 1)[:, None]
    c = np.empty((n, 3, 3))
    for (a, b), t in (((0, 0), 3), ((0, 1), 4), ((0, 2), 5), ((1, 1), 6), ((1, 2), 7), ((2, 2), 8)):
        c[:, a, b] = c[:, b, a] = m[:, t] - m[:, a] * m[:, b]
    return c


# ---------------------------------------------------------------------------------------------------------------------------------
# (c)
# ---------------------------------------------------------------------------------------------------------------------------------
def statistical_outliers(mean_distances: np.ndarray, std_ratio: float):
    """(kept indices ascending, threshold) of open3d's RemoveStatisticalOutliers given each point's mean distance to its
    min(nb_neighbors, N) nearest points (itself included): valid = mean > 0; the cloud mean and the Bessel-corrected standard deviation
    over the valid points; kept = valid and mean < mean + std_ratio std.  No valid point keeps nothing (threshold NaN)."""
    m = np.asarray(mean_distances, dtype=np.float64)
    valid = m > 0
    nv = int(valid.sum())
    if nv == 0:
        return np.zeros(0, np.int64), float("nan")
    cloud_mean = m[valid].sum() / nv
    with np.errstate(invalid="ignore", divide="ignore"):
        std = np.sqrt(((m[valid] - cloud_mean) ** 2).sum() / np.float64(nv - 1))
    threshold = cloud_mean + std_ratio * std
    return np.nonzero(valid & (m < threshold))[0].astype(np.int64), float(threshold)
