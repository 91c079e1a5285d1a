"""Times the point-cloud exporter's neighbour search (sdfb200_knn) and outlier removal with CUDA events after warm-up, next to
scipy's cKDTree on the host cores and a chunked ATen cdist + topk on the same GPU, and breaks a whole point_cloud export down into
its stages.

- Clouds: surface-like (points on a sphere of radius 0.5 and on a floor plane, 4:1, with 0.2 % noise of 1e-3, the shape rendered
  points take) at 1 M points (the exporter's default) and 10 M, and a uniform volume cloud of 1 M points in [-1, 1]^3.
- sdfb200_knn at k = 20 (mean distances only, as the outlier removal asks) and k = 30 (neighbour lists, as the normals ask), and
  remove_statistical_outlier (20 neighbours, std_ratio 10) as a whole (box read-back, bucketing, search, reductions); five repeats of
  the event timing each, reported as min / median / max.  The grid each cloud gets (cells, occupied cells, points per occupied cell)
  is reported beside it.
- scipy.spatial.cKDTree(points).query(points, k, workers=-1) on the host (build and query timed separately), when scipy imports: the
  nearest stand-in for open3d's CPU KD-tree, not open3d.  ATen: torch.cdist over chunks of 2048 queries + topk(k, largest=False), fp32,
  at 1 M points.
- point_cloud at its defaults (1 M points, 32768 rays per batch, outliers removed) on a seeded SDFField through a SurfaceRenderer
  (NeuSSampler 64 + 64): the rendering loop, the outlier removal and the PLY write, each timed with a device synchronise.

Prints one JSON line and writes it to --out.

    python tools/pointcloud_bench.py [--out profiles/r16_pointcloud_bench.json]
"""
import argparse
import math
import os
import statistics
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import sdfstudio_b200 as sb  # noqa: E402
from bench_common import cuda_ms, header, report  # noqa: E402
from oracle.make_golden_tsdf import look_at, on_sphere  # noqa: E402
from sdfstudio_b200 import pointcloud, synthetic  # noqa: E402
from sdfstudio_b200.cameras import Cameras  # noqa: E402

AABB = torch.tensor([[-1.0, -1, -1], [1, 1, 1]])


def surface_cloud(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ns = n * 4 // 5
    s = torch.randn(ns, 3, generator=g, device="cuda")
    s = 0.5 * s / s.norm(dim=1, keepdim=True)
    f = torch.rand(n - ns, 3, generator=g, device="cuda") * 2 - 1
    f[:, 2] = -0.6
    p = torch.cat([s, f])
    noisy = torch.rand(n, generator=g, device="cuda") < 0.002
    return p + noisy[:, None] * 1e-3 * torch.randn(n, 3, generator=g, device="cuda")


def volume_cloud(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(n, 3, generator=g, device="cuda") * 2 - 1


def grid_stats(p):
    box = torch.cat([p.amin(0), p.amax(0)]).cpu()
    e = pointcloud.cell_log2(len(p), box)
    cmin, dims = pointcloud._grid(box, e)
    c = (torch.floor(p.double() * math.ldexp(1.0, -e)) - torch.tensor(cmin, dtype=torch.float64, device="cuda")).long()
    key = (c[:, 2] * dims[1] + c[:, 1]) * dims[0] + c[:, 0]
    occupied = int(torch.unique(key).numel())
    return dict(log2_cell=e, dims=dims, cells=math.prod(dims), occupied=occupied, points_per_occupied=len(p) / occupied)


def spread(fn, reps, repeats=5):
    t = [cuda_ms(fn, reps) for _ in range(repeats)]
    return dict(min_ms=min(t), median_ms=statistics.median(t), max_ms=max(t), repeats=repeats, reps=reps)


def scipy_run(p, k):
    try:
        from scipy.spatial import cKDTree
    except ImportError as e:
        return dict(unavailable=str(e))
    x = p.cpu().numpy()
    t0 = time.perf_counter()
    tree = cKDTree(x)
    t1 = time.perf_counter()
    tree.query(x, k, workers=-1)
    t2 = time.perf_counter()
    return dict(k=k, build_ms=(t1 - t0) * 1e3, query_ms=(t2 - t1) * 1e3, host_cpus=os.cpu_count())


def aten_run(p, k, chunk=2048):
    def run():
        for i in range(0, len(p), chunk):
            torch.cdist(p[i:i + chunk], p).topk(k, dim=1, largest=False)

    t = cuda_ms(run, 1)
    return dict(k=k, chunk=chunk, ms=t, dtype="fp32")


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def export_breakdown():
    cfg = sb.SDFFieldConfig(use_grid_feature=True, num_layers=2, num_layers_color=2, inside_outside=False, bias=0.5, precision="fp32")
    torch.manual_seed(0)
    field = synthetic.perturb_field_(sb.SDFField(cfg, AABB, num_images=49), seed=0).cuda().eval()
    renderer = sb.SurfaceRenderer(field, sb.NeuSSampler(num_samples=64, num_samples_importance=64).eval(), collider=sb.NearFarCollider(0.05, 5.0),
                                  kind="neus").eval()
    cams = Cameras(look_at(on_sphere(49, 2.5, 0))[:, :3, :], 172.8, 172.8, 96.0, 96.0, 192, 192, device=torch.device("cuda"))
    out = {}
    for num_points in (20000, 1000000):   # the first pass warms every shape
        rays = pointcloud._PixelRays(cams, 32768, 0)
        pipe = pointcloud._RendererPipeline(renderer, rays)
        cloud, out["render_ms"] = timed(lambda: pointcloud.generate_point_cloud(pipe, num_points=num_points, remove_outliers=False))
        (kept, _), out["outlier_removal_ms"] = timed(lambda: pointcloud.remove_statistical_outlier(cloud.points, 20, 10.0))
        cloud = pointcloud.PointCloud(cloud.points[kept], cloud.colors[kept])
        with tempfile.TemporaryDirectory() as d:
            _, out["write_ms"] = timed(lambda: cloud.export(os.path.join(d, "point_cloud.ply")))
            _, out["point_cloud_total_ms"] = timed(lambda: pointcloud.point_cloud(renderer, cams, d, num_points=num_points))
    out.update(num_points=1000000, kept=len(cloud), rays_per_batch=32768, sampler="NeuSSampler 64 + 64", field="SDFField fp32",
               cameras="49 x 192^2")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "pointcloud_bench needs a GPU"
    result = header("pointcloud_bench")
    clouds = {"surface_1m": surface_cloud(1_000_000, 0), "surface_10m": surface_cloud(10_000_000, 1), "volume_1m": volume_cloud(1_000_000, 2)}
    result["clouds"] = {}
    for name, p in clouds.items():
        reps = 2 if len(p) > 2_000_000 else 10
        r = dict(points=len(p), grid=grid_stats(p))
        r["knn_k20_mean"] = spread(lambda: pointcloud.nearest_neighbours(p, 20, neighbours=False), reps)
        r["knn_k30_indices"] = spread(lambda: pointcloud.nearest_neighbours(p, 30, mean_distances=False), reps)
        r["remove_statistical_outlier"] = spread(lambda: pointcloud.remove_statistical_outlier(p, 20, 10.0), reps)
        r["scipy_ckdtree_k20"] = scipy_run(p, 20)
        if len(p) <= 1_000_000:
            r["aten_cdist_topk_k20"] = aten_run(p, 20)
        result["clouds"][name] = r
        print(name, r, flush=True)
    result["point_cloud_export"] = export_breakdown()
    report(result, args.out)


if __name__ == "__main__":
    main()
