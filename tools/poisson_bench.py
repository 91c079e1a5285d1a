"""Times the Poisson reconstruction (sdfstudio_b200.poisson) by phase with CUDA events, on surface-like clouds (the shapes
tools/pointcloud_bench.py uses: points on a sphere of radius 0.5 and on a floor plane, 4:1, with exact normals and 0.2 % of them
displaced by 1e-3) of 1 M and 10 M points at depth 9 and 10 M at depth 10, and on a clustered cloud of 1 M points (five blobs of
sigma 0.01, so that cells hold hundreds of points) at depth 9.

Phases, each bracketed by CUDA events on the current stream (the calls synchronise inside, so the span is the device time of the
phase): build_system (bucketing, screening blocks and right-hand side, coarse blocks), solve (with its cycles and residual, and the
iso value), mesh (marching cubes, density and colour), trim (the 10 % density quantile and remove_vertices_by_mask), and the whole
create_from_point_cloud_poisson call after one warm-up call.  The finest-level operator apply (sdfb200_poisson_apply) is timed over
repeated launches; its bytes are the least it must move (x read and y written once, the slot map once, each occupied cell's 8x8
block once) and are reported over kernel time against the H100 SXM's 3.35 TB/s.  The card's name, power limit and max SM clock are
read in the same run, and the peak allocated device memory of each case is reported.

    python tools/poisson_bench.py [--out profiles/r18_poisson_bench.json]
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sdfstudio_b200 as sb  # noqa: E402
from bench_common import cuda_ms, header, report  # noqa: E402
from sdfstudio_b200 import poisson  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def surface_cloud(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ns = n * 4 // 5
    s = torch.randn(ns, 3, generator=g, device="cuda")
    s = s / s.norm(dim=1, keepdim=True)
    f = torch.rand(n - ns, 3, generator=g, device="cuda") * 2 - 1
    f[:, 2] = -0.6
    p = torch.cat([0.5 * s, f])
    nrm = torch.cat([s, torch.tensor([[0.0, 0.0, 1.0]], device="cuda").expand(n - ns, 3)])
    noisy = torch.rand(n, generator=g, device="cuda") < 0.002
    p = p + noisy[:, None] * 1e-3 * torch.randn(n, 3, generator=g, device="cuda")
    return sb.PointCloud(p.contiguous(), torch.rand(n, 3, generator=g, device="cuda"), nrm.contiguous())


def clustered_cloud(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    centres = torch.rand(5, 3, generator=g, device="cuda") - 0.5
    d = torch.randn(n, 3, generator=g, device="cuda")
    p = centres[torch.arange(n, device="cuda") % 5] + 0.01 * d
    return sb.PointCloud(p, torch.rand(n, 3, generator=g, device="cuda"), d / d.norm(dim=1, keepdim=True))


def event_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    out = fn()
    e.record()
    torch.cuda.synchronize()
    return out, s.elapsed_time(e)


def run_case(pcd, depth):
    torch.cuda.reset_peak_memory_stats()
    poisson.create_from_point_cloud_poisson(pcd, depth=depth)       # warm-up: every shape of the timed calls
    torch.cuda.synchronize()
    r = dict(points=len(pcd), depth=depth, nodes=(2 ** depth + 1) ** 3)
    system, r["build_system_ms"] = event_ms(lambda: poisson.build_system(pcd.points, pcd.normals, pcd.colors, depth))
    _, r["solve_ms"] = event_ms(lambda: poisson.solve(system))
    r.update(cycles=system.cycles, residual=system.residual)
    (mesh, dens), r["mesh_ms"] = event_ms(lambda: poisson.mesh_from_system(system))
    r.update(vertices=len(mesh.vertices), faces=len(mesh.faces))
    _, r["trim_ms"] = event_ms(lambda: poisson.remove_vertices_by_mask(mesh, poisson.low_density_mask(dens)))
    occupied = system.mats[depth].shape[0]
    r.update(occupied_cells=occupied, points_per_occupied_cell=len(system.points) / occupied)
    x = torch.randn(r["nodes"], device="cuda")
    apply_ms = cuda_ms(lambda: poisson.apply_operator(system, depth, x), 10)
    nbytes = 8 * r["nodes"] + 4 * 8 ** depth + 256 * occupied
    r["apply"] = dict(ms=apply_ms, min_bytes=nbytes, bytes_per_s=nbytes / (apply_ms * 1e-3),
                      share_of_3_35_tb_s=nbytes / (apply_ms * 1e-3) / HBM_BYTES_PER_S)
    del system, mesh, dens, x
    _, r["create_from_point_cloud_poisson_ms"] = event_ms(lambda: poisson.create_from_point_cloud_poisson(pcd, depth=depth))
    r["peak_allocated_gb"] = torch.cuda.max_memory_allocated() / 1e9
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "poisson_bench needs a GPU"
    result = header("poisson_bench")
    try:
        result["max_sm_clock"] = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader", "-i",
                                                 str(torch.cuda.current_device())], capture_output=True, text=True, check=True,
                                                timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        result["max_sm_clock"] = f"unavailable ({e})"
    result["cases"] = {}
    for name, make, n, depth in (("surface_1m_d9", surface_cloud, 1_000_000, 9), ("clustered_1m_d9", clustered_cloud, 1_000_000, 9),
                                 ("surface_10m_d9", surface_cloud, 10_000_000, 9), ("surface_10m_d10", surface_cloud, 10_000_000, 10)):
        r = run_case(make(n, 0), depth)
        result["cases"][name] = r
        print(name, r, flush=True)
        torch.cuda.empty_cache()
    report(result, args.out)


if __name__ == "__main__":
    main()
