"""Times TSDF fusion (sdfb200_tsdf_integrate) with CUDA events after a warm-up of every shape, next to the reference's ATen fusion on
the same GPU, and breaks a whole tsdf_mesh export down into its stages.

- Fusion of 49 cameras at 192 x 192 (DTU-shaped: 49 views, rendered at downscale 2) into 128^3, 256^3 and 512^3, all images in one
  call.  Bytes = 52 per voxel (voxel_coords 12, values and weights 4 + 4, colors 12, each read, then values, weights and colors
  written) plus the images; (voxel, image) pairs = voxels x 49.
- Restatement (a) of oracle/tsdf.py (the reference's ops) at the exporter's batch_size=10 on the same GPU: the time of all five batches,
  or the out-of-memory error it raises.
- tsdf_mesh on a seeded SDFField through a SurfaceRenderer (NeuSSampler 64 + 64, fp32 field), 49 cameras of 192 x 192 at downscale 2,
  resolution 256: render, integrate, marching cubes (get_mesh) and write (export_mesh), each timed with a device synchronise.

Prints one JSON line and writes it to --out.

    python tools/tsdf_bench.py [--out profiles/r15_tsdf_bench.json]
"""
import argparse
import os
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import sdfstudio_b200 as sb  # noqa: E402
from bench_common import cuda_ms, header, report  # noqa: E402
from oracle import tsdf as ot  # noqa: E402
from oracle.make_golden_tsdf import intrinsics, look_at, on_sphere, sphere_images  # noqa: E402
from sdfstudio_b200 import synthetic, tsdf  # noqa: E402
from sdfstudio_b200.cameras import Cameras  # noqa: E402

N_CAMS, HW = 49, 192
BYTES_PER_VOXEL = 52
AABB = torch.tensor([[-1.0, -1, -1], [1, 1, 1]])


def images():
    c2w = look_at(on_sphere(N_CAMS, 2.5, 0))
    K = intrinsics(N_CAMS, 0.9 * HW, HW, HW)
    depth, color = sphere_images(c2w, K, HW, HW, 1)
    return c2w.cuda(), K.cuda(), depth.cuda(), color.cuda()


def kernel_run(res, c2w, K, depth, color, reps):
    t = tsdf.TSDF.from_aabb(AABB, torch.tensor([res] * 3)).to("cuda")
    ms = cuda_ms(lambda: t.integrate_tsdf(c2w, K, depth, color), reps)
    n = res**3
    nbytes = BYTES_PER_VOXEL * n + (depth.numel() + color.numel()) * 4
    return dict(resolution=res, voxels=n, images=N_CAMS, image_hw=[HW, HW], kernel_ms=ms, bytes=nbytes, bytes_per_s=nbytes / (ms * 1e-3),
                pairs=n * N_CAMS, pairs_per_s=n * N_CAMS / (ms * 1e-3))


def reference_run(res, c2w, K, depth, color, batch_size=10):
    run = dict(resolution=res, batch_size=batch_size)
    try:
        st = [x.cuda() for x in ot.from_aabb(AABB, torch.tensor([res] * 3))]
        tr = ot.truncation(st[4])
        ot.integrate(*st[:4], tr, c2w[:batch_size], K[:batch_size], depth[:batch_size], color[:batch_size])   # warm-up
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        ot.integrate_batched(st[:4], tr, c2w, K, depth, color, batch_size)
        e.record()
        torch.cuda.synchronize()
        run["ms"] = s.elapsed_time(e)
    except torch.cuda.OutOfMemoryError as err:
        run["out_of_memory"] = str(err).split("\n")[0]
    st = None
    torch.cuda.empty_cache()
    run["peak_allocated_gb"] = torch.cuda.max_memory_allocated() / 1e9
    torch.cuda.reset_peak_memory_stats()
    return run


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def export_breakdown(res=256, downscale=2):
    cfg = sb.SDFFieldConfig(use_grid_feature=True, num_layers=2, num_layers_color=2, inside_outside=False, bias=0.5, precision="fp32")
    torch.manual_seed(0)
    field = synthetic.perturb_field_(sb.SDFField(cfg, AABB, num_images=49), seed=0).cuda().eval()
    renderer = sb.SurfaceRenderer(field, sb.NeuSSampler(num_samples=64, num_samples_importance=64).eval(), collider=sb.NearFarCollider(0.05, 5.0),
                                  kind="neus").eval()
    out = {}
    for warm in (True, False):
        cams = Cameras(look_at(on_sphere(N_CAMS, 2.5, 0))[:, :3, :], 0.9 * HW, 0.9 * HW, HW / 2, HW / 2, HW, HW, device=torch.device("cuda"))
        t = tsdf.TSDF.from_aabb(AABB, torch.tensor([32 if warm else res] * 3)).to("cuda")
        (rgb, depth), out["render_ms"] = timed(lambda: tsdf.render_images(renderer, cams, "rgb", "depth", "cuda", 1.0 / downscale))
        c2w = torch.cat([cams.camera_to_worlds, torch.tensor([0.0, 0, 0, 1], device="cuda").expand(N_CAMS, 1, 4)], dim=1)
        _, out["integrate_ms"] = timed(lambda: t.integrate_tsdf(c2w, cams.get_intrinsics_matrices(), depth, rgb))
        mesh, out["marching_cubes_ms"] = timed(t.get_mesh)
        with tempfile.TemporaryDirectory() as d:
            _, out["write_ms"] = timed(lambda: tsdf.TSDF.export_mesh(mesh, os.path.join(d, "tsdf_mesh.ply")))
    out.update(resolution=res, cameras=N_CAMS, rendered_hw=list(rgb.shape[-2:]), rays=N_CAMS * rgb.shape[-1] * rgb.shape[-2],
               vertices=len(mesh.vertices), faces=len(mesh.faces), sampler="NeuSSampler 64 + 64", field="SDFField fp32")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tsdf_bench needs a GPU"
    result = header("tsdf_bench")
    c2w, K, depth, color = images()
    result["kernel"] = [kernel_run(r, c2w, K, depth, color, reps) for r, reps in ((128, 50), (256, 20), (512, 5))]
    result["reference_ops_batch10"] = [reference_run(r, c2w, K, depth, color) for r in (128, 256, 512)]
    result["tsdf_mesh_export"] = export_breakdown()
    report(result, args.out)


if __name__ == "__main__":
    main()
