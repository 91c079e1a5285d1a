"""Times the mesh renderer at 1920 x 1080 with CUDA events after warm-up: the rasterizer (sdfb200_mesh_rasterize, keys only), the shader
(sdfb200_mesh_shade, "rgb" and "normal", on the rasterizer's keys), render_frames as a whole (camera packing, the mesh checks, vertex
normals, both kernels), the PNG encoding of both outputs (texturing.png_bytes_u8 on a thread pool, host clock) and
the whole render_trajectory_video call (PLY read, rendering, PNG files; host clock around a device synchronise), in ms per frame and
frames per second.

- Workloads: marching-cubes spheres (radius 0.45 of the lattice, bumped along the radius) of about 1 M and about 10 M faces seen whole
  by an orbit of 8 cameras; a decimated-scale UV sphere (about 20 k faces) seen close up; a camera inside a room (a box of 12 x 12
  quads per side), where faces cover up to a large part of the frame.
- The rasterizer's two paths: the same keys through the debug library's hook with every face on its own thread (threshold 2^62),
  every face on the block path (threshold 0) and the product threshold (SDFB200_MESH_LARGE_TRIANGLE_PIXELS), five repeats each,
  min / median / max.

The reference renders through open3d's OpenGL window and has no headless run on this machine to compare against.  Prints one JSON line
and writes it to --out.

    python tools/render_mesh_bench.py [--out profiles/r19_render_mesh_bench.json]
"""
import argparse
import concurrent.futures
import ctypes
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bench_common import cuda_ms, header, report  # noqa: E402
from oracle.make_golden_tsdf import look_at, on_sphere  # noqa: E402
from sdfstudio_b200 import _lib, meshing, render_mesh, texturing  # noqa: E402
from sdfstudio_b200.cameras import Cameras  # noqa: E402

H, W, FRAMES = 1080, 1920, 8


def mc_sphere(n):
    x = torch.arange(n, device="cuda", dtype=torch.float32) - (n - 1) / 2
    vol = (x.view(-1, 1, 1) ** 2 + x.view(1, -1, 1) ** 2 + x.view(1, 1, -1) ** 2).sqrt_() - 0.45 * (n - 1)
    v, f, _ = meshing.marching_cubes(vol, 0.0)
    del vol
    v = v / (n - 1) - 0.5
    return (v * (1 + 0.03 * torch.sin(9 * v[:, :1]) * torch.cos(7 * v[:, 1:2]))).contiguous(), f.long()


def uv_sphere(n_lat, n_lon):
    from test_gpu_render_mesh import uv_sphere as s

    v, f = s(n_lat, n_lon, 0.5)
    return torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()


def room(n):
    from test_gpu_render_mesh import box

    v, f = box(-1.0, 1.0, n, inward=True)
    return torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()


def orbit(dist, seed, target=(0.0, 0.0, 0.0), f=1400.0):
    return Cameras(look_at(on_sphere(FRAMES, dist, seed), target=target)[:, :3], f, f, W / 2, H / 2, W, H, device=torch.device("cuda"))


def spread(fn, reps, repeats=5):
    t = [cuda_ms(fn, reps) for _ in range(repeats)]
    return dict(min_ms=min(t), median_ms=statistics.median(t), max_ms=max(t), repeats=repeats, reps=reps)


def per_frame(ms):
    return dict(ms_per_frame=ms / FRAMES, frames_per_s=1e3 * FRAMES / ms)


def workload(v, f, cams):
    vv, ff, rows = render_mesh._prepare(v, f, cams)
    centre, ext = render_mesh._box(vv)
    zn = render_mesh._z_near(None, ext)
    out = dict(faces=len(ff), vertices=len(vv), frames=FRAMES, height=H, width=W)
    keys = render_mesh._keys(vv, ff, rows, H, W, zn)
    face = render_mesh.split_keys(keys)[0]
    out["covered_fraction"] = float((face >= 0).float().mean())
    dbg = _lib.load_debug()
    kd = torch.empty_like(keys)
    paths = {}
    for name, large in (("thread_per_face", 2**62), ("block_per_face", 0), ("product", None)):
        def run(large=large):
            if large is None:
                render_mesh._keys(vv, ff, rows, H, W, zn)
            else:
                _lib.check(dbg.sdfb200_debug_mesh_rasterize(_lib.ptr(vv), _lib.ptr(ff), len(ff), _lib.ptr(rows), FRAMES, H, W, zn, _lib.ptr(kd), large,
                                                            _lib.stream_ptr()))
        paths[name] = spread(run, 3)
        if large is not None:
            assert torch.equal(kd, keys), name
        paths[name].update(per_frame(paths[name]["median_ms"]))
    out["rasterize"] = paths
    normals = _lib.f32c(texturing.vertex_normals_area_weighted(vv, ff))
    lights = render_mesh.light_positions(rows, centre, ext)
    params = render_mesh.light_params()
    rgb = torch.empty(FRAMES, H, W, 3, dtype=torch.uint8, device="cuda")
    nrm = torch.empty_like(rgb)

    def shade():
        _lib.check(_lib.load().sdfb200_mesh_shade(_lib.ptr(keys), FRAMES, H, W, _lib.ptr(vv), _lib.ptr(normals), _lib.ptr(ff), len(ff), _lib.ptr(rows),
                                                  _lib.ptr(lights), params.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), _lib.ptr(rgb), _lib.ptr(nrm),
                                                  _lib.stream_ptr()))

    t = spread(shade, 3)
    t.update(per_frame(t["median_ms"]))
    out["shade_both_outputs"] = t
    # render_frames as a whole: camera packing, the mesh checks (host reads), vertex normals, rasterize and shade
    t = spread(lambda: render_mesh.render_frames(vv, ff, cams), 3)
    t.update(per_frame(t["median_ms"]))
    out["render_frames"] = t
    frames = {k: x.cpu().numpy() for k, x in render_mesh.render_frames(vv, ff, cams).items()}
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(32, os.cpu_count() or 1)) as pool:
        t0 = time.perf_counter()
        list(pool.map(texturing.png_bytes_u8, [frames[n][k] for n in frames for k in range(FRAMES)]))
        ms = (time.perf_counter() - t0) * 1e3
    out["png_both_outputs"] = dict(ms=ms, host_cpus=os.cpu_count(), **per_frame(ms))
    with tempfile.TemporaryDirectory() as d:
        ply = os.path.join(d, "mesh.ply")
        meshing.write_ply(ply, v.cpu().numpy(), f.cpu().numpy(), None)
        runs = []
        for _ in range(2):   # the first call warms up
            c = Cameras(cams.camera_to_worlds, cams.fx, cams.fy, cams.cx, cams.cy, W, H, device=cams.device)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            render_mesh.render_trajectory_video(ply, c, os.path.join(d, "out", "video.mp4"), ["rgb", "normal"], output_format="images")
            torch.cuda.synchronize()
            runs.append((time.perf_counter() - t0) * 1e3)
        out["whole_call_images"] = dict(ms=runs[-1], **per_frame(runs[-1]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "render_mesh_bench needs a GPU"
    result = header("render_mesh_bench")
    try:
        result["max_sm_clock"] = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader", "-i",
                                                 str(torch.cuda.current_device())], capture_output=True, text=True, check=True,
                                                timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        result["max_sm_clock"] = f"unavailable ({e})"
    result["baseline"] = "none: the reference renders through open3d's OpenGL window, which has no headless run here"
    result["workloads"] = {}
    for name, make, cams in (("mc_1m", lambda: mc_sphere(448), orbit(1.6, 1)), ("mc_10m", lambda: mc_sphere(1400), orbit(1.6, 2)),
                             ("decimated_20k_close_up", lambda: uv_sphere(100, 100), orbit(0.75, 3, f=1000.0)),
                             ("inside_room", lambda: room(12), orbit(0.3, 4, target=(0.2, -0.1, 0.1), f=800.0))):
        v, f = make()
        r = workload(v, f, cams)
        del v, f
        torch.cuda.empty_cache()
        result["workloads"][name] = r
        print(name, r, flush=True)
    report(result, args.out)


if __name__ == "__main__":
    main()
