"""Times meshing.extract_mesh on a perturbed neus-facto-shaped SDFField at resolution 512 and 1024, split into SDF evaluation, the
marching-cubes calls and the rest (lattice, pyramid, masks, host reads: torch plumbing), with CUDA events after a warm-up of every shape.
The two marching-cubes passes are also timed alone on the last block's volume: bytes = the volume read by both passes + the outputs,
over their kernel time, against the H100 SXM's 3.35 TB/s.  Prints one JSON line (and writes it to --out).

    python tools/mesh_bench.py [--precision bf16x3] [--out mesh_bench.json]
"""
import argparse
import ctypes as C
import os
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sdfstudio_b200 as sb  # noqa: E402
from bench_common import header, report  # noqa: E402
from sdfstudio_b200 import _lib, meshing, synthetic  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def make_field(precision):
    # object-centred (inside_outside=False): a sphere of radius 0.5 at initialisation, perturbed
    cfg = sb.SDFFieldConfig(use_grid_feature=True, num_layers=2, num_layers_color=2, inside_outside=False, bias=0.5, precision=precision)
    torch.manual_seed(0)                                                 # the geometric initialisation draws from the global RNG
    f = sb.SDFField(cfg, torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), num_images=49).cuda().eval()
    f = synthetic.perturb_field_(f, seed=0)
    # the perturbation moves the initial sphere's level by up to ~0.8: shift the SDF head's bias so that the SDF is -0.5 at the origin
    with torch.no_grad():
        s0 = meshing.sdf_fn(f)(torch.zeros(1, 3, device="cuda")).item()
        getattr(f, f"glin{f.num_layers - 2}").bias[0] -= s0 + 0.5
    return f


class Timed:
    """wraps a callable; the device time of its calls, measured by event pairs read after the run."""

    def __init__(self, fn):
        self.fn, self.events, self.count, self.last = fn, [], 0, None

    def __call__(self, *a, **k):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = self.fn(*a, **k)
        e.record()
        self.events.append((s, e))
        self.count += 1
        return out

    def ms(self):
        return sum(s.elapsed_time(e) for s, e in self.events)


def run(field, resolution, out_dir):
    sdf = Timed(meshing.sdf_fn(field))
    mc_calls = []
    mc = Timed(meshing.marching_cubes)

    def mc_rec(volume, *a, **k):
        r = mc(volume, *a, **k)
        mc_calls.append((volume, r[1].shape[0], r[0].shape[0], k.get("mask", a[2] if len(a) > 2 else None)))
        return r

    orig_sdf_fn, orig_mc = meshing.sdf_fn, meshing.marching_cubes
    meshing.sdf_fn, meshing.marching_cubes = (lambda field, level=0.0: sdf), mc_rec
    try:
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        s.record()
        meshing.extract_mesh(field, resolution=resolution, output_path=os.path.join(out_dir, f"mesh_{resolution}.ply"))
        e.record()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    finally:
        meshing.sdf_fn, meshing.marching_cubes = orig_sdf_fn, orig_mc
    total = s.elapsed_time(e)
    return dict(resolution=resolution, total_ms=total, wall_s=wall, sdf_ms=sdf.ms(), sdf_calls=sdf.count, marching_cubes_ms=mc.ms(),
                marching_cubes_calls=mc.count, plumbing_ms=total - sdf.ms() - mc.ms(),
                triangles=sum(c[1] for c in mc_calls), vertices=sum(c[2] for c in mc_calls)), mc_calls


def count_points(field, resolution, out_dir):
    n = [0]
    f = meshing.sdf_fn(field)

    def counting(x):
        n[0] += x.shape[0]
        return f(x)

    orig = meshing.sdf_fn
    meshing.sdf_fn = lambda field, level=0.0: counting
    try:
        meshing.extract_mesh(field, resolution=resolution, output_path=os.path.join(out_dir, "count.ply"))
    finally:
        meshing.sdf_fn = orig
    return n[0]


def kernel_passes(volume, mask, reps=10):
    """device time of the count and emit passes alone on `volume` (same calls as meshing.marching_cubes)."""
    lib = _lib.load()
    vol = volume.contiguous()
    m = None if mask is None else mask.to(torch.uint8).contiguous()
    dims = (C.c_int64 * 3)(*vol.shape)
    org, sp = (C.c_float * 3)(0, 0, 0), (C.c_float * 3)(1, 1, 1)
    U = vol.shape[0] * vol.shape[1]
    counts = torch.empty(2, U, device="cuda", dtype=torch.int32)
    stream = _lib.stream_ptr()

    def count():
        _lib.check(lib.sdfb200_marching_cubes(_lib.ptr(vol), dims, 0.0, _lib.ptr(m), org, sp, None, _lib.ptr(counts), None, None, None, stream))

    count()
    offsets = torch.zeros(2, U + 1, device="cuda", dtype=torch.int64)
    torch.cumsum(counts, 1, out=offsets[:, 1:])
    nv, nf = (int(v) for v in offsets[:, -1].cpu())
    off = offsets[:, :-1].contiguous()
    verts, normals = torch.empty(nv, 3, device="cuda"), torch.empty(nv, 3, device="cuda")
    faces = torch.empty(nf, 3, device="cuda", dtype=torch.int32)

    def emit():
        _lib.check(lib.sdfb200_marching_cubes(_lib.ptr(vol), dims, 0.0, _lib.ptr(m), org, sp, _lib.ptr(off), _lib.ptr(counts), _lib.ptr(verts),
                                              _lib.ptr(normals), _lib.ptr(faces), stream))

    res = {}
    for name, fn in (("count", count), ("emit", emit)):
        fn()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(reps):
            fn()
        e.record()
        torch.cuda.synchronize()
        res[f"{name}_ms"] = s.elapsed_time(e) / reps
    kernel_ms = res["count_ms"] + res["emit_ms"]
    nbytes = 2 * vol.numel() * 4 + (0 if m is None else 2 * m.numel()) + nv * 24 + nf * 12 + counts.numel() * 4 * 2 + off.numel() * 8
    res.update(volume=list(vol.shape), vertices=nv, triangles=nf, bytes=nbytes, kernel_ms=kernel_ms,
               bytes_per_s=nbytes / (kernel_ms * 1e-3), share_of_3_35_TBps=nbytes / (kernel_ms * 1e-3) / HBM_BYTES_PER_S)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="bf16x3")
    ap.add_argument("--resolutions", default="512,1024")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_bench needs a CUDA device")
    field = make_field(args.precision)
    result = dict(header("mesh_bench"), precision=args.precision, runs=[])
    with tempfile.TemporaryDirectory() as tmp:
        for res in (int(r) for r in args.resolutions.split(",")):
            run(field, res, tmp)                                         # warm-up of every shape this resolution uses
            r, calls = run(field, res, tmp)
            r["points"] = count_points(field, res, tmp)
            vol, _, _, mask = calls[-1]
            r["marching_cubes_kernels_last_block"] = kernel_passes(vol, mask)
            result["runs"].append(r)
            del calls
    report(result, args.out)


if __name__ == "__main__":
    main()
