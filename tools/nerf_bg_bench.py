"""Measures the "mlp" background field (NeRFField) on one GPU and writes profiles/r08_nerf_bg_bench.json (or --out):

(a) eval forward at 4096 x 32 and 65 536 x 32 samples: the fused kernel (k_nerf_field_tc, bf16x3 and bf16) against the reference-shaped
    module run as ATen fp32 layers, TF32 off and on, alternated; medians of CUDA-event timings over many launches after warm-up;
    samples/s, achieved TFLOP/s from the shapes and the share of the dense BF16 peak; max output difference against ATen fp32;
(b) the training composition (linear_ops GEMMs, bf16x3), forward + backward at 8192 x 48, against ATen fp32;
(c) SurfaceRenderer(kind="volsdf") at 4096 rays with and without the background, alternated.

    python tools/nerf_bg_bench.py [--out path] [--reps N]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import sdfstudio_b200 as sb  # noqa: E402

MAC_PER_SAMPLE = 63 * 256 + 3 * 256 * 256 + 319 * 256 + 3 * 256 * 256 + 256 + 283 * 128 + 128 * 128 + 128 * 3   # 544 256
BF16_DENSE_PEAK = 989e12     # H100 SXM data sheet, dense BF16, FLOP/s


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def make(precision, dev):
    pe = sb.NeRFEncoding(3, 10, 0.0, 9.0, include_input=True)
    de = sb.NeRFEncoding(3, 4, 0.0, 3.0, include_input=True)
    torch.manual_seed(0)
    f = sb.NeRFField(position_encoding=pe, direction_encoding=de, spatial_distortion=sb.SceneContraction(order=float("inf")), precision=precision)
    return f.to(dev)


def ray_samples(R, S, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    o = torch.randn(R, 3, generator=g) * 0.3
    d = torch.randn(R, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True)
    fars = 1.5 + 2.0 * torch.rand(R, 1, generator=g)
    rb = sb.RayBundle(origins=o.to(dev), directions=d.to(dev), pixel_area=torch.ones(R, 1, device=dev), camera_indices=torch.zeros(R, 1, dtype=torch.long, device=dev),
                      nears=fars.to(dev), fars=torch.full((R, 1), 1000.0, device=dev))
    return sb.LinearDisparitySampler(num_samples=S).eval()(rb)


def time_ms(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def alternate(fns, reps, rounds=7, warmup=3):
    """{name: median ms} of `rounds` rounds, each timing every fn over `reps` calls in turn."""
    for fn in fns.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    t = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            t[k].append(time_ms(fn, reps))
    return {k: statistics.median(v) for k, v in t.items()}


def eval_section(dev, reps):
    res = {}
    fields = {p: make(p, dev).eval() for p in ("bf16x3", "bf16", "fp32")}
    for R in (4096, 65536):
        rs = ray_samples(R, 32, dev)
        N = R * 32
        outs = {}

        def run(p):
            def f():
                with torch.no_grad():
                    outs[p] = fields[p](rs)
            return f

        def aten(tf32):
            def f():
                torch.backends.cuda.matmul.allow_tf32 = tf32
                with torch.no_grad():
                    outs["tf32" if tf32 else "fp32"] = fields["fp32"](rs)
                torch.backends.cuda.matmul.allow_tf32 = False
            return f

        r = max(2, reps * 4096 // R)
        t = alternate({"kernel_bf16x3": run("bf16x3"), "kernel_bf16": run("bf16"), "aten_fp32": aten(False), "aten_tf32": aten(True)}, r)
        ref = outs["fp32"]
        entry = {"samples": N, "ms": t, "launches_per_forward": None}
        n0 = sb._lib.launch_count()
        run("bf16x3")()
        torch.cuda.synchronize()
        entry["launches_per_forward"] = sb._lib.launch_count() - n0
        for k, key in (("kernel_bf16x3", "bf16x3"), ("kernel_bf16", "bf16"), ("aten_tf32", "tf32")):
            o = outs[key]
            entry[f"max_diff_vs_aten_fp32_{k}"] = {"density": float((o[sb.FieldHeadNames.DENSITY] - ref[sb.FieldHeadNames.DENSITY]).abs().max()),
                                                   "rgb": float((o[sb.FieldHeadNames.RGB] - ref[sb.FieldHeadNames.RGB]).abs().max())}
        for k, ms in t.items():
            flop = 2.0 * MAC_PER_SAMPLE * N
            entry[f"{k}_samples_per_s"] = N / (ms * 1e-3)
            entry[f"{k}_tflops_from_shapes"] = flop / (ms * 1e-3) / 1e12
        for k, mma in (("kernel_bf16x3", 3), ("kernel_bf16", 1)):
            entry[f"{k}_share_of_dense_bf16_peak"] = mma * 2.0 * MAC_PER_SAMPLE * N / BF16_DENSE_PEAK / (t[k] * 1e-3)
        res[f"{R}x32"] = entry
    return res


def train_section(dev, reps):
    rs = ray_samples(8192, 48, dev, seed=1)
    fields = {p: make(p, dev).train() for p in ("bf16x3", "fp32")}

    def step(p):
        def f():
            out = fields[p](rs)
            loss = out[sb.FieldHeadNames.RGB].sum() + out[sb.FieldHeadNames.DENSITY].sum() * 1e-3
            loss.backward()
        return f

    return {"samples": 8192 * 48, "ms_forward_backward": alternate({"compose_bf16x3": step("bf16x3"), "aten_fp32": step("fp32")}, max(2, reps // 8))}


def volsdf_section(dev, reps):
    import bench
    from sdfstudio_b200.synthetic import dtu_like_rays

    field = bench.make_field(dev, "bf16x3", beta_init=bench.VOLSDF_BETA).eval()
    sampler = sb.ErrorBoundedSampler(num_samples=64, num_samples_eval=128, num_samples_extra=32, eps=0.1, beta_iters=10, max_total_iters=5).eval()
    R = 4096
    o, d, cam, nears, fars = dtu_like_rays(R, 1000)
    pix = torch.ones(R, 1, device=dev)
    rb = sb.RayBundle(origins=o.to(dev), directions=d.to(dev), pixel_area=pix, directions_norm=pix, camera_indices=cam.view(R, 1).to(dev),
                      nears=nears.to(dev), fars=fars.to(dev))
    bgf = make("bf16x3", dev).eval()
    plain = sb.SurfaceRenderer(field, sampler, kind="volsdf", background_color="white").eval()
    with_bg = sb.SurfaceRenderer(field, sampler, kind="volsdf", background_color="white", field_background=bgf).eval()

    def run(m):
        def f():
            with torch.no_grad():
                m.get_outputs(rb)
        return f

    t = alternate({"volsdf_without_background": run(plain), "volsdf_with_mlp_background": run(with_bg)}, max(2, reps // 16))
    return {"rays": R, "ms": t, "background_cost_ms": t["volsdf_with_mlp_background"] - t["volsdf_without_background"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r08_nerf_bg_bench.json"))
    ap.add_argument("--reps", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("nerf_bg_bench needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    torch.backends.cuda.matmul.allow_tf32 = False
    res = {"card": card(), "mac_per_sample": MAC_PER_SAMPLE,
           "note": "TFLOP/s from the shapes count 2 x 544 256 FLOP per sample; bf16x3 issues 3 MMAs per product, so its share of the dense "
                   "BF16 peak counts 3x the shape FLOPs (the kernel's bound is the tensor-core rate)",
           "eval": eval_section(dev, args.reps), "train": train_section(dev, args.reps), "volsdf_render": volsdf_section(dev, args.reps)}
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
