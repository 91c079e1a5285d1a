"""Field-call time of shapes OUTSIDE the fused kernel's family (generic kernels): exact-fp32 CUDA-core GEMMs vs the tensor-core Linear
engine (csrc/tc_linear.cu).  bakedsdf-shaped (off-axis PE deg 8, ref-nerf heads, L-inf contraction; SURVEY.md 8d config 5) and the stock
volsdf / neus 8x256 MLP without grid (config 3).  Prints one JSON line per (shape, precision).

    python tools/generic_bench.py [--rays 4096] [--samples 128]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sdfstudio_b200 as sb  # noqa: E402
from sdfstudio_b200 import synthetic  # noqa: E402

SHAPES = {
    "bakedsdf": dict(num_layers=2, num_layers_color=2, hidden_dim=256, use_grid_feature=True, position_encoding_max_degree=8, off_axis=True,
                     use_diffuse_color=True, use_specular_tint=True, use_reflections=True, use_n_dot_v=True, bias=0.05, beta_init=0.1, inside_outside=False),
    "volsdf_stock": dict(num_layers=8, num_layers_color=4, hidden_dim=256, use_grid_feature=False, bias=0.8, beta_init=0.1, inside_outside=True),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=4096)
    ap.add_argument("--samples", type=int, default=128)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--shape", default=None, choices=[None, *SHAPES])
    ap.add_argument("--precision", default=None, help="only this precision (skips the fp32 reference run and the rgb diff)")
    args = ap.parse_args()
    dev = torch.device("cuda")
    R, S = args.rays, args.samples
    o, d, cam, nears, fars = synthetic.dtu_like_rays(R, 11)
    rb = sb.RayBundle(origins=o.to(dev), directions=d.to(dev), pixel_area=torch.ones(R, 1, device=dev), directions_norm=torch.ones(R, 1, device=dev),
                      camera_indices=cam.view(R, 1).to(dev), nears=nears.to(dev), fars=fars.to(dev))
    rs = sb.UniformSampler(num_samples=S).eval()(rb)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    ref = {}
    for shape, kw in SHAPES.items():
        if args.shape and shape != args.shape:
            continue
        for prec in ((args.precision,) if args.precision else ("fp32", "bf16x3", "bf16")):
            torch.manual_seed(0)
            cfg = sb.SDFFieldConfig(grid_layout="torch", precision=prec, **kw)
            sd = sb.SceneContraction(order=float("inf")) if shape == "bakedsdf" else None
            field = synthetic.perturb_field_(sb.SDFField(cfg, torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), num_images=49, spatial_distortion=sd), 0).to(dev).eval()
            with torch.no_grad():
                for _ in range(2):
                    out = field(rs, return_alphas=True)
                torch.cuda.synchronize()
                tot = 0.0
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                for _ in range(args.steps):
                    flush.zero_()
                    e0.record()
                    out = field(rs, return_alphas=True)
                    e1.record()
                    torch.cuda.synchronize()
                    tot += e0.elapsed_time(e1)
            rgb = out[sb.FieldHeadNames.RGB]
            if prec == "fp32":
                ref[shape] = rgb
            err = float((rgb - ref[shape]).abs().max()) if shape in ref else None
            ms = tot / args.steps
            print(json.dumps({"shape": shape, "precision": prec, "rays": R, "samples": S, "field_ms": ms, "rays_per_s": R / ms * 1e3,
                              "max_abs_rgb_diff_vs_fp32": err}))


if __name__ == "__main__":
    main()
