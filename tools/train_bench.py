"""Training-step throughput of the differentiable path (DESIGN.md section 3b) on one GPU: NeuSSampler (fused kernels, no_grad) ->
SDFField training forward (ATen dense layers + this package's twice-differentiable grid operator) -> fused alpha compositing ->
rgb L1 + eikonal loss -> backward -> Adam.  Prints one JSON line; not the headline metric (bench.py is), but the number to hold
against the reference's README-derived ~45 k train-rays/s (RTX 3090, tcnn).

    python tools/train_bench.py [--rays 2048] [--steps 20] [--warmup 5] [--samples 64 --importance 64]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sdfstudio_b200 as sb  # noqa: E402
from sdfstudio_b200 import synthetic  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--samples", type=int, default=64)
    ap.add_argument("--importance", type=int, default=64)
    ap.add_argument("--precision", default="bf16x3", help="precision of the no_grad (sampler) kernels")
    ap.add_argument("--train-gemm", default="auto", choices=["auto", "tc", "aten"], help="dense layers of the training path: tensor-core GEMMs (linear_ops) or ATen")
    ap.add_argument("--no-tf32", action="store_true", help="keep ATen matmuls in fp32 (the reference trains with TF32, scripts/train.py:59)")
    args = ap.parse_args()
    dev = torch.device("cuda")
    torch.backends.cuda.matmul.allow_tf32 = not args.no_tf32
    torch.manual_seed(0)
    cfg = sb.SDFFieldConfig(use_grid_feature=True, num_layers=2, num_layers_color=2, hidden_dim=256, bias=0.5, beta_init=0.3, inside_outside=False,
                            grid_layout="torch", precision=args.precision, train_gemm=args.train_gemm)
    field = synthetic.perturb_field_(sb.SDFField(cfg, torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), num_images=49), 0).to(dev).train()
    sampler = sb.NeuSSampler(num_samples=args.samples, num_samples_importance=args.importance, num_samples_outside=0, num_upsample_steps=4).train()
    opt = torch.optim.Adam(field.parameters(), lr=5e-4, eps=1e-15)
    R = args.rays
    o, d, cam, nears, fars = synthetic.dtu_like_rays(R, 11)
    rb = sb.RayBundle(origins=o.to(dev), directions=d.to(dev), pixel_area=torch.ones(R, 1, device=dev), directions_norm=torch.ones(R, 1, device=dev),
                      camera_indices=cam.view(R, 1).to(dev), nears=nears.to(dev), fars=fars.to(dev))
    target = torch.rand(R, 3, device=dev)
    white = torch.ones(3, device=dev)
    ev = {k: [torch.cuda.Event(enable_timing=True) for _ in range(2)] for k in ("sample", "forward", "backward", "optim")}
    acc = {k: 0.0 for k in ev}

    def step(timed):
        def mark(k, i):
            if timed:
                ev[k][i].record()
        mark("sample", 0)
        with torch.no_grad():
            rs = sampler(rb, sdf_fn=field.get_sdf)
        mark("sample", 1); mark("forward", 0)
        fo = field(rs, return_alphas=True)
        out = sb.render_from_alphas(fo[sb.FieldHeadNames.ALPHA], fo[sb.FieldHeadNames.RGB], fo[sb.FieldHeadNames.NORMAL], rs, white, training=True)
        eik = ((fo[sb.FieldHeadNames.GRADIENT].norm(2, dim=-1) - 1) ** 2).mean()
        loss = (out["rgb"] - target).abs().mean() + 0.1 * eik
        mark("forward", 1); mark("backward", 0)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        mark("backward", 1); mark("optim", 0)
        opt.step()
        mark("optim", 1)
        if timed:
            torch.cuda.synchronize()
            for k in ev:
                acc[k] += ev[k][0].elapsed_time(ev[k][1])
        return float(loss.detach()) if timed else None

    for _ in range(args.warmup):
        step(False)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.steps):
        step(False)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / args.steps
    for _ in range(3):
        last = step(True)
    S = args.samples + args.importance
    print(json.dumps({"metric": "train rays/sec (NeuS sampler + SDFField fwd/bwd + Adam)", "value": R / ms * 1e3, "unit": "rays/s", "rays": R,
                      "samples_per_ray": S, "ms_per_step": ms, "phase_ms": {k: v / 3 for k, v in acc.items()}, "loss": last, "tf32_matmul": not args.no_tf32, "train_gemm": args.train_gemm,
                      "reference_note": "README-derived ~45k train-rays/s on RTX 3090 (SURVEY.md 8d iii)"}))


if __name__ == "__main__":
    main()
