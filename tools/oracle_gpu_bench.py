"""Context row (BASELINE.md section 3, optional): the headline step computed by the ORACLE modules (the restatement of the reference's
PyTorch code: torch-layout HashEncoding, nn.Linear-style matmuls, autograd for the sdf gradient) placed on the GPU, i.e. the reference's
pure-PyTorch path on ATen / cuBLAS kernels with TF32 matmuls like scripts/train.py:59.  NOT the tiny-cuda-nn path (that cannot be built
here: no source, no network) -- it is what `use_tcnn=False`-style PyTorch code achieves on the same GPU.
    python tools/oracle_gpu_bench.py [--rays 4096] [--steps 10]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from oracle import render, samplers  # noqa: E402
from oracle.field import FieldSpec, OracleField  # noqa: E402
from sdfstudio_b200.synthetic import dtu_like_rays  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--no-tf32", action="store_true")
    args = ap.parse_args()
    dev = torch.device("cuda")
    torch.backends.cuda.matmul.allow_tf32 = not args.no_tf32
    field = bench.make_field("cpu")
    spec = FieldSpec(num_layers=2, num_layers_color=2, hidden_dim=256, use_grid_feature=True, grid_layout="torch")
    sd = {k: v.detach().to(dev) for k, v in field.state_dict().items()}
    sd["hash_table"] = sd.pop("encoding.hash_table")
    R, S = args.rays, 128
    o, d, cam, nears, fars = (t.to(dev) for t in dtu_like_rays(R, 1000))
    torch.set_default_device(dev)      # the oracle creates its constants with the default device (it is written for the CPU)
    oracle = OracleField(spec, sd)
    white = torch.ones(3, device=dev)
    def step():
        b = samplers.spaced_sampler(nears, fars, S, "uniform")
        out = oracle.get_outputs(o, d, b.starts, b.deltas, cam, return_alphas=True)
        w, _ = samplers.weights_from_alphas(out["alphas"][..., 0])
        w = w[..., None]
        return (render.render_rgb(out["rgb"], w, white), render.render_depth(w, b.starts[..., None], b.ends[..., None], "expected"),
                render.render_semantics(out["normals"], w), render.render_accumulation(w))

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    print(json.dumps({"impl": "oracle modules on cuda (ATen / cuBLAS, TF32 matmuls)" if not args.no_tf32 else "oracle modules on cuda (ATen fp32)",
                      "metric": "rays/sec at 4096 rays x 128 samples", "value": R / ms * 1e3, "unit": "rays/s", "ms_per_step": ms, "rays": R, "samples_per_ray": S,
                      "note": "context only: the reference's pure-PyTorch path on the same GPU, not tiny-cuda-nn"}))


if __name__ == "__main__":
    main()
