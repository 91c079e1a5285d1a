"""The grid background field (TCNNNerfactoField, default shape: 16 levels x 2 features, T = 2^19, base MLP 32-64-16, colour MLP
64-64-64-16) on one GPU:

(a) eval forward (one kernel launch) at 8192 x 48 and 65536 x 48 samples: kernel ms from CUDA events after warm-up, samples/s, achieved
    GB/s of hash-grid gathers and GFLOP/s (counted from the shapes), and the share of the bounding data-sheet peak;
(b) forward + backward of the training composition at 8192 x 48 samples;
(c) the angelo training step of tools/train_workload.py with and without this field and the reference's merge
    (forward_background_field_and_merge, models/base_surface_model.py:266-290), alternated in one process.

Writes one JSON line to <out-dir>/nerfacto_bg_bench.json and prints it.

    python tools/nerfacto_bg_bench.py --out-dir <dir>
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

PEAK_FP32_TFLOPS, PEAK_HBM_TBS = 67.0, 3.35   # H100 SXM data sheet (700 W)


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power, sm, sm_max = [v.strip() for v in q.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def _time_ms(fn, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def per_sample_cost(f):
    """(MACs, bytes of hash-grid gathers) of one sample of the eval kernel, from the descriptor"""
    nb, nh = f.mlp_base, f.mlp_head
    H, HC = nb.hidden_dim, nh.hidden_dim
    macs = nb.in_dim * H + (nb.n_hidden_layers - 1) * H * H + nb.n_output_dims * H
    macs += nh.in_dim * HC + (nh.n_hidden_layers - 1) * HC * HC + nh.n_output_dims * HC
    gathers = nb.desc.n_levels * 8 * nb.desc.n_features * 4
    return macs, gathers


def rays(R, S, seed):
    from sdfstudio_b200.synthetic import dtu_like_rays

    o, d, cam, nears, fars = dtu_like_rays(R, seed)
    bins = (nears + (fars * 2.5 - nears) * torch.linspace(0, 1, S + 1)[None]).float()   # reach well past the unit sphere
    return o, d, cam, bins


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "nerfacto_bg_bench needs a CUDA device"

    import sdfstudio_b200 as sb
    from sdfstudio_b200 import _lib
    from sdfstudio_b200.rays import make_ray_samples
    from sdfstudio_b200.synthetic import dtu_like_rays

    dev = torch.device("cuda")
    torch.manual_seed(0)
    aabb = torch.tensor([[-1.0, -1, -1], [1, 1, 1]])
    f = sb.TCNNNerfactoField(aabb, num_images=49, spatial_distortion=sb.SceneContraction(order=float("inf"))).to(dev)
    with torch.no_grad():
        nb = f.mlp_base
        nb.params[nb.n_net:].uniform_(-1, 1)
    macs, gather_bytes = per_sample_cost(f)
    res = {"workload": "TCNNNerfactoField default shape (SurfaceModel background_model='grid'), L-inf contraction", "card": _card(),
           "per_sample": {"macs": macs, "gather_bytes": gather_bytes}}

    lib = _lib.load()
    evals = {}
    for R in (8192, 65536):
        S = 48
        o, d, cam, bins = rays(R, S, 1)
        o, d, bins = o.to(dev), d.to(dev), bins.to(dev).contiguous()
        N = R * S
        dens, pre = torch.empty(N, device=dev), torch.empty(N, device=dev)
        rgb = torch.empty(N, 3, device=dev)
        p, ph = nb.params.detach(), f.mlp_head.params.detach()
        desc, nd = nb.desc, f._desc(S)
        app = f.embedding_appearance.mean(dim=0).detach().contiguous()

        def kernel():
            _lib.check(lib.sdfb200_nerfacto_field_forward(desc, nd, p[nb.n_net:].data_ptr(), p.data_ptr(), ph.data_ptr(), None, o.data_ptr(),
                                                          d.data_ptr(), bins.data_ptr(), R, app.data_ptr(), 0, dens.data_ptr(), rgb.data_ptr(),
                                                          pre.data_ptr(), None, _lib.stream_ptr()))

        kernel()
        ms = _time_ms(kernel, args.reps)
        flops, bytes_ = 2.0 * macs * N, float(gather_bytes) * N
        t_flop, t_mem = flops / (PEAK_FP32_TFLOPS * 1e12) * 1e3, bytes_ / (PEAK_HBM_TBS * 1e12) * 1e3
        rb = sb.RayBundle(origins=o, directions=d, pixel_area=torch.ones(R, 1, device=dev), camera_indices=cam.view(R, 1).to(dev))
        rs = make_ray_samples(rb, bins, bins, None)
        f.eval()
        with torch.no_grad():
            f(rs)
            module_ms = _time_ms(lambda: f(rs), max(5, args.reps // 5))
        evals[f"{R}x{S}"] = {"kernel_ms": ms, "module_forward_ms": module_ms, "samples_per_s": N / ms * 1e3, "gather_gbs": bytes_ / ms / 1e6,
                             "gflops": flops / ms / 1e6, "bound": "fp32" if t_flop > t_mem else "hbm",
                             "share_of_bounding_peak": max(t_flop, t_mem) / ms,
                             "peaks": {"fp32_tflops": PEAK_FP32_TFLOPS, "hbm_tbs": PEAK_HBM_TBS, "source": "H100 SXM data sheet"}}
    res["eval"] = evals

    # (b) the training composition, forward + backward
    R, S = 8192, 48
    o, d, cam, bins = rays(R, S, 2)
    rb = sb.RayBundle(origins=o.to(dev), directions=d.to(dev), pixel_area=torch.ones(R, 1, device=dev), camera_indices=cam.view(R, 1).to(dev))
    rs = make_ray_samples(rb, bins.to(dev).contiguous(), bins.to(dev).contiguous(), None)
    f.train()

    def train_fb():
        out = f(rs)
        loss = out[sb.FieldHeadNames.RGB].mean() + out[sb.FieldHeadNames.DENSITY].mean()
        f.zero_grad(set_to_none=True)
        loss.backward()

    train_fb()
    res["train_fwd_bwd"] = {"samples": R * S, "ms": _time_ms(train_fb, max(5, args.reps // 5))}

    # (c) the angelo step of tools/train_workload.py (its field, proposal sampler, step module and optimiser settings, TF32 for the ATen
    # leftovers, L2 flushed between timed steps) with and without the background field and the merge
    import train_workload as tw

    class StepWithBackground(tw.Step):
        """the angelo step with forward_background_field_and_merge (models/base_surface_model.py:257-290) between field and compositing"""

        def __init__(self, field, background):
            super().__init__(field)
            self.background = background

        def merge(self, rs_, alpha, rgb_):
            inside = (rs_.frustums.get_start_positions().norm(dim=-1, keepdim=True) < 1.0).float()
            fb = self.background(rs_)
            return (alpha * inside + (1.0 - inside) * rs_.get_alphas(fb[sb.FieldHeadNames.DENSITY]),
                    rgb_ * inside + (1.0 - inside) * fb[sb.FieldHeadNames.RGB])

    torch.backends.cuda.matmul.allow_tf32 = True                       # as tools/train_workload.py
    field = tw.make_angelo_field(dev, "bf16x3")
    sampler, fns = tw.make_proposal_sampler(dev)
    bg = sb.TCNNNerfactoField(aabb, num_images=49, spatial_distortion=sb.SceneContraction(order=float("inf"))).to(dev).train()
    models = {False: tw.Step(field), True: StepWithBackground(field, bg)}
    opts = {k: torch.optim.Adam([p for p in m.parameters() if p.requires_grad], lr=5e-4, eps=1e-15, fused=True) for k, m in models.items()}
    R = tw.R_TRAIN
    o, d, cam, nears, fars = dtu_like_rays(R, 2000)
    bundle = sb.RayBundle(origins=o.to(dev), directions=d.to(dev), pixel_area=torch.ones(R, 1, device=dev), directions_norm=torch.ones(R, 1, device=dev),
                          camera_indices=cam.view(-1, 1).to(dev), nears=nears.to(dev), fars=fars.to(dev))
    target = torch.rand(R, 3, device=dev)
    white = torch.ones(3, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def step(with_bg):
        with torch.no_grad():
            rs_, _, _ = sampler(bundle, density_fns=fns)
        loss = models[with_bg](rs_, target, white)
        opts[with_bg].zero_grad(set_to_none=True)
        loss.backward()
        opts[with_bg].step()

    for _ in range(3):
        step(False)
        step(True)
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for _ in range(args.steps):
        for with_bg in (False, True):
            flush.zero_()
            times[with_bg].append(_time_ms(lambda: step(with_bg), 1))
    ms_off, ms_on = (sorted(times[k])[len(times[k]) // 2] for k in (False, True))
    res["angelo_step"] = {"rays": R, "samples_per_ray": tw.S_TRAIN, "alternated_steps": args.steps, "l2": "flushed between timed steps (256 MiB write)",
                          "without_background": {"ms_median": ms_off, "train_rays_per_s": R / ms_off * 1e3},
                          "with_background_and_merge": {"ms_median": ms_on, "train_rays_per_s": R / ms_on * 1e3},
                          "background_share_ms": ms_on - ms_off}
    line = json.dumps(res)
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "nerfacto_bg_bench.json"), "w") as fh:
        fh.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
