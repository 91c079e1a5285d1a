"""neus-acc path on one GPU: occupancy prune, two-pass march, packed compositing, eval throughput and a training step.

Stock NeuS field (8 x 256, geometric init = a sphere of radius 0.8, perturbed with synthetic.perturb_field_), variance set for
inv_s ~ 1e3 (step_size = 14 / inv_s / 16), a 128^3 grid after one prune, DTU-like rays (synthetic.dtu_like_rays).  Writes one JSON line to
<out-dir>/neus_acc_bench.json and prints it.

    python tools/neus_acc_bench.py --out-dir <dir>
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "neus_acc_bench needs a CUDA device"

    import sdfstudio_b200 as sb
    from sdfstudio_b200 import _lib
    from sdfstudio_b200.synthetic import dtu_like_rays, perturb_field_

    dev = torch.device("cuda")
    torch.manual_seed(0)
    aabb = torch.tensor([[-1.0, -1, -1], [1, 1, 1]])
    field = perturb_field_(sb.SDFField(sb.SDFFieldConfig(inside_outside=False), aabb, 49), 0, scale=0.002)
    with torch.no_grad():
        field.deviation_network.variance.fill_(math.log(1000.0) / 10.0)
    field = field.to(dev).eval()
    inv_s = field.deviation_network.get_variance
    sdf_fn = lambda x: field.forward_geonetwork(x)[:, 0].contiguous()  # noqa: E731

    def fresh():
        s = sb.NeuSAccSampler(aabb=aabb, neus_sampler=sb.NeuSSampler(), resolution=128, steps_warpup=0, steps_per_grid_update=1).to(dev)
        s.update_step_size(0, inv_s=inv_s)
        return s

    with torch.no_grad():
        fresh().update_binary_grid(0, sdf_fn=sdf_fn, inv_s=inv_s)   # warm-up of every shape of the prune
        s = fresh()
        prune_ms = _time_ms(lambda: s.update_binary_grid(0, sdf_fn=sdf_fn, inv_s=inv_s), 1)
    res = {"workload": "neus-acc stock NeuS 8x256, 128^3 grid, inv_s ~ 1e3", "card": _card(), "step_size": s.step_size,
           "occupied_voxels": int(s._binary.sum()), "prune_ms_incl_sdf_eval": prune_ms}

    lib = _lib.load()
    march = {}
    for R in (2048, 32768):
        o, d, cam, nears, fars = dtu_like_rays(R, 1)
        o, d, nears, fars = o.to(dev), d.to(dev), nears[:, 0].to(dev).contiguous(), fars[:, 0].to(dev).contiguous()
        roi = (_lib.C.c_float * 6)(*s._roi_aabb)
        a = (_lib.ptr(o), _lib.ptr(d), _lib.ptr(nears), _lib.ptr(fars), R, roi, s._binary.data_ptr(), 128, s.step_size)
        counts = torch.empty(R, device=dev, dtype=torch.int32)
        count = lambda: _lib.check(lib.sdfb200_occupancy_march(*a, None, _lib.ptr(counts), None, None, None, _lib.stream_ptr()))  # noqa: E731
        count()
        off = torch.zeros(R + 1, device=dev, dtype=torch.int64)
        torch.cumsum(counts, 0, out=off[1:])
        n = int(off[-1])
        ri, ts, te = (torch.empty(n, device=dev, dtype=t) for t in (torch.int64, torch.float32, torch.float32))
        write = lambda: _lib.check(lib.sdfb200_occupancy_march(*a, _lib.ptr(off), None, _lib.ptr(ri), _lib.ptr(ts), _lib.ptr(te),  # noqa: E731
                                                               _lib.stream_ptr()))
        write()
        march[str(R)] = {"count_ms": _time_ms(count, args.reps), "write_ms": _time_ms(write, args.reps), "samples_per_ray": n / R}
    res["march"] = march

    R = 1 << 15
    o, d, cam, nears, fars = dtu_like_rays(R, 2)
    bundle = sb.RayBundle(origins=o.to(dev), directions=d.to(dev), pixel_area=torch.ones(R, 1, device=dev), directions_norm=torch.ones(R, 1, device=dev),
                          camera_indices=cam.view(R, 1).to(dev), nears=nears.to(dev), fars=fars.to(dev))

    def render():
        rs, ri = s(bundle, sdf_fn=field.get_sdf, alpha_fn=field.get_alpha)
        fo = field(rs, return_alphas=True)
        w = sb.packed.render_weight_from_alpha(fo[sb.FieldHeadNames.ALPHA], ray_indices=ri, n_rays=R)
        for v in (fo[sb.FieldHeadNames.RGB], fo[sb.FieldHeadNames.NORMAL], None, (rs.frustums.starts + rs.frustums.ends) / 2):
            sb.packed.accumulate_along_rays(w, ri, values=v, n_rays=R)
        return ri.numel()

    with torch.no_grad():
        n_eval = render()
        eval_ms = _time_ms(render, max(2, args.reps // 4))
    res["eval"] = {"rays": R, "samples_per_ray": n_eval / R, "ms": eval_ms, "rays_per_s": R / eval_ms * 1e3}

    Rt = 2048
    sub = sb.RayBundle(origins=bundle.origins[:Rt], directions=bundle.directions[:Rt], pixel_area=bundle.pixel_area[:Rt],
                       directions_norm=bundle.directions_norm[:Rt], camera_indices=bundle.camera_indices[:Rt], nears=bundle.nears[:Rt],
                       fars=bundle.fars[:Rt])
    target = torch.rand(Rt, 3, device=dev)
    field.train()

    def step():
        rs, ri = s(sub, sdf_fn=field.get_sdf, alpha_fn=field.get_alpha)
        fo = field(rs, return_alphas=True)
        w = sb.packed.render_weight_from_alpha(fo[sb.FieldHeadNames.ALPHA], ray_indices=ri, n_rays=Rt)
        rgb = sb.packed.accumulate_along_rays(w, ri, values=fo[sb.FieldHeadNames.RGB], n_rays=Rt)
        loss = (rgb - target).abs().mean() + 0.1 * ((fo[sb.FieldHeadNames.GRADIENT].norm(2, dim=-1) - 1) ** 2).mean()
        field.zero_grad(set_to_none=True)
        loss.backward()

    step()
    res["train_step"] = {"rays": Rt, "ms": _time_ms(step, max(2, args.reps // 4))}
    line = json.dumps(res)
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "neus_acc_bench.json"), "w") as fh:
        fh.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
