"""Time of the interlevel loss, forward + backward, for the package's kernels and for the same arithmetic through ATen.

    python tools/interlevel_bench.py [--calls 200] [--warmup 20] [--out profiles/NAME.json]

Both forms (interlevel_loss, interlevel_loss_zip) over neus-facto's levels, (256, 96) proposal samples against 48 final samples, at
R = 2048, 4096 and 8192 rays.  The ATen side is oracle/losses.py moved to the GPU: the reference's operations, one ATen call each, without
its host-side assert.  The two sides alternate in blocks inside one process; each block is timed with CUDA events around all of its calls,
so a figure is a mean over at least --calls calls.  Kernel launches per call are counted with torch.profiler in a separate, untimed call.
Prints one JSON line (and writes it to --out).  Needs a GPU: it fails without one."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LEVELS = (256, 96, 48)
RAYS = (2048, 4096, 8192)
BLOCKS = 4


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                       capture_output=True, text=True)
    if q.returncode != 0 or not q.stdout.strip():
        return {"name": torch.cuda.get_device_name(), "power_limit": "unavailable"}
    name, power, sm_max = [v.strip() for v in q.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "sm_clock_max": sm_max}


def histogram(R, S, g):
    widths = torch.rand(R, S, generator=g) ** 2 + 0.02
    edges = torch.cat([torch.zeros(R, 1), torch.cumsum(widths, -1) / widths.sum(-1, keepdim=True)], -1)
    w = torch.rand(R, S, generator=g) ** 3
    return edges.cuda().contiguous(), (w / w.sum(-1, keepdim=True) * 0.9).cuda().contiguous()


def make_steps(R, form):
    """(package step, ATen step): each runs forward + backward once on the same inputs."""
    import types

    import sdfstudio_b200 as sb
    from oracle import losses as olosses

    g = torch.Generator().manual_seed(R)
    hist = [histogram(R, s, g) for s in LEVELS]
    leaves = [w.clone().requires_grad_(True) for _, w in hist[:-1]]
    samples = [types.SimpleNamespace(spacing_starts=e[:, :-1, None], spacing_ends=e[:, 1:, None], _spacing_bins=e) for e, _ in hist]
    weights = [x[..., None] for x in leaves] + [hist[-1][1][..., None]]
    ours = sb.interlevel_loss if form == "outer" else sb.interlevel_loss_zip
    theirs = olosses.interlevel_loss if form == "outer" else olosses.interlevel_loss_zip
    edges = [e for e, _ in hist]

    def package():
        for x in leaves:
            x.grad = None
        ours(weights, samples).backward()

    def aten():
        for x in leaves:
            x.grad = None
        theirs(edges, leaves + [hist[-1][1]]).backward()

    return package, aten


def time_ms(fn, calls):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(calls):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / calls


def kernels_per_call(fn):
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower() and "memset" not in e.name.lower())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("interlevel_bench needs a CUDA device")
    import sdfstudio_b200 as sb

    result = dict(tool="interlevel_bench", card=card(), levels=list(LEVELS), calls_per_figure=BLOCKS * args.calls, runs=[])
    for form in ("outer", "zip"):
        for R in RAYS:
            package, aten = make_steps(R, form)
            for _ in range(args.warmup):
                package()
                aten()
            torch.cuda.synchronize()
            n0 = sb._lib.launch_count()
            package()
            own_launches = sb._lib.launch_count() - n0
            t = {"package": [], "aten": []}
            for _ in range(BLOCKS):                              # alternate the two sides so that drift hits both
                t["package"].append(time_ms(package, args.calls))
                t["aten"].append(time_ms(aten, args.calls))
            run = dict(form=form, rays=R,
                       package_ms=sum(t["package"]) / BLOCKS, package_ms_blocks=[round(x, 5) for x in t["package"]],
                       aten_ms=sum(t["aten"]) / BLOCKS, aten_ms_blocks=[round(x, 5) for x in t["aten"]],
                       package_library_launches=own_launches, package_kernels=kernels_per_call(package), aten_kernels=kernels_per_call(aten))
            run["aten_over_package"] = round(run["aten_ms"] / run["package_ms"], 2)
            run["package_ms"], run["aten_ms"] = round(run["package_ms"], 5), round(run["aten_ms"], 5)
            result["runs"].append(run)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
