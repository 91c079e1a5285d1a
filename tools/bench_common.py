"""What the export bench tools (mesh_bench, texture_bench, tsdf_bench) share: device timing, the leading keys of their JSON result and
its output."""
import json
import os
import subprocess

import torch


def cuda_ms(fn, reps):
    """Device time per call of ``fn`` over ``reps`` calls, by CUDA events, after one warm-up call."""
    fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def header(tool):
    """tool, device and power_limit: the card's name and power limit belong beside every number measured on it."""
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                               capture_output=True, text=True, check=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        power = f"unavailable ({e})"
    return dict(tool=tool, device=torch.cuda.get_device_name(), power_limit=power)


def report(result, out=None):
    """Prints ``result`` as one JSON line and writes the line to ``out`` when given."""
    line = json.dumps(result)
    print(line)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as fh:
            fh.write(line + "\n")
