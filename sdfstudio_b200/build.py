"""Builds libsdfb200.so (sm_90a) in-tree with nvcc.  `python -m sdfstudio_b200.build [--force]`."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libsdfb200.so")
LIB_DEBUG = os.path.join(HERE, "libsdfb200_dbg.so")   # product objects + the building-block validation hooks (tests only)
SOURCES = ["api.cu", "grid_encode.cu", "field_simt.cu", "field_tc.cu", "field_tc_p2_torch.cu", "field_tc_p2_tcnn.cu", "field_tc_p1_torch.cu", "field_tc_p1_tcnn.cu", "tc_linear.cu", "tc_wgrad.cu", "samplers.cu", "render.cu", "render_backward.cu", "density_field.cu", "rays_gen.cu"]
DEBUG_SOURCES = ["tc_test.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
         "-Xptxas", "-v"]


def _stale():
    if not os.path.exists(LIB) or not os.path.exists(LIB_DEBUG):
        return True
    t = min(os.path.getmtime(LIB), os.path.getmtime(LIB_DEBUG))
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", h) for h in ("sdfb200.h", "sdfb200_debug.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    if not os.path.exists(NVCC):
        raise RuntimeError(f"nvcc not found at {NVCC}; cannot build {LIB}")
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    dbg_objs = []
    for s in SOURCES + DEBUG_SOURCES:
        o = os.path.join(objdir, s.replace(".cu", ".o"))
        (dbg_objs if s in DEBUG_SOURCES else objs).append(o)
        cmd = [NVCC, *FLAGS, "-c", os.path.join(CSRC, s), "-o", o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    # the debug library carries a second build of the fused kernel with per-phase clock64 stamps (tools/tc_timing.py)
    timing_obj = os.path.join(objdir, "field_tc_p2_torch_timing.o")
    procs.append(("field_tc_p2_torch.cu [timing]", subprocess.Popen([NVCC, *FLAGS, "-DSDFB200_TC_TIMING", "-c", os.path.join(CSRC, "field_tc_p2_torch.cu"), "-o", timing_obj],
                                                                   stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for s, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {s}\n{out}")
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {s}:\n{out}")
    with open(os.path.join(objdir, "ptxas.log"), "w") as fh:
        fh.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    subprocess.check_call([NVCC, "-shared", "-o", LIB, *objs, "-lcudart"])
    dbg_all = [o for o in objs if not o.endswith("field_tc_p2_torch.o")] + [timing_obj] + dbg_objs
    subprocess.check_call([NVCC, "-shared", "-o", LIB_DEBUG, *dbg_all, "-lcudart"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
