"""Per-phase cycle breakdown of the fused tensor-core field kernel (CTA 0, thread 0, first tiles): tile start, the end of every layer
(its MMAs plus the epilogue that precedes the next one start with the next stamp) and the tile end.  Uses the timing build of the kernel
inside libsdfb200_dbg.so (sdfstudio_b200/build.py).   usage: tools/tc_timing.py [precision] [log2T] [table dtype] [fused|unfused]"""
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from sdfstudio_b200 import _lib  # noqa: E402

_lib.LIB_PATH = os.path.join(_lib.HERE, "libsdfb200_dbg.so")     # same ABI + the stamped kernel
import sdfstudio_b200 as sb  # noqa: E402
from sdfstudio_b200.synthetic import dtu_like_rays, perturb_field_  # noqa: E402

prec = sys.argv[1] if len(sys.argv) > 1 else "bf16x3"
dev = torch.device("cuda")
log2t = int(sys.argv[2]) if len(sys.argv) > 2 else 19
tdt = sys.argv[3] if len(sys.argv) > 3 else "fp32"
fused = (sys.argv[4] if len(sys.argv) > 4 else "fused") == "fused"
torch.manual_seed(0)
cfg = sb.SDFFieldConfig(use_grid_feature=True, num_layers=2, num_layers_color=2, hidden_dim=256, bias=0.5, beta_init=0.3, inside_outside=False,
                        log2_hashmap_size=log2t, grid_layout="torch", precision=prec, table_dtype=tdt)
field = perturb_field_(sb.SDFField(cfg, torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), num_images=49), 0).to(dev).eval()
o, d, cam, nears, fars = dtu_like_rays(4096, 1000)
rb = sb.RayBundle(origins=o.to(dev), directions=d.to(dev), pixel_area=torch.ones(4096, 1, device=dev), directions_norm=torch.ones(4096, 1, device=dev),
                  camera_indices=cam.view(-1, 1).to(dev), nears=nears.to(dev), fars=fars.to(dev))
rs = sb.UniformSampler(num_samples=128).eval()(rb)
with torch.no_grad():
    for _ in range(3):
        if fused:
            field.render(rs, torch.ones(3, device=dev))
        else:
            field(rs, return_alphas=True)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
ms = []
with torch.no_grad():
    for _ in range(10):
        flush.zero_()
        e0.record()
        field.render(rs, torch.ones(3, device=dev)) if fused else field(rs, return_alphas=True)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
print(f"field call {sorted(ms)[len(ms)//2]:.3f} ms (median of 10, L2 flushed)")
lib = _lib.load()
lib.sdfb200_debug_tc_timing.argtypes = [ctypes.c_void_p]
buf = (ctypes.c_longlong * 512)()
assert lib.sdfb200_debug_tc_timing(buf) == 0
# stamps written by the kernel (field_tc_kernel.cuh, TC_STAMP): [0] tile start, [1 + L] end of layer L in the order the kernel runs them,
# [15] end of the tile (heads / compositing done); stamp 1 + L minus stamp L = the layer's MMAs + the epilogue before them
layers = ["encode+G0", "E0+G1", "E1+B1", "EB1+B0", "EB0+C0 misc", "h2 reload+C0 h2", "EC0+C1"]
for t in (5, 10):
    st = [buf[t * 32 + k] for k in range(32)]
    print(f"tile {t}: total {st[15] - st[0]} cycles  " + "  ".join(f"{n} {st[L + 1] - st[L]}" for L, n in enumerate(layers)) + f"  EC1+heads {st[15] - st[7]}")
