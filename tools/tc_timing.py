"""Per-phase cycle breakdown of the fused tensor-core field kernel (CTA 0, consumer thread 0, first tiles): the wait for the staged geo
input, every epilogue and every layer's MMAs apart, EC1, the cycles the consumers waited for weights and the producer for a
free ring slot, each encoder warp's cycles staging the tile and running its heads, encoder thread 0's heads split by kind of work and
its slot and barrier waits.  Uses the timing build of the kernel
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
buf = (ctypes.c_longlong * 768)()
assert lib.sdfb200_debug_tc_timing(buf) == 0
# stamps written by the kernel (field_tc_kernel.cuh, TC_STAMP / TC_PUT), consumer thread 0: [0] tile start, [8] the tile's geo input
# has landed (a_full), [1 + L] end of layer L's MMAs in the order the kernel runs them, [18..23] end of the epilogues E0, E1, EB1, EB0,
# h2 operand (the late h2 bulk copy issued), EC0 (the epilogue in front of layers 1..6), [15] end of the tile (EC1 done, head inputs handed to the heads warp).  An
# epilogue's cycles run from the end of the layer before it to its own stamp; a layer's MMA cycles from the end of the epilogue in front
# of it (or the a_full stamp for G0) to the layer's stamp, so they include the warpgroup barrier and any wait for weights.  Cycle sums
# over the tile: [9] consumer thread 0 waiting for weights, [10] producer waiting for a free ring slot, [12] encoder thread 0 busy
# staging the tile, [13] encoder thread 0 waiting for the tile's staging slot (enc_empty), [14] encoder thread 0 running the tile's
# heads and compositing, [16] consumer thread 0 waiting for the tile's head-input buffer (hs_empty), [17] encoder thread 0 waiting for
# the tile's head inputs (hs_full); per encoder warp w0 / w1 / w2 (lane 0): busy staging [12] [24] [25] and running
# the tile's heads [14] [26] [27]; encoder thread 0's heads split [28] per-row heads, [29] transmittance scan + weights, [30] sums and
# ray finish, and [31] its wait at the encoder warps' barrier; [32 + 3 w + k] encoder warp w's staging split by item kind k (grid,
# PE, colour-static); [41 + w] encoder warp w's staging of the tile's point geometry (with the encoder warps' barrier after it).
layers = ["G0", "G1", "B1", "B0", "C0 misc", "C0 h2", "C1"]
epis = ["E0", "E1", "EB1", "EB0", "h2 operand", "EC0"]     # epis[L - 1] runs in front of layer L; "h2 operand": the late h2 copy is issued
for t in (5, 10):
    st = [buf[t * 48 + k] for k in range(48)]
    epi = [st[18 + L] - st[1 + L] for L in range(6)] + [st[15] - st[7]]
    mma = [st[1] - st[8]] + [st[2 + L] - st[18 + L] for L in range(6)]
    print(f"tile {t}: total {st[15] - st[0]} cycles  a_full wait {st[8] - st[0]}  |  epilogues {sum(epi)}: "
          + "  ".join(f"{n} {v}" for n, v in zip(epis + ["EC1"], epi))
          + f"  |  MMAs {sum(mma)}: " + "  ".join(f"{n} {v}" for n, v in zip(layers, mma))
          + f"  |  consumer weight wait {st[9]}  hs_empty wait {st[16]}  producer slot wait {st[10]}"
          + f"  |  encoder busy {st[12]}  encoder slot wait {st[13]}  heads {st[14]}  heads wait {st[17]}"
          + f"  |  encoder warps w0/w1/w2: staging {st[12]}/{st[24]}/{st[25]}  heads {st[14]}/{st[26]}/{st[27]}"
          + f"  busy {st[12] + st[14]}/{st[24] + st[26]}/{st[25] + st[27]}"
          + f"  |  w0 heads: rows {st[28]}  scan+weights {st[29]}  sums+finish {st[30]}  barrier wait {st[31]}"
          + "  |  staging by kind (grid/PE/colour-static): "
          + "  ".join(f"w{w} {st[32 + 3 * w]}/{st[33 + 3 * w]}/{st[34 + 3 * w]}" for w in range(3))
          + "  |  point geometry w0/w1/w2: " + "/".join(str(st[41 + w]) for w in range(3)))
