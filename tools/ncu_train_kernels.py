"""Driver for ncu captures of the training-step kernels at the angelo-train-8192 shapes: grouped grid forward / table-gradient scatter
(7 taps per sample, ray-coherent samples, 2.1 GB table, 8 of 16 levels active), tensor-core forward GEMM + weight-gradient GEMM.  Run under
    ncu --set full --clock-control none -k regex:'k_grid_encode_grouped|k_grid_encode_bwd_grouped|k_tc_wgrad|k_tc_linear' -c 8 -o gpurun_out/r02_train python tools/ncu_train_kernels.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import sdfstudio_b200 as sb  # noqa: E402
from sdfstudio_b200 import linear_ops as lo  # noqa: E402
from sdfstudio_b200.synthetic import dtu_like_rays  # noqa: E402

dev = torch.device("cuda")
torch.manual_seed(0)
R, S = 8192, 48
o, d, cam, nears, fars = dtu_like_rays(R, 5)
t = nears + (fars - nears) * (torch.arange(S) + 0.5)[None] / S
x = (o[:, None] + d[:, None] * t[..., None]).reshape(-1, 3).to(dev)                     # [R*S, 3] in the scene box
delta = 1.0 / 4096.0
offs = torch.tensor([[0, 0, 0], [delta, 0, 0], [-delta, 0, 0], [0, delta, 0], [0, -delta, 0], [0, 0, delta], [0, 0, -delta]], device=dev)
pts = ((x[None] + offs[:, None, :]).reshape(-1, 3) + 2.0) / 4.0
enc = sb.HashEncoding(num_levels=16, min_res=64, max_res=4096, log2_hashmap_size=22, features_per_level=8).to(dev)
enc.set_active_levels(8)
with enc.point_groups(7):
    out = enc(pts)                                                                         # k_grid_encode_grouped
out.backward(torch.randn_like(out))                                                        # k_grid_encode_bwd_grouped
torch.cuda.synchronize()
N = pts.shape[0]
xin = torch.randn(N, 176, device=dev)
W = torch.randn(256, 167, device=dev, requires_grad=True)
b = torch.zeros(256, device=dev, requires_grad=True)
y = lo.linear(xin, W, b, 1, "bf16x3")                                                      # k_tc_linear (softplus epilogue)
y.backward(torch.randn_like(y))                                                            # k_tc_wgrad (+ reduce)
torch.cuda.synchronize()
print("done", N)
