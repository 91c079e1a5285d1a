"""Times the texture-export kernels with CUDA events after a warm-up of every shape, next to the reference's ATen search on the same GPU.

- sdfb200_uv_rasterize at 50 000 faces x 2048^2 texels (texture.py's defaults) and 5 000 faces x 1024^2, chunk 10, on random chart
  layouts; face-texel pairs per second = floor(F / 10) * 10 * P over the kernel time.
- The custom unwrap at px_per_uv_triangle=4 over 50 000 faces (sdfb200_uv_unwrap_grid + sdfb200_uv_texel_rays).
- The texel render: SurfaceRenderer.get_outputs_for_camera_ray_bundle (NeuSSampler 64 + 64, fp32 field) over the 1024^2 texel rays.
- The oracle's restatement of the reference's chunk loop (oracle/texture.rasterize, the same ATen ops) on the GPU: at the smaller size in
  full, at the larger over its first ORACLE_CHUNKS chunks, scaled linearly to all 5 000 chunks (labelled "scaled").

Prints one JSON line and writes it to --out.

    python tools/texture_bench.py [--out profiles/r14_texture_bench.json]
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import sdfstudio_b200 as sb  # noqa: E402
from bench_common import cuda_ms, header, report  # noqa: E402
from oracle import texture as otex  # noqa: E402
from sdfstudio_b200 import synthetic, texturing  # noqa: E402
from test_gpu_texture import random_charts  # noqa: E402

CHUNK = 10
ORACLE_CHUNKS = 200


def rasterize_run(n_faces, n, reps):
    uv = random_charts(n_faces, n_faces)
    ms = cuda_ms(lambda: texturing.uv_rasterize(uv, n, CHUNK), reps)
    pairs = n_faces // CHUNK * CHUNK * n * n
    return dict(faces=n_faces, texels=n * n, chunk=CHUNK, kernel_ms=ms, face_texel_pairs=pairs, pairs_per_s=pairs / (ms * 1e-3))


def oracle_run(n_faces, n, chunks):
    uv = random_charts(n_faces, n_faces)
    total = n_faces // CHUNK
    sub = uv[:chunks * CHUNK] if chunks < total else uv
    ms = cuda_ms(lambda: otex.rasterize(sub, n, CHUNK), 1)
    run = dict(faces=n_faces, texels=n * n, chunks_timed=min(chunks, total), chunks_total=total, measured_ms=ms)
    if chunks < total:
        run["scaled_ms"] = ms * total / chunks
        run["scaled"] = f"linear extrapolation from {chunks} of {total} chunks"
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "texture_bench needs a GPU"
    result = header("texture_bench")
    result["rasterize"] = [rasterize_run(50000, 2048, 3), rasterize_run(5000, 1024, 10)]
    ppt, nf = 4, 50000
    g = torch.Generator().manual_seed(0)
    vertices = (torch.rand(nf, 3, generator=g) * 2 - 1).cuda()
    normals = torch.randn(nf, 3, generator=g).cuda()
    faces = torch.randint(0, nf, (nf, 3), generator=g).cuda()

    def custom():
        _, face, bary, _ = texturing.uv_unwrap_grid(nf, ppt, "cuda")
        return texturing.uv_texel_rays(vertices, faces, normals, face, bary, torch.ones((), device="cuda"))

    w, h = texturing.grid_layout(nf, ppt)[2:]
    result["custom_unwrap"] = dict(faces=nf, px_per_uv_triangle=ppt, texels=w * h, ms=cuda_ms(custom, 20))

    face, bary = texturing.uv_rasterize(random_charts(5000, 5000), 1024, CHUNK)
    o, d, fars = texturing.uv_texel_rays(vertices, faces[:5000], normals, face, bary, torch.full((), 0.2, device="cuda"))
    one = torch.ones(o.shape[0], 1, device="cuda")
    bundle = sb.RayBundle(origins=o * 0.5, directions=d, pixel_area=one, camera_indices=0 * one, directions_norm=one, nears=0 * one,
                          fars=fars[:, None])
    cfg = sb.SDFFieldConfig(use_grid_feature=True, num_layers=2, num_layers_color=2, inside_outside=False, bias=0.5, precision="fp32")
    torch.manual_seed(0)
    field = synthetic.perturb_field_(sb.SDFField(cfg, torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), num_images=49), seed=0).cuda().eval()
    renderer = sb.SurfaceRenderer(field, sb.NeuSSampler(num_samples=64, num_samples_importance=64).eval(), kind="neus").eval()
    with torch.no_grad():
        result["texel_render"] = dict(rays=o.shape[0], ms=cuda_ms(lambda: renderer.get_outputs_for_camera_ray_bundle(bundle), 2))

    result["oracle_aten_loop"] = [oracle_run(5000, 1024, 10 ** 9), oracle_run(50000, 2048, ORACLE_CHUNKS)]
    report(result, args.out)


if __name__ == "__main__":
    main()
