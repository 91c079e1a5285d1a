"""TEST INFRASTRUCTURE -- mints tests/golden/texture.npz + texture.json from the UNMODIFIED reference
nerfstudio/exporter/texture_utils.py on CPU (needs the reference source tree, see oracle/ref_import.py).

mediapy, xatlas, pymeshlab, open3d and the reference's Pipeline module are absent or unusable here, so stubs stand in:
``mediapy.write_image`` captures the image it is given; ``xatlas.parametrize`` returns the case's per-corner UVs (``uvs`` [3F,2],
``indices`` [F,3] = 0..3F-1); ``pymeshlab``, ``open3d`` and ``nerfstudio.pipelines.base_pipeline`` are empty modules.
``export_textured_mesh`` runs with a fake pipeline whose model records the RayBundle it receives and returns a fixed colour function of
the rays, so the golden pins the texel bundle, the image handed to mediapy and the OBJ / MTL text.

    python -m oracle.make_golden_texture
"""
import json
import os
import sys
import tempfile
import types
from pathlib import Path

import numpy as np
import torch

from . import ref_import

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
BUNDLE_FIELDS = ("origins", "directions", "pixel_area", "camera_indices", "directions_norm", "nears", "fars")


def colour(origins, directions, fars):
    """The fake model's rgb: a smooth function of every bundle field the texture depends on."""
    return torch.sigmoid(1.3 * origins + 0.7 * directions + 0.1 * fars)


def mesh(seed, n_vertices, n_faces):
    g = torch.Generator().manual_seed(seed)
    vertices = torch.rand(n_vertices, 3, generator=g) * 2 - 1
    faces = torch.stack([torch.randperm(n_vertices, generator=g)[:3] for _ in range(n_faces)])
    normals = torch.randn(n_vertices, 3, generator=g)
    return vertices, faces, normals


def chart_uvs(seed, n_faces, cells, n):
    """[F,3,2] fp32 UVs: face i is a random triangle inside cell i of a cells x cells grid of [0.05, 0.95]^2 (unused cells and the margin
    hold texels outside every chart)."""
    g = torch.Generator().manual_seed(seed)
    size = 0.9 / cells
    cell = torch.arange(n_faces)
    lo = torch.stack([cell % cells, cell // cells], dim=-1).float() * size + 0.05
    return (lo[:, None, :] + torch.rand(n_faces, 3, 2, generator=g) * size * 1.2).float()


def overlap_uvs(n):
    """20 faces of chart_uvs plus: faces 4 and 5 identical (a tie inside chunk 0), face 15 a copy of face 3 (a tie across chunks), face 12
    a zero-area triangle along the centre row 10 of the texture (0/0 = NaN for the texels on that row: chunk 1 yields nothing there) with
    face 13 a large triangle over that row."""
    uv = chart_uvs(5, 20, 5, n)
    uv[5] = uv[4]
    uv[15] = uv[3]
    row = torch.linspace(0.5 / n, 1 - 0.5 / n, n)[10]
    uv[12] = torch.tensor([[0.1, 0.0], [0.5, 0.0], [0.9, 0.0]]) + torch.tensor([0.0, 1.0]) * row
    uv[13] = torch.tensor([[0.05, 0.2], [0.95, 0.25], [0.5, 0.6]])
    return uv.float()


def cases():
    """name -> (mesh seed, V, F, export kwargs, per-corner UVs or None)."""
    return {
        "custom_odd": (0, 12, 13, dict(unwrap_method="custom", px_per_uv_triangle=4), None),
        "custom_none": (1, 9, 8, dict(unwrap_method="custom", px_per_uv_triangle=3, raylen_method="none"), None),
        "xatlas_30": (2, 25, 30, dict(num_pixels_per_side=40), chart_uvs(2, 30, 6, 40)),
        "xatlas_37": (3, 30, 37, dict(num_pixels_per_side=48), chart_uvs(3, 37, 7, 48)),
        "xatlas_7": (4, 10, 7, dict(num_pixels_per_side=16), chart_uvs(4, 7, 3, 16)),
        "xatlas_overlap": (5, 16, 20, dict(num_pixels_per_side=32), overlap_uvs(32)),
        "xatlas_none": (6, 20, 24, dict(num_pixels_per_side=24, raylen_method="none"), chart_uvs(6, 24, 5, 24)),
    }


def install_stubs(state):
    media = types.ModuleType("mediapy")
    media.write_image = lambda path, image: state.__setitem__("image", np.array(image, dtype=np.float32))
    sys.modules["mediapy"] = media

    xatlas = types.ModuleType("xatlas")

    def parametrize(vertices, faces, normals):
        uv = state["uvs"].numpy().reshape(-1, 2)
        return np.arange(len(uv), dtype=np.uint32), np.arange(len(uv), dtype=np.uint32).reshape(-1, 3), uv

    xatlas.parametrize = parametrize
    sys.modules["xatlas"] = xatlas

    pm = types.ModuleType("pymeshlab")
    pm.Mesh = type("Mesh", (), {})
    pm.MeshSet = type("MeshSet", (), {})
    sys.modules["pymeshlab"] = pm
    sys.modules["open3d"] = types.ModuleType("open3d")
    bp = types.ModuleType("nerfstudio.pipelines.base_pipeline")
    bp.Pipeline = type("Pipeline", (), {})
    sys.modules["nerfstudio.pipelines.base_pipeline"] = bp
    sys.modules["nerfstudio.configs.base_config"].Config = type("Config", (), {})


class FakeModel:
    def __init__(self, state):
        self.state = state

    def get_outputs_for_camera_ray_bundle(self, bundle):
        self.state["bundle"] = {k: getattr(bundle, k).clone() for k in BUNDLE_FIELDS}
        return {"rgb": colour(bundle.origins, bundle.directions, bundle.fars)}


def main():
    ref_import.install_shims()
    state = {}
    install_stubs(state)
    from nerfstudio.exporter import texture_utils

    pipeline = types.SimpleNamespace(device=torch.device("cpu"), model=FakeModel(state))
    arrays, meta = {}, {"cases": {}}
    for name, (seed, nv, nf, kw, uvs) in cases().items():
        vertices, faces, normals = mesh(seed, nv, nf)
        state.clear()
        state["uvs"] = uvs
        ref_mesh = types.SimpleNamespace(vertices=vertices, faces=faces, normals=normals)
        with tempfile.TemporaryDirectory() as d:
            texture_utils.export_textured_mesh(ref_mesh, pipeline, Path(d), **kw)
            obj = (Path(d) / "mesh.obj").read_text()
            mtl = (Path(d) / "material_0.mtl").read_text()
        arrays[f"{name}/vertices"], arrays[f"{name}/faces"], arrays[f"{name}/normals"] = vertices.numpy(), faces.numpy(), normals.numpy()
        if uvs is not None:
            arrays[f"{name}/uvs"] = uvs.numpy()
        for k, v in state["bundle"].items():
            arrays[f"{name}/{k}"] = v.numpy()
        arrays[f"{name}/image"] = state["image"]
        meta["cases"][name] = dict(kwargs=kw, obj=obj, mtl=mtl, shape=list(state["image"].shape))
        print(name, state["image"].shape, flush=True)
    np.savez_compressed(os.path.join(GOLDEN_DIR, "texture.npz"), **arrays)
    with open(os.path.join(GOLDEN_DIR, "texture.json"), "w") as fh:
        json.dump(meta, fh, indent=1)


if __name__ == "__main__":
    main()
