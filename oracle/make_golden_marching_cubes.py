"""TEST INFRASTRUCTURE -- mints tests/golden/marching_cubes.npz + marching_cubes.json from the UNMODIFIED reference
nerfstudio/utils/marching_cubes.py on CPU (needs the reference source tree, see oracle/ref_import.py).

skimage, trimesh and pymeshlab are absent here, so stubs stand in: ``skimage.measure.marching_cubes`` records its arguments (volume,
level, spacing, mask) and returns an empty-but-one-vertex mesh at the origin, so that the offset the reference adds afterwards is what
reaches ``trimesh.Trimesh``; trimesh / pymeshlab record and do nothing.  ``torch.Tensor.cuda`` is the identity.

Stored per case: one entry per ``measure.marching_cubes`` call (level, spacing, offset, mask count), and of the volume the values at the
lowest corners of the cubes that cross the level (every ``stride``-th one, the stride chosen to keep the file small) plus one strided
slice.  The three functions' signatures are parsed with ``ast`` from the reference source.

    python -m oracle.make_golden_marching_cubes
"""
import ast
import json
import math
import os
import sys
import types

import numpy as np
import torch

from . import ref_import

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
FUNCTIONS = ("get_surface_sliding", "get_surface_occupancy", "get_surface_sliding_with_contraction")
MAX_CROSSING = 20000


def sphere(c, r):
    c = torch.tensor(c)
    return lambda x: (x - c.to(x)).norm(dim=-1) - r


def torus(R, r):
    return lambda x: torch.sqrt((torch.sqrt(x[:, 0] ** 2 + x[:, 1] ** 2) - R) ** 2 + x[:, 2] ** 2) - r


def union(*fs):
    return lambda x: torch.stack([f(x) for f in fs]).amin(0)


def inv_contract(x):
    """scripts/extract_mesh.py:79-84 with the L2 scene contraction."""
    mag = torch.linalg.norm(x, ord=None, dim=-1)
    mask = mag >= 1
    x_new = x.clone()
    x_new[mask] = (1 / (2 - mag[mask][..., None])) * (x[mask] / mag[mask][..., None])
    return x_new


def coarse_mask_sliding():
    """[16]^3 bool grid over [-1, 1]^3 ('ij' order), set where x < 0.25."""
    g = torch.linspace(-1, 1, 16)
    return (g[:, None, None] < 0.25).expand(16, 16, 16).contiguous()


def coarse_mask_contraction():
    """[1, 1, 32, 32, 32] float visibility grid of the contracted cube, indexed (z, y, x) as grid_sample reads it: set inside radius 1.7
    of the [-2, 2] cube except where z > 1."""
    g = torch.linspace(-2, 2, 32)
    z, y, x = torch.meshgrid(g, g, g, indexing="ij")
    return (((x * x + y * y + z * z) < 1.7**2) & (z <= 1.0)).float()[None, None]


def cases():
    """name -> (function, kwargs without the callable, callable)."""
    return {
        "sliding_512": ("get_surface_sliding", dict(resolution=512), sphere((0.1, -0.05, 0.0), 0.3)),
        "sliding_512_mask": ("get_surface_sliding", dict(resolution=512, coarse_mask=coarse_mask_sliding()), torus(0.45, 0.15)),
        "sliding_1024_partial": ("get_surface_sliding", dict(resolution=1024, bounding_box_min=(-1.0, -1.0, -1.0), bounding_box_max=(1.0, 1.0, 1.2)),
                                 union(sphere((-0.5, -0.5, -0.5), 0.3), sphere((0.6, -0.6, -0.2), 0.5))),
        "contraction_512": ("get_surface_sliding_with_contraction", dict(resolution=512, bounding_box_min=(-2.0, -2.0, -2.0),
                                                                          bounding_box_max=(2.0, 2.0, 2.0), coarse_mask=coarse_mask_contraction(),
                                                                          inv_contraction=inv_contract), sphere((0.0, 0.0, 0.0), 1.2)),
        "occupancy_100": ("get_surface_occupancy", dict(resolution=100, level=0.5),
                          (lambda s: (lambda x: torch.sigmoid(10 * s(x))))(sphere((0.05, 0.0, -0.1), 0.55))),
    }


def crossing_sample(vol, level):
    """(flat indices, values) at the lowest corners of the cubes whose corners straddle `level`, every stride-th one."""
    inside = vol < level
    nx, ny, nz = vol.shape
    anyin = np.zeros((nx - 1, ny - 1, nz - 1), bool)
    allin = np.ones((nx - 1, ny - 1, nz - 1), bool)
    for n in range(8):
        s = inside[n & 1:nx - 1 + (n & 1), (n >> 1) & 1:ny - 1 + ((n >> 1) & 1), (n >> 2) & 1:nz - 1 + ((n >> 2) & 1)]
        anyin |= s
        allin &= s
    i, j, k = np.nonzero(anyin & ~allin)
    idx = (i.astype(np.int64) * ny + j) * nz + k
    stride = max(1, math.ceil(len(idx) / MAX_CROSSING))
    idx = idx[::stride]
    return idx, vol.reshape(-1)[idx]


def signatures():
    src = open(os.path.join(ref_import.REFERENCE_ROOT, "nerfstudio", "utils", "marching_cubes.py")).read()
    out = {}
    for node in ast.parse(src).body:
        if isinstance(node, ast.FunctionDef) and node.name in FUNCTIONS:
            args = node.args.args
            defaults = [None] * (len(args) - len(node.args.defaults)) + list(node.args.defaults)
            out[node.name] = [[a.arg, None if d is None else ast.unparse(d)] for a, d in zip(args, defaults)]
    return out


def install_stubs(calls):
    sk = types.ModuleType("skimage")
    measure = types.ModuleType("skimage.measure")

    def marching_cubes(volume, level, spacing, mask=None):
        calls.append(dict(volume=np.array(volume, dtype=np.float32), level=level, spacing=[float(s) for s in spacing],
                          mask=None if mask is None else np.array(mask, dtype=bool)))
        return np.zeros((1, 3), np.float32), np.zeros((0, 3), np.int64), np.zeros((1, 3), np.float32), None

    measure.marching_cubes = marching_cubes
    sk.measure = measure
    sys.modules["skimage"], sys.modules["skimage.measure"] = sk, measure

    tm = types.ModuleType("trimesh")

    class Trimesh:
        def __init__(self, vertices, faces, vertex_normals=None):
            self.vertices = np.asarray(vertices, dtype=np.float64)
            if calls and "offset" not in calls[-1] and len(self.vertices) == 1:
                calls[-1]["offset"] = self.vertices[0].tolist()

        def merge_vertices(self, digits_vertex=None):
            pass

        def export(self, path):
            pass

    util = types.SimpleNamespace(concatenate=lambda meshes: Trimesh(np.concatenate([m.vertices for m in meshes]) if meshes else np.zeros((0, 3)), None))
    tm.Trimesh, tm.util = Trimesh, util
    sys.modules["trimesh"] = tm

    pm = types.ModuleType("pymeshlab")

    class MeshSet:
        def __getattr__(self, name):
            return lambda *a, **k: None

    pm.MeshSet = MeshSet
    sys.modules["pymeshlab"] = pm


def main():
    ref_import.install_shims()
    calls = []
    install_stubs(calls)
    torch.Tensor.cuda = lambda self, *a, **k: self
    import nerfstudio.utils.marching_cubes as ref_mc

    arrays, meta = {}, {"signatures": signatures(), "cases": {}}
    for name, (fn, kw, f) in cases().items():
        calls.clear()
        key = "occupancy_fn" if fn == "get_surface_occupancy" else "sdf"
        getattr(ref_mc, fn)(**{key: f}, **kw, output_path=__import__("pathlib").Path(os.devnull + ".ply"),
                            **({} if fn == "get_surface_occupancy" else {"simplify_mesh": False}))
        entries = []
        for n, c in enumerate(calls):
            vol = c["volume"]
            idx, val = crossing_sample(vol, np.float32(c["level"]))
            arrays[f"{name}/{n}/cross_idx"] = idx
            arrays[f"{name}/{n}/cross_val"] = val
            mid = vol.shape[0] // 2
            arrays[f"{name}/{n}/slice"] = vol[mid, ::4, ::4]
            entries.append(dict(level=float(c["level"]), spacing=c["spacing"], offset=c["offset"], shape=list(vol.shape),
                                mask_count=None if c["mask"] is None else int(c["mask"].sum())))
        meta["cases"][name] = entries
        print(name, [(e["offset"], e["mask_count"]) for e in entries], flush=True)
    np.savez_compressed(os.path.join(GOLDEN_DIR, "marching_cubes.npz"), **arrays)
    with open(os.path.join(GOLDEN_DIR, "marching_cubes.json"), "w") as fh:
        json.dump(meta, fh, indent=1)


if __name__ == "__main__":
    main()
