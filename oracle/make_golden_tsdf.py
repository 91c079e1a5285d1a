"""TEST INFRASTRUCTURE -- mints tests/golden/tsdf.npz + tsdf.json from the UNMODIFIED reference nerfstudio/exporter/tsdf_utils.py on
CPU (needs the reference source tree, see oracle/ref_import.py).

skimage, pymeshlab, open3d, mediapy, xatlas and the reference's Pipeline module are absent or unusable here, so stubs stand in:
``skimage.measure.marching_cubes`` records the volume it is given and returns fixed vertices (some with .5 coordinates, to pin the
rounding of the colour gather); ``pymeshlab.Mesh`` / ``MeshSet`` record the matrices and the file name; the others are empty modules.
``export_tsdf_mesh`` runs with a fake pipeline that holds real reference ``Cameras`` and a model whose rgb and depth come from an
analytic sphere.

    python -m oracle.make_golden_tsdf
"""
import dataclasses
import importlib.util
import inspect
import json
import os
import sys
import types
from pathlib import Path

import numpy as np
import torch

from . import ref_import

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
SPHERE_CENTRE, SPHERE_RADIUS = torch.tensor([0.1, -0.05, 0.0]), 0.55


def sphere_hit(origins, directions):
    """(depth along the ray to the sphere or 0 on a miss, rgb = 0.5 + 0.5 normal there, 0 on a miss) for rays [..., 3]."""
    d = directions / directions.norm(dim=-1, keepdim=True)
    oc = origins - SPHERE_CENTRE
    b = (oc * d).sum(-1)
    disc = b * b - ((oc * oc).sum(-1) - SPHERE_RADIUS**2)
    t = -b - torch.sqrt(disc.clamp(min=0))
    hit = (disc > 0) & (t > 0)
    depth = torch.where(hit, t, torch.zeros_like(t))
    n = (origins + t[..., None] * d - SPHERE_CENTRE) / SPHERE_RADIUS
    return depth, torch.where(hit[..., None], 0.5 + 0.5 * n, torch.zeros_like(n))


def look_at(positions, target=(0.0, 0.0, 0.0)):
    """[C,4,4] OpenGL camera-to-world (camera looks down -z, y up)."""
    p = torch.as_tensor(positions, dtype=torch.float32)
    back = p - torch.tensor(target)
    back = back / back.norm(dim=-1, keepdim=True)
    up0 = torch.tensor([0.0, 0.0, 1.0]).expand_as(back)
    right = torch.cross(up0, back, dim=-1)
    right = right / right.norm(dim=-1, keepdim=True)
    up = torch.cross(back, right, dim=-1)
    c2w = torch.zeros(len(p), 4, 4)
    c2w[:, :3, 0], c2w[:, :3, 1], c2w[:, :3, 2], c2w[:, :3, 3], c2w[:, 3, 3] = right, up, back, p, 1.0
    return c2w


def pixel_rays(c2w, K, H, W):
    """World-space (origins, directions) [C,H,W,3] through the pixel centres."""
    j, i = torch.meshgrid(torch.arange(W) + 0.5, torch.arange(H) + 0.5, indexing="xy")
    dirs = []
    for c in range(len(c2w)):
        d = torch.stack([(j - K[c, 0, 2]) / K[c, 0, 0], -(i - K[c, 1, 2]) / K[c, 1, 1], -torch.ones_like(j)], dim=-1)
        dirs.append(d @ c2w[c, :3, :3].T)
    d = torch.stack(dirs)
    return c2w[:, None, None, :3, 3].expand_as(d), d


def intrinsics(C, f, H, W):
    K = torch.zeros(C, 3, 3)
    K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = f, f * 1.05, W / 2 + 0.3, H / 2 - 0.2, 1.0
    return K


def sphere_images(c2w, K, H, W, seed, noise=0.02):
    """depth [C,1,H,W] and colour [C,3,H,W] of the sphere, with seeded noise, a band of zeros, NaNs and infinities."""
    g = torch.Generator().manual_seed(seed)
    o, d = pixel_rays(c2w, K, H, W)
    depth, rgb = sphere_hit(o, d)
    depth = depth + noise * torch.randn(depth.shape, generator=g) * (depth > 0)
    depth = torch.where(depth > 0, depth, torch.zeros_like(depth))
    r = torch.rand(depth.shape, generator=g)
    depth = torch.where(r < 0.03, torch.full_like(depth, float("nan")), depth)
    depth = torch.where((r > 0.97) & (depth > 0), torch.full_like(depth, float("inf")), depth)
    depth[:, H // 3, :] = 0.0
    rgb = (rgb + 0.1 * torch.rand(rgb.shape, generator=g)).clamp(0, 1)
    return depth[:, None].contiguous(), rgb.permute(0, 3, 1, 2).contiguous()


def on_sphere(n, radius, seed):
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(n, 3, generator=g)
    return radius * v / v.norm(dim=-1, keepdim=True)


def cases():
    """name -> (aabb [2,3], volume dims [3], c2w [C,4,4], K [C,3,3], depth [C,1,H,W], colour [C,3,H,W], batch size)."""
    out = {}
    # cameras outside the volume, a narrow field of view (pixels out of bounds), 24 x 32 images, batches of 10 (10 + 3)
    c2w = look_at(on_sphere(13, 3.0, 1))
    K = intrinsics(13, 1.2 * 32, 24, 32)
    out["outside_b10"] = (torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), torch.tensor([16, 16, 16]), c2w, K, *sphere_images(c2w, K, 24, 32, 2), 10)
    # cameras inside a non-cubic 7 x 33 x 64 volume (voxels behind them), random depths with zeros, batches of 3 (3 + 3 + 1)
    g = torch.Generator().manual_seed(3)
    pos = torch.tensor([0.1, 0.2, 0.3]) + 0.2 * torch.randn(7, 3, generator=g)
    c2w = look_at(pos, target=(0.4, -0.3, 0.5))
    c2w[:4] = look_at(pos[:4], target=(-0.5, 0.6, -0.2))
    K = intrinsics(7, 9.0, 20, 20)
    depth = 0.2 + 2.3 * torch.rand(7, 1, 20, 20, generator=g)
    depth[torch.rand(depth.shape, generator=g) < 0.1] = 0.0
    depth[torch.rand(depth.shape, generator=g) < 0.05] = float("nan")
    colour = torch.rand(7, 3, 20, 20, generator=g)
    out["inside_b3"] = (torch.tensor([[-1.0, -0.8, -0.6], [0.9, 1.1, 1.3]]), torch.tensor([7, 33, 64]), c2w, K, depth, colour, 3)
    # 1 x 1 images, batches of 1
    c2w = look_at(on_sphere(5, 2.5, 4))
    K = intrinsics(5, 0.4, 1, 1)
    g = torch.Generator().manual_seed(5)
    depth = torch.tensor([2.4, 2.0, 0.0, 2.6, float("nan")]).view(5, 1, 1, 1)
    out["tiny_b1"] = (torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), torch.tensor([9, 9, 9]), c2w, K, depth, torch.rand(5, 3, 1, 1, generator=g), 1)
    return out


# ---------------------------------------------------------------------------------------------------------------------------------
# stubs
# ---------------------------------------------------------------------------------------------------------------------------------
MC_VERTICES = np.array([[0.5, 1.5, 2.5], [2.5, 0.5, 1.0], [1.49, 3.5, 4.51], [0.0, 0.0, 0.0], [3.5, 2.5, 1.5], [4.0, 4.5, 5.5]],
                       dtype=np.float32)
MC_FACES = np.array([[0, 1, 2], [2, 3, 4], [1, 4, 5]], dtype=np.int32)
MC_NORMALS = np.array([[0.0, 0.0, 1.0], [0.0, 1.0, 0.0], [1.0, 0.0, 0.0], [0.6, 0.8, 0.0], [0.0, 0.6, 0.8], [0.8, 0.0, 0.6]],
                      dtype=np.float32)


def install_stubs(state):
    skimage = types.ModuleType("skimage")
    measure = types.ModuleType("skimage.measure")

    def marching_cubes(volume, level, allow_degenerate):
        state["mc"] = dict(volume=np.array(volume), level=level, allow_degenerate=allow_degenerate)
        return MC_VERTICES.copy(), MC_FACES.copy(), MC_NORMALS.copy(), np.zeros(len(MC_VERTICES), np.float32)

    measure.marching_cubes = marching_cubes
    skimage.measure = measure
    sys.modules["skimage"], sys.modules["skimage.measure"] = skimage, measure

    pm = types.ModuleType("pymeshlab")

    class Mesh:
        def __init__(self, **kw):
            state["pymeshlab_mesh"] = {k: np.array(v) for k, v in kw.items()}

    class MeshSet:
        def add_mesh(self, m, name):
            state["pymeshlab_name"] = name

        def save_current_mesh(self, filename):
            state["pymeshlab_file"] = filename

    pm.Mesh, pm.MeshSet = Mesh, MeshSet
    sys.modules["pymeshlab"] = pm
    for name in ("open3d", "mediapy", "xatlas"):
        sys.modules[name] = types.ModuleType(name)
    bp = types.ModuleType("nerfstudio.pipelines.base_pipeline")
    bp.Pipeline = type("Pipeline", (), {})
    sys.modules["nerfstudio.pipelines.base_pipeline"] = bp
    ev = types.ModuleType("nerfstudio.utils.eval_utils")
    ev.eval_setup = None
    sys.modules["nerfstudio.utils.eval_utils"] = ev
    sys.modules["nerfstudio.configs.base_config"].Config = type("Config", (), {})


class FakeModel:
    def get_outputs_for_camera_ray_bundle(self, bundle):
        depth, rgb = sphere_hit(bundle.origins, bundle.directions)
        return {"rgb": rgb, "depth": depth[..., None], "accumulation": (depth > 0).float()[..., None]}


# export flow: real reference Cameras, 41 x 31 pixels rendered at downscale 2 (20 x 15 after truncation)
FLOW = dict(n=6, width=41, height=31, f=36.7, downscale_factor=2, resolution=[12, 10, 14], batch_size=4)


def fake_pipeline(cameras_cls, camera_type):
    c2w = look_at(on_sphere(FLOW["n"], 2.2, 6))[:, :3, :]
    n = FLOW["n"]
    cams = cameras_cls(camera_to_worlds=c2w, fx=torch.full((n, 1), FLOW["f"]), fy=torch.full((n, 1), FLOW["f"] * 0.97),
                       cx=torch.full((n, 1), FLOW["width"] / 2 + 0.25), cy=torch.full((n, 1), FLOW["height"] / 2 - 0.5),
                       width=torch.full((n, 1), FLOW["width"]), height=torch.full((n, 1), FLOW["height"]), camera_type=camera_type)
    outputs = types.SimpleNamespace(cameras=cams, scene_box=types.SimpleNamespace(aabb=torch.tensor([[-1.5, -1.5, -1.5], [1.5, 1.5, 1.5]])))
    dm = types.SimpleNamespace(train_dataset=types.SimpleNamespace(_dataparser_outputs=outputs))
    return types.SimpleNamespace(device=torch.device("cpu"), datamanager=dm, model=FakeModel()), c2w


def describe_default(v):
    if v is inspect.Parameter.empty or v is dataclasses.MISSING:
        return {"required": True}
    if isinstance(v, dataclasses.Field):
        return {"field_default_factory": v.default_factory()}
    return {"default": list(v) if isinstance(v, tuple) else v}


def signatures(tsdf_utils, exporter):
    sig = {}
    sig["TSDF"] = {"fields": [[f.name, describe_default(f.default)] for f in dataclasses.fields(tsdf_utils.TSDF)],
                   "members": sorted(k for k in vars(tsdf_utils.TSDF) if not k.startswith("__")),
                   "export_mesh_is_classmethod": isinstance(vars(tsdf_utils.TSDF)["export_mesh"], classmethod),
                   "from_aabb_is_staticmethod": isinstance(vars(tsdf_utils.TSDF)["from_aabb"], staticmethod),
                   "integrate_tsdf": [[p.name, describe_default(p.default)] for p in inspect.signature(tsdf_utils.TSDF.integrate_tsdf).parameters.values()]}
    sig["export_tsdf_mesh"] = [[p.name, describe_default(p.default)] for p in inspect.signature(tsdf_utils.export_tsdf_mesh).parameters.values()]
    fields = []
    for f in dataclasses.fields(exporter.ExportTSDFMesh):
        d = f.default_factory() if f.default_factory is not dataclasses.MISSING else f.default
        fields.append([f.name, describe_default(d)])
    sig["ExportTSDFMesh"] = fields
    return sig


def main():
    ref_import.install_shims()
    state = {}
    install_stubs(state)
    from nerfstudio.cameras.cameras import Cameras, CameraType
    from nerfstudio.exporter import tsdf_utils

    spec = importlib.util.spec_from_file_location("ref_exporter_script", os.path.join(ref_import.REFERENCE_ROOT, "scripts", "exporter.py"))
    exporter = sys.modules[spec.name] = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(exporter)

    arrays, meta = {}, {"cases": {}, "signatures": signatures(tsdf_utils, exporter)}
    for name, (aabb, dims, c2w, K, depth, colour, bs) in cases().items():
        t = tsdf_utils.TSDF.from_aabb(aabb, volume_dims=dims)
        for k in ("voxel_coords", "voxel_size", "origin", "values", "weights", "colors"):
            arrays[f"{name}/init_{k}"] = getattr(t, k).numpy().copy()
        for i in range(0, len(c2w), bs):
            t.integrate_tsdf(c2w[i:i + bs], K[i:i + bs], depth[i:i + bs], color_images=colour[i:i + bs])
        for k, v in dict(aabb=aabb, dims=dims, c2w=c2w, K=K, depth=depth, color=colour).items():
            arrays[f"{name}/{k}"] = v.numpy()
        for k in ("values", "weights", "colors"):
            arrays[f"{name}/{k}"] = t.values.numpy() if k == "values" else getattr(t, k).numpy()
        meta["cases"][name] = dict(batch_size=bs, truncation=float(t.truncation), truncation_margin=t.truncation_margin,
                                   weights_set=int((t.weights > 0).sum()))
        # get_mesh on the fused volume: the volume skimage receives, the world vertices and the gathered colours
        if name == "outside_b10":
            mesh = t.get_mesh()
            arrays[f"{name}/mc_volume"] = state["mc"]["volume"]
            meta["cases"][name]["mc_args"] = dict(level=state["mc"]["level"], allow_degenerate=state["mc"]["allow_degenerate"])
            arrays[f"{name}/mesh_vertices"], arrays[f"{name}/mesh_colors"] = mesh.vertices.numpy(), mesh.colors.numpy()
            arrays[f"{name}/mesh_faces"], arrays[f"{name}/mesh_normals"] = mesh.faces.numpy(), mesh.normals.numpy()
            tsdf_utils.TSDF.export_mesh(mesh, "mesh.ply")
            for k, v in state["pymeshlab_mesh"].items():
                arrays[f"{name}/pymeshlab_{k}"] = v
        print(name, meta["cases"][name], flush=True)
    arrays["mc_vertices"], arrays["mc_faces"], arrays["mc_normals"] = MC_VERTICES, MC_FACES, MC_NORMALS

    # the whole export_tsdf_mesh flow, recording what reaches integrate_tsdf
    calls = []
    original = tsdf_utils.TSDF.integrate_tsdf

    def recording(self, c2w, K, depth_images, color_images=None, mask_images=None):
        calls.append((c2w.clone(), K.clone(), depth_images.clone(), color_images.clone()))
        return original(self, c2w, K, depth_images, color_images, mask_images)

    tsdf_utils.TSDF.integrate_tsdf = recording
    pipeline, c2w = fake_pipeline(Cameras, CameraType.PERSPECTIVE)
    state.clear()
    tsdf_utils.export_tsdf_mesh(pipeline, Path("out"), downscale_factor=FLOW["downscale_factor"], resolution=FLOW["resolution"],
                                batch_size=FLOW["batch_size"])
    arrays["flow/c2w_in"] = c2w.numpy()
    for k, i in (("c2w", 0), ("K", 1), ("depth", 2), ("color", 3)):
        arrays[f"flow/{k}"] = torch.cat([c[i] for c in calls]).numpy()
    arrays["flow/mc_volume"] = state["mc"]["volume"]
    for k, v in state["pymeshlab_mesh"].items():
        arrays[f"flow/pymeshlab_{k}"] = v
    cams = pipeline.datamanager.train_dataset._dataparser_outputs.cameras
    meta["flow"] = dict(FLOW, calls=[len(c[0]) for c in calls], image_hw=list(calls[0][2].shape[-2:]), file=state["pymeshlab_file"],
                        rescaled_width=cams.width.view(-1).tolist(), rescaled_height=cams.height.view(-1).tolist())
    tsdf_utils.TSDF.integrate_tsdf = original
    # the omitted resolution (a dataclasses.Field default) and a tuple raise before anything is rendered
    errors = {}
    for label, kw in (("omitted", {}), ("tuple", dict(resolution=(8, 8, 8)))):
        pipeline, _ = fake_pipeline(Cameras, CameraType.PERSPECTIVE)
        try:
            tsdf_utils.export_tsdf_mesh(pipeline, Path("out"), **kw)
            errors[label] = None
        except ValueError as e:
            errors[label] = str(e)
    meta["resolution_errors"] = errors
    print(meta["flow"], errors, flush=True)

    np.savez_compressed(os.path.join(GOLDEN_DIR, "tsdf.npz"), **arrays)
    with open(os.path.join(GOLDEN_DIR, "tsdf.json"), "w") as fh:
        json.dump(meta, fh, indent=1)


if __name__ == "__main__":
    main()
