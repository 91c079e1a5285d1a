"""TEST INFRASTRUCTURE -- mints tests/golden/pointcloud.npz + pointcloud.json from the UNMODIFIED reference
nerfstudio/exporter/exporter_utils.py (generate_point_cloud) on CPU (needs the reference source tree, see oracle/ref_import.py).

open3d, pymeshlab and the reference's Pipeline module are absent here, so stubs stand in: the open3d stub's ``PointCloud`` records the
arrays it is given, its ``remove_statistical_outlier`` records (nb_neighbors, std_ratio) and keeps the fixed subset ``stub_kept`` (so
that the masking of the normals is pinned), and ``estimate_normals`` records the call.  The pipeline is ``oracle.pointcloud.FakePipeline``
with the reference's own RayBundle.

    python -m oracle.make_golden_pointcloud
"""
import dataclasses
import importlib.util
import json
import os
import sys
import types

import numpy as np
import torch

from . import ref_import
from .make_golden_tsdf import describe_default
from .pointcloud import FakePipeline

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

# name -> (FakePipeline arguments, generate_point_cloud arguments)
CASES = {
    # 1500 points from batches of 1000 rays (about 360 kept per batch), every third batch keeping nothing; normals masked
    "normals_masked": (dict(n=1000, seed=1, miss_every=3), dict(num_points=1500, normal_output_name="normal")),
    "estimate": (dict(n=800, seed=2), dict(num_points=700, estimate_normals=True, std_ratio=2.5)),
    "no_outliers": (dict(n=600, seed=3), dict(num_points=900, remove_outliers=False, normal_output_name="normal")),
    "no_box": (dict(n=500, seed=4), dict(num_points=1200, use_bounding_box=False, remove_outliers=False)),
    "no_box_estimate": (dict(n=500, seed=5), dict(num_points=400, use_bounding_box=False, estimate_normals=True)),
    "small_box": (dict(n=700, seed=6), dict(num_points=250, bounding_box_min=(-0.1, -0.6, -0.3), bounding_box_max=(0.7, 0.2, 0.6))),
    "zero_points": (dict(n=300, seed=7), dict(num_points=0)),
}
ERRORS = {
    "missing_rgb": (dict(n=100, seed=8), dict(rgb_output_name="colour")),
    "missing_depth": (dict(n=100, seed=8), dict(depth_output_name="z")),
    "missing_normal": (dict(n=100, seed=8), dict(normal_output_name="normals")),
    "estimate_and_normal_output": (dict(n=400, seed=9), dict(num_points=300, estimate_normals=True, normal_output_name="normal")),
}


def stub_kept(n: int):
    """The indices the open3d stub's remove_statistical_outlier keeps out of n: every i with i % 3 != 1."""
    return [i for i in range(n) if i % 3 != 1]


def install_stubs(state):
    o3d = types.ModuleType("open3d")
    o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.array(a, dtype=np.float64))

    class PointCloud:
        def __init__(self):
            self.points, self.colors, self.normals = None, None, None

        def remove_statistical_outlier(self, nb_neighbors, std_ratio):
            state["outlier_args"] = [nb_neighbors, std_ratio]
            state["outlier_input"] = (self.points.copy(), self.colors.copy())
            ind = stub_kept(len(self.points))
            out = PointCloud()
            out.points, out.colors = self.points[ind], self.colors[ind]
            return out, ind

        def estimate_normals(self):
            state["estimated"] = True

    o3d.geometry = types.SimpleNamespace(PointCloud=PointCloud)
    sys.modules["open3d"] = o3d
    sys.modules["pymeshlab"] = types.ModuleType("pymeshlab")
    bp = types.ModuleType("nerfstudio.pipelines.base_pipeline")
    bp.Pipeline = type("Pipeline", (), {})
    sys.modules["nerfstudio.pipelines.base_pipeline"] = bp
    ev = types.ModuleType("nerfstudio.utils.eval_utils")
    ev.eval_setup = None
    sys.modules["nerfstudio.utils.eval_utils"] = ev
    for name in ("mediapy", "xatlas", "skimage", "skimage.measure"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["nerfstudio.configs.base_config"].Config = type("Config", (), {})


def main():
    ref_import.install_shims()
    state = {}
    install_stubs(state)
    from nerfstudio.cameras.rays import RayBundle
    from nerfstudio.exporter import exporter_utils

    spec = importlib.util.spec_from_file_location("ref_exporter_script", os.path.join(ref_import.REFERENCE_ROOT, "scripts", "exporter.py"))
    exporter = sys.modules[spec.name] = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(exporter)

    def bundle(origins, directions):
        return RayBundle(origins=origins, directions=directions, pixel_area=torch.ones(origins.shape[0], 1))

    arrays, meta = {}, {"cases": {}, "errors": {}}
    for name, (pk, gk) in CASES.items():
        state.clear()
        pipeline = FakePipeline(bundle_cls=bundle, **pk)
        pcd = exporter_utils.generate_point_cloud(pipeline, **gk)
        arrays[f"{name}/points"], arrays[f"{name}/colors"] = pcd.points.astype(np.float32), pcd.colors.astype(np.float32)
        if pcd.normals is not None:
            arrays[f"{name}/normals"] = pcd.normals.astype(np.float32)
        if "outlier_input" in state:
            arrays[f"{name}/outlier_points"], arrays[f"{name}/outlier_colors"] = (a.astype(np.float32) for a in state["outlier_input"])
        meta["cases"][name] = dict(pipeline=pk, kwargs=gk, batches=pipeline.datamanager.calls, outlier_args=state.get("outlier_args"),
                                   estimated=state.get("estimated", False), n_points=len(pcd.points))
        print(name, meta["cases"][name], flush=True)
    for name, (pk, gk) in ERRORS.items():
        pipeline = FakePipeline(bundle_cls=bundle, outputs=("rgb", "depth", "normal"), **pk)
        try:
            exporter_utils.generate_point_cloud(pipeline, **gk)
            raise AssertionError(f"{name} did not fail")
        except SystemExit as e:
            meta["errors"][name] = dict(pipeline=pk, kwargs=gk, exit_code=e.code, batches=pipeline.datamanager.calls)
    try:
        exporter_utils.generate_point_cloud(FakePipeline(n=50, seed=10, bundle_cls=bundle), bounding_box_min=(0, 0, 0), bounding_box_max=(1, 0, 1))
    except AssertionError as e:
        meta["errors"]["box_min_not_below_max"] = dict(message=str(e))
    print(meta["errors"], flush=True)

    meta["signatures"] = {
        "generate_point_cloud": [[p.name, describe_default(p.default)]
                                 for p in __import__("inspect").signature(exporter_utils.generate_point_cloud).parameters.values()],
        "ExportPointCloud": [[f.name, describe_default(f.default_factory() if f.default_factory is not dataclasses.MISSING else f.default)]
                             for f in dataclasses.fields(exporter.ExportPointCloud)],
    }
    np.savez_compressed(os.path.join(GOLDEN_DIR, "pointcloud.npz"), **arrays)
    with open(os.path.join(GOLDEN_DIR, "pointcloud.json"), "w") as fh:
        json.dump(meta, fh, indent=1)


if __name__ == "__main__":
    main()
