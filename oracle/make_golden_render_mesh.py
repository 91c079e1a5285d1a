"""TEST INFRASTRUCTURE -- mints tests/golden/render_mesh.npz + render_mesh.json from the UNMODIFIED reference scripts/render_mesh.py and
nerfstudio/cameras/camera_paths.py on CPU (needs the reference source tree, see oracle/ref_import.py).

open3d, mediapy, cv2, zmq and the data-manager modules are stubbed.  The open3d stub's visualizer runs the script's animation callback
until it unregisters itself; ``capture_screen_image`` records the file name and the render option it was taken with, and the cv2 stub's
``imread`` returns a fixed BGR image per (output, frame), so the frames the mediapy stub receives pin the merge layout.  Recorded:
RenderTrajectory's fields and defaults, scripts/render.json, the spiral, ellipse, interpolate and JSON camera paths for fixed camera sets,
three_js_perspective_camera_focal_length, the merged frames of "half" and "concat" and the PNG paths.

    python -m oracle.make_golden_render_mesh
"""
import dataclasses
import importlib.util
import json
import os
import sys
import tempfile
import types
from pathlib import Path

import numpy as np
import torch

from . import ref_import
from .make_golden_tsdf import describe_default, look_at, on_sphere

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
MERGE_H, MERGE_W = 6, 9   # an odd width pins the W // 2 split of "half"


def stub_frame(name: str, index: int) -> np.ndarray:
    """The BGR image the cv2 stub returns for output ``name`` and frame ``index``: distinct per output, channel, row, column and frame."""
    base = {"rgb": 10, "normal": 100, "depth": 190}[name]
    y, x, c = np.meshgrid(np.arange(MERGE_H), np.arange(MERGE_W), np.arange(3), indexing="ij")
    return (base + 20 * c + 2 * y + x + index).astype(np.uint8)


def install_stubs(state):
    o3d = types.ModuleType("open3d")

    class Option:
        mesh_color_option = None

        def load_from_json(self, path):
            state["render_json_path"] = path

    class Param:
        def __init__(self):
            self.intrinsic = types.SimpleNamespace(set_intrinsics=lambda **kw: state["intrinsics"].append(kw))
            self.extrinsic = None

    class Control:
        def convert_to_pinhole_camera_parameters(self):
            return Param()

        def convert_from_pinhole_camera_parameters(self, param, allow_arbitrary):
            state["extrinsics"].append(np.array(param.extrinsic))

    class Visualizer:
        def __init__(self):
            self.cb, self.option = None, Option()

        def create_window(self, name, width, height):
            state["window"] = [width, height]

        def add_geometry(self, g):
            pass

        def get_render_option(self):
            return self.option

        def get_view_control(self):
            return Control()

        def register_animation_callback(self, cb):
            self.cb = cb

        def run(self):
            while self.cb is not None:
                self.cb(self)

        def destroy_window(self):
            pass

        def capture_screen_image(self, path, do_render):
            state["captures"].append([os.path.relpath(path, state["root"]), str(self.option.mesh_color_option)])

    class Mesh:
        def compute_vertex_normals(self):
            pass

        def paint_uniform_color(self, c):
            state["paint"] = list(c)

    o3d.io = types.SimpleNamespace(read_triangle_mesh=lambda path: Mesh())
    o3d.visualization = types.SimpleNamespace(VisualizerWithKeyCallback=Visualizer,
                                              MeshColorOption=types.SimpleNamespace(Normal="Normal", Color="Color"))
    sys.modules["open3d"] = o3d
    cv2 = types.ModuleType("cv2")

    def imread(path):
        p = Path(path)
        return stub_frame(p.parent.name, int(p.stem))

    cv2.imread = imread
    sys.modules["cv2"] = cv2
    media = types.ModuleType("mediapy")
    media.write_video = lambda path, images, fps: state["video"].append((str(path), [np.array(i) for i in images], fps))
    sys.modules["mediapy"] = media
    zmq = types.ModuleType("zmq")
    sys.modules.setdefault("zmq", zmq)
    dm = types.ModuleType("nerfstudio.data.datamanagers.base_datamanager")
    dm.AnnotatedDataParserUnion = object
    sys.modules["nerfstudio.data.datamanagers.base_datamanager"] = dm
    dp = types.ModuleType("nerfstudio.data.dataparsers.sdfstudio_dataparser")
    dp.SDFStudioDataParserConfig = type("SDFStudioDataParserConfig", (), {"__repr__": lambda self: "SDFStudioDataParserConfig()"})
    sys.modules["nerfstudio.data.dataparsers.sdfstudio_dataparser"] = dp
    ic = types.ModuleType("nerfstudio.utils.install_checks")
    ic.check_ffmpeg_installed = lambda: None
    sys.modules["nerfstudio.utils.install_checks"] = ic
    sys.modules["nerfstudio.configs.base_config"].Config = type("Config", (), {})


def camera_set(n, seed, fx=120.0, fy=110.0, cx=40.0, cy=30.5, H=61, W=80):
    c2w = look_at(on_sphere(n, 3.0, seed), target=(0.1, -0.2, 0.05))[:, :3, :]
    return dict(c2w=c2w, fx=fx, fy=fy, cx=cx, cy=cy, H=H, W=W)


def json_path(seed):
    g = torch.Generator().manual_seed(seed)
    c2w = look_at(on_sphere(5, 2.0, seed))
    fovs = [30.0 + 10 * float(torch.rand(1, generator=g)) for _ in range(5)]
    return {"render_height": 48, "render_width": 64, "seconds": 3.5,
            "camera_path": [{"camera_to_world": c2w[i].reshape(-1).tolist(), "fov": fovs[i]} for i in range(5)]}


def main():
    ref_import.install_shims()
    state = {"intrinsics": [], "extrinsics": [], "captures": [], "video": []}
    install_stubs(state)
    from nerfstudio.cameras import camera_paths
    from nerfstudio.cameras.cameras import Cameras, CameraType
    from nerfstudio.viewer.server.utils import three_js_perspective_camera_focal_length

    spec = importlib.util.spec_from_file_location("ref_render_mesh", os.path.join(ref_import.REFERENCE_ROOT, "scripts", "render_mesh.py"))
    rm = sys.modules[spec.name] = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(rm)

    def ref_cameras(s):
        n = len(s["c2w"])
        return Cameras(camera_to_worlds=s["c2w"], fx=torch.full((n, 1), s["fx"]), fy=torch.full((n, 1), s["fy"]), cx=torch.full((n, 1), s["cx"]),
                       cy=torch.full((n, 1), s["cy"]), width=torch.full((n, 1), s["W"]), height=torch.full((n, 1), s["H"]),
                       camera_type=CameraType.PERSPECTIVE)

    def record(prefix, cams):
        arrays[f"{prefix}/c2w"] = cams.camera_to_worlds.numpy().astype(np.float32)
        for k in ("fx", "fy", "cx", "cy"):
            arrays[f"{prefix}/{k}"] = getattr(cams, k).numpy().reshape(-1).astype(np.float32)
        arrays[f"{prefix}/hw"] = np.array([int(cams.height.view(-1)[0]), int(cams.width.view(-1)[0])])

    arrays, meta = {}, {"paths": {}}
    sets = {"a": camera_set(7, 1), "b": camera_set(4, 2, fx=90.0, fy=90.0, cx=32.0, cy=24.0, H=48, W=64)}
    for name, s in sets.items():
        for k, v in s.items():
            arrays[f"set_{name}/{k}"] = np.asarray(v, dtype=np.float32) if k != "c2w" else v.numpy()
    paths = {
        "spiral_a": lambda: camera_paths.get_spiral_path(ref_cameras(sets["a"]), steps=12, radius=1.0),
        "spiral_b_radiuses": lambda: camera_paths.get_spiral_path(ref_cameras(sets["b"]), steps=5, radiuses=(0.5, 0.7, 0.2), rots=1, zrate=0.25),
        "ellipse_a": lambda: camera_paths.generate_ellipse_path(ref_cameras(sets["a"]), n_frames=9, const_speed=False),
        "ellipse_b": lambda: camera_paths.generate_ellipse_path(ref_cameras(sets["b"]), n_frames=6, const_speed=False, z_variation=0.5,
                                                                z_phase=0.25),
        "interpolate_a": lambda: rm._interpolate_trajectory(ref_cameras(sets["a"]), num_views=11),
        "interpolate_b": lambda: rm._interpolate_trajectory(ref_cameras(sets["b"]), num_views=7),
    }
    for name, fn in paths.items():
        record(name, fn())
    cp = json_path(3)
    meta["json_path"] = cp
    record("json", camera_paths.get_path_from_json(cp))
    meta["three_js_focal"] = [[fov, h, float(three_js_perspective_camera_focal_length(fov, h))] for fov, h in ((50.0, 480), (33.3, 61), (90.0, 7))]
    meta["three_js_focal_none"] = three_js_perspective_camera_focal_length(None, 100)

    # the merge layout: three frames through _render_trajectory_video with the visualizer, cv2 and mediapy stubs
    meta["merge"] = {}
    with tempfile.TemporaryDirectory() as root:
        state["root"] = root
        for merge_type, names in (("half", ["rgb", "normal"]), ("half", ["normal", "rgb", "depth"]), ("concat", ["rgb", "normal"]),
                                  ("concat", ["normal", "depth", "rgb"])):
            state["captures"].clear()
            state["video"].clear()
            s = dict(sets["b"], c2w=sets["b"]["c2w"][:3], H=MERGE_H, W=MERGE_W, cx=MERGE_W / 2, cy=MERGE_H / 2)
            out = Path(root) / "renders" / "out.mp4"
            rm._render_trajectory_video(Path("mesh.ply"), ref_cameras(s), out, names, 1.0, seconds=1.5, output_format="video", merge_type=merge_type)
            key = f"{merge_type}_{'_'.join(names)}"
            path, frames, fps = state["video"][0]
            arrays[f"merge/{key}"] = np.stack(frames)
            meta["merge"][key] = dict(names=names, fps=fps, video=os.path.relpath(path, root), captures=list(state["captures"]))
    meta["paint_uniform_color"] = state["paint"]
    meta["render_json_path"] = state["render_json_path"]
    meta["merge_frame_hw"] = [MERGE_H, MERGE_W]

    fields = []
    for f in dataclasses.fields(rm.RenderTrajectory):
        d = f.default_factory() if f.default_factory is not dataclasses.MISSING else f.default
        fields.append([f.name, describe_default(str(d) if isinstance(d, Path) else d) if f.name != "data" else {"default": repr(d)}])
    meta["RenderTrajectory"] = fields
    sig = __import__("inspect").signature
    meta["signatures"] = {fn: [[p.name, describe_default(p.default)] for p in sig(getattr(mod, fn)).parameters.values()]
                          for mod, fn in ((rm, "_render_trajectory_video"), (rm, "_interpolate_trajectory"), (camera_paths, "get_spiral_path"),
                                          (camera_paths, "generate_ellipse_path"), (camera_paths, "get_path_from_json"))}
    with open(os.path.join(ref_import.REFERENCE_ROOT, "scripts", "render.json"), encoding="utf-8") as fh:
        meta["render_json"] = json.load(fh)
    np.savez_compressed(os.path.join(GOLDEN_DIR, "render_mesh.npz"), **arrays)
    with open(os.path.join(GOLDEN_DIR, "render_mesh.json"), "w") as fh:
        json.dump(meta, fh, indent=1)


if __name__ == "__main__":
    main()
