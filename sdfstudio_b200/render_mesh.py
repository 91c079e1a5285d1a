"""Mesh rendering on the GPU: drop-ins for ``scripts/render_mesh.py`` (``ns-render-mesh``) and the camera paths it uses
(``nerfstudio/cameras/camera_paths.py``).

The reference draws the mesh with open3d's OpenGL visualizer, which needs a display, captures every frame to a PNG and reads it back
with cv2.  Here the mesh is rasterized by one kernel (sdfb200_mesh_rasterize: one 64-bit depth-and-face key per pixel, exact in double,
independent of scheduling) and shaded by another (sdfb200_mesh_shade: "rgb", the Phong shading of a white mesh under the four lights of
the reference's ``scripts/render.json``, and "normal", the camera-space normal as colour), on a headless GPU.  The frames stay on the
device until they are encoded.

The pixel convention is nerfstudio's (``Cameras.generate_rays``): pixel (i, j) is centred at (i + 0.5, j + 0.5), so a mesh frame lines up
with the field's render of the same camera.  The shading is this package's reading of open3d's legacy shaders; it is not pinned to
open3d's pixels.
"""
import collections
import concurrent.futures
import ctypes
import json
import math
import os
from pathlib import Path
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, meshing, texturing
from .cameras import PERSPECTIVE, Cameras
from .tsdf import pack_cams

OUTPUTS = ("rgb", "normal")
# scripts/render.json, the values the shading reads (tests/golden/render_mesh.json holds the reference's file)
RENDER_OPTIONS = {
    "background_color": [1.0, 1.0, 1.0],
    "light0_color": [0.69999999999999996] * 3, "light0_diffuse_power": 0.66000000000000014, "light0_position": [0.0, 0.0, 2.0],
    "light0_specular_power": 0.20000000000000001, "light0_specular_shininess": 10.0,
    "light1_color": [0.69999999999999996] * 3, "light1_diffuse_power": 0.66000000000000014, "light1_position": [0.0, 0.0, -2.0],
    "light1_specular_power": 0.20000000000000001, "light1_specular_shininess": 10.0,
    "light2_color": [0.69999999999999996] * 3, "light2_diffuse_power": 0.36000000000000015, "light2_position": [2.0, 2.0, 0.0],
    "light2_specular_power": 1.0000000000000001e-17, "light2_specular_shininess": 10.0,
    "light3_color": [0.69999999999999996] * 3, "light3_diffuse_power": 0.10000000000000014, "light3_position": [-2.0, -2.0, 0.0],
    "light3_specular_power": 9.9999999999999998e-17, "light3_specular_shininess": 0.10000000000000001,
    "light_ambient_color": [0.29999999999999999] * 3,
    "light_on": True,
    "mesh_show_back_face": False,
}  # fmt: skip
KEY_BUDGET_BYTES = 256 << 20   # the key buffer of one launch; frames are batched to stay within it
Z_NEAR_FRACTION = 0.01         # the default near plane: this fraction of the mesh box's largest extent
MAX_PNG_JOBS_PER_WORKER = 4    # PNG jobs queued per encoding thread before the renderer waits for the oldest


def light_params() -> np.ndarray:
    """[27] fp32: per light k = 0..3 colour r, g, b, diffuse, specular, shininess, then the ambient colour (sdfb200_mesh_shade)."""
    o = RENDER_OPTIONS
    rows = [[*o[f"light{k}_color"], o[f"light{k}_diffuse_power"], o[f"light{k}_specular_power"], o[f"light{k}_specular_shininess"]]
            for k in range(4)]
    return np.array(sum(rows, []) + o["light_ambient_color"], dtype=np.float32)


def light_positions(cams: torch.Tensor, centre: torch.Tensor, extent: float) -> torch.Tensor:
    """[B,4,3] fp32: light k of each frame at centre + extent (p.x right + p.y up + p.z front) in world space (right, up and front the
    camera's axes, front toward the eye), in the frame's camera space: the camera-space centre plus extent p."""
    p = torch.tensor([RENDER_OPTIONS[f"light{k}_position"] for k in range(4)], dtype=torch.float32, device=cams.device)
    m = cams[:, :12].view(-1, 3, 4)
    c = (m[:, :, :3] @ centre.view(3, 1)).view(-1, 1, 3) + m[:, :, 3].view(-1, 1, 3)
    return (c + extent * p.view(1, 4, 3)).contiguous()


# ---------------------------------------------------------------------------------------------------------------------------------
# rasterize and shade
# ---------------------------------------------------------------------------------------------------------------------------------
def _check_cameras(cameras: Cameras):
    if not isinstance(cameras, Cameras):
        raise ValueError(f"expected the package's Cameras, got {type(cameras).__name__}")
    if bool((cameras.camera_type != PERSPECTIVE).any()):
        raise ValueError("only perspective cameras can be rendered")


def package_cameras(cameras) -> Cameras:
    """``cameras`` as the package's :class:`Cameras`: itself, or a copy of the reference's ``nerfstudio.cameras.cameras.Cameras`` (which
    ``RenderTrajectory.main`` builds): its [N,3,4] poses, its [N,1] (or [N]) fx, fy, cx, cy and camera_type, and its per-camera width and
    height, which must be one size for all cameras.  Anything else raises ValueError."""
    if isinstance(cameras, Cameras):
        return cameras
    names = ("camera_to_worlds", "fx", "fy", "cx", "cy", "width", "height", "camera_type")
    if not all(hasattr(cameras, n) for n in names):
        raise ValueError(f"expected the package's or the reference's Cameras, got {type(cameras).__name__}")
    c2w = torch.as_tensor(cameras.camera_to_worlds).reshape(-1, 3, 4)
    flat = {n: torch.as_tensor(getattr(cameras, n)).reshape(-1) for n in names[1:]}
    h, w = flat["height"], flat["width"]
    if len(h) != len(c2w) or len(w) != len(c2w) or (len(h) and (bool((h != h[0]).any()) or bool((w != w[0]).any()))):
        raise ValueError("the cameras must share one image size")
    return Cameras(c2w, flat["fx"], flat["fy"], flat["cx"], flat["cy"], int(w[0]) if len(w) else 0, int(h[0]) if len(h) else 0,
                   flat["camera_type"].to(torch.int32), device=c2w.device)


def _check_mesh(vertices: torch.Tensor, faces: torch.Tensor):
    if vertices.dim() != 2 or vertices.shape[1] != 3 or faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError(f"expected vertices [V,3] and faces [F,3], got {tuple(vertices.shape)} and {tuple(faces.shape)}")
    if not bool(torch.isfinite(vertices).all()):
        raise ValueError("the mesh has non-finite vertices")
    if len(faces) and (int(faces.min()) < 0 or int(faces.max()) >= len(vertices)):
        raise ValueError(f"face indices must lie in [0, {len(vertices)})")


def _box(vertices: torch.Tensor) -> Tuple[torch.Tensor, float]:
    """(centre [3], largest extent) of the mesh's bounding box; (0, 0) for an empty mesh."""
    if len(vertices) == 0:
        return torch.zeros(3, device=vertices.device), 0.0
    lo, hi = vertices.amin(0), vertices.amax(0)
    return (lo + hi) / 2, float((hi - lo).max())


def _prepare(vertices, faces, cameras: Cameras):
    _check_cameras(cameras)
    _lib.require_cuda(cameras.device, "render_mesh")
    v = _lib.f32c(torch.as_tensor(vertices).to(cameras.device))
    f = torch.as_tensor(faces).to(cameras.device, torch.int64).contiguous()
    _check_mesh(v, f)
    c2w = torch.cat([cameras.camera_to_worlds, torch.tensor([0.0, 0, 0, 1], device=cameras.device).expand(len(cameras), 1, 4)], dim=1)
    return v, f, pack_cams(c2w, cameras.get_intrinsics_matrices())


def _z_near(z_near, extent: float) -> float:
    if z_near is not None:
        if not (math.isfinite(float(z_near)) and float(z_near) > 0):
            raise ValueError(f"z_near must be finite and > 0, got {z_near}")
        return float(z_near)
    return Z_NEAR_FRACTION * extent if extent > 0 else Z_NEAR_FRACTION


def _keys(v, f, cams, H, W, z_near) -> torch.Tensor:
    keys = torch.empty(cams.shape[0], H, W, dtype=torch.int64, device=v.device)
    _lib.check(_lib.load().sdfb200_mesh_rasterize(_lib.ptr(v), _lib.ptr(f), len(f), _lib.ptr(cams), cams.shape[0], H, W, z_near, _lib.ptr(keys),
                                                  _lib.stream_ptr()), "sdfb200_mesh_rasterize")
    return keys


def split_keys(keys: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(face ids int32, -1 for background; view depth fp32, +inf for background) of rasterizer keys (int64 storage)."""
    bg = keys == -1
    face = torch.where(bg, -1, keys & 0xFFFFFFFF).to(torch.int32)
    depth = (keys >> 32).to(torch.int32).view(torch.float32)
    return face, torch.where(bg, torch.full_like(depth, math.inf), depth)


def rasterize(vertices: torch.Tensor, faces: torch.Tensor, cameras: Cameras, z_near: Optional[float] = None):
    """Face ids [B,H,W] int32 (-1 for background) and view depth [B,H,W] fp32 (+inf for background) of the mesh in every camera: the
    nearest front-facing (counter-clockwise on screen) face whose closed triangle the ray through the pixel centre meets at view depth
    >= ``z_near``, ties to the smaller id (sdfb200_mesh_rasterize).  ``z_near`` defaults to 0.01 x the largest extent of the mesh's box;
    there is no far plane.  CUDA only."""
    v, f, cams = _prepare(vertices, faces, cameras)
    return split_keys(_keys(v, f, cams, cameras.height, cameras.width, _z_near(z_near, _box(v)[1])))


def _check_outputs(outputs: Sequence[str]):
    bad = [n for n in outputs if n not in OUTPUTS]
    if bad or not outputs:
        raise ValueError(f"rendered outputs must be among {list(OUTPUTS)}, got {list(outputs)}")


def render_frames(vertices: torch.Tensor, faces: torch.Tensor, cameras: Cameras, outputs: Sequence[str] = OUTPUTS,
                  z_near: Optional[float] = None) -> Dict[str, torch.Tensor]:
    """Each requested output ("rgb", "normal") as uint8 frames [B,H,W,3] on the device.  Vertex normals are the area-weighted ones
    (``texturing.vertex_normals_area_weighted``, open3d's compute_vertex_normals); the background is white.  Frames go through the
    kernels in batches whose keys fit KEY_BUDGET_BYTES."""
    _check_outputs(outputs)
    v, f, cams = _prepare(vertices, faces, cameras)
    H, W, B = cameras.height, cameras.width, len(cameras)
    centre, extent = _box(v)
    zn = _z_near(z_near, extent)
    normals = _lib.f32c(texturing.vertex_normals_area_weighted(v, f)) if len(f) else torch.zeros_like(v)
    lights = light_positions(cams, centre, extent)
    params = light_params()
    params_ptr = params.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    out = {n: torch.empty(B, H, W, 3, dtype=torch.uint8, device=v.device) for n in outputs}
    step = max(1, KEY_BUDGET_BYTES // (H * W * 8))
    for b0 in range(0, B, step):
        c = cams[b0:b0 + step]
        keys = _keys(v, f, c, H, W, zn)
        _lib.check(_lib.load().sdfb200_mesh_shade(_lib.ptr(keys), c.shape[0], H, W, _lib.ptr(v), _lib.ptr(normals), _lib.ptr(f), len(f), _lib.ptr(c),
                                                  _lib.ptr(lights[b0:b0 + step]), params_ptr,
                                                  _lib.ptr(out["rgb"][b0:b0 + step]) if "rgb" in out else None,
                                                  _lib.ptr(out["normal"][b0:b0 + step]) if "normal" in out else None, _lib.stream_ptr()),
                   "sdfb200_mesh_shade")
    return out


# ---------------------------------------------------------------------------------------------------------------------------------
# scripts/render_mesh.py
# ---------------------------------------------------------------------------------------------------------------------------------
def merge_frames(images: Sequence[np.ndarray], merge_type: str) -> np.ndarray:
    """The frame the reference puts in the video (render_mesh.py:144-149): "concat" places the outputs side by side, "half" takes the
    left W // 2 columns from the first output and the rest from the second."""
    if merge_type == "concat":
        return np.concatenate(images, axis=1)
    if merge_type == "half":
        out = images[1].copy()
        out[:, : out.shape[1] // 2] = images[0][:, : out.shape[1] // 2]
        return out
    raise ValueError(f"merge_type must be 'half' or 'concat', not {merge_type!r}")


def _check_render_args(rendered_output_names, output_filename, output_format, merge_type):
    _check_outputs(list(rendered_output_names))
    if output_format not in ("images", "video"):
        raise ValueError(f"output_format must be 'images' or 'video', not {output_format!r}")
    if merge_type not in ("half", "concat"):
        raise ValueError(f"merge_type must be 'half' or 'concat', not {merge_type!r}")
    if merge_type == "half" and len(rendered_output_names) < 2:
        raise ValueError('merge_type="half" needs two rendered outputs')
    if output_format == "video" and not str(output_filename).endswith(".mp4"):
        raise ValueError(f"the video path must end in .mp4, got {str(output_filename)!r}")


def _import_mediapy():
    return meshing.import_optional("mediapy", 'output_format="video" needs the mediapy package, which is not installed; install it or use '
                                              'output_format="images"')


def render_trajectory_video(meshfile: Path, cameras: Cameras, output_filename: Path, rendered_output_names: Sequence[str],
                            rendered_resolution_scaling_factor: float = 1.0, seconds: float = 5.0, output_format: str = "video",
                            merge_type: str = "half") -> None:
    """render_mesh.py:71-183: renders the binary PLY ``meshfile`` from every camera (rescaled in place by
    ``rendered_resolution_scaling_factor``) and writes ``output_filename.parent / output_filename.stem / <name> / {index:05d}.png`` for
    every output name and frame; with ``output_format="video"`` also the merged frames to ``output_filename`` (mp4, through mediapy, at
    len(frames) / seconds frames per second).  ``cameras``: the package's :class:`Cameras` or the reference's (see
    :func:`package_cameras`), so that the function can replace the reference script's own.  Needs no display, open3d or ffmpeg for
    PNGs.  At most MAX_PNG_JOBS_PER_WORKER frames per encoding thread wait in host memory for their PNG."""
    output_filename = Path(output_filename)
    _check_render_args(rendered_output_names, output_filename, output_format, merge_type)
    _check_cameras(package_cameras(cameras))
    media = _import_mediapy() if output_format == "video" else None
    cameras.rescale_output_resolution(rendered_resolution_scaling_factor)
    cameras = package_cameras(cameras)
    vertices, faces, _ = meshing.read_ply(str(meshfile))
    device = cameras.device if cameras.device.type == "cuda" else meshing.work_device()
    if device.type != "cuda":
        raise RuntimeError("sdfstudio_b200.render_mesh runs on CUDA only (there is no CPU path)")
    if cameras.device != device:
        cameras = Cameras(cameras.camera_to_worlds, cameras.fx, cameras.fy, cameras.cx, cameras.cy, cameras.width, cameras.height,
                          cameras.camera_type, device=device)
    v, f = torch.from_numpy(vertices).to(device), torch.from_numpy(faces).to(device)
    _check_mesh(v, f)
    out_dir = output_filename.parent / output_filename.stem
    for name in rendered_output_names:
        (out_dir / name).mkdir(parents=True, exist_ok=True)
    names = list(dict.fromkeys(rendered_output_names))
    H, W = cameras.height, cameras.width
    step = max(1, KEY_BUDGET_BYTES // max(1, H * W * 8))
    merged = []
    workers = min(32, os.cpu_count() or 1)
    with concurrent.futures.ThreadPoolExecutor(max_workers=workers) as pool:
        pending = collections.deque()
        for b0 in range(0, len(cameras), step):
            sub = Cameras(cameras.camera_to_worlds[b0:b0 + step], cameras.fx[b0:b0 + step], cameras.fy[b0:b0 + step], cameras.cx[b0:b0 + step],
                          cameras.cy[b0:b0 + step], W, H, cameras.camera_type[b0:b0 + step], device=device)
            frames = {n: t.cpu().numpy() for n, t in render_frames(v, f, sub, names).items()}
            for k in range(len(sub)):
                for name in rendered_output_names:
                    path = out_dir / name / f"{b0 + k:05d}.png"
                    pending.append(pool.submit(lambda p, img: p.write_bytes(texturing.png_bytes_u8(img)), path, frames[name][k]))
                    while len(pending) > MAX_PNG_JOBS_PER_WORKER * workers:   # the GPU renders far faster than the threads encode
                        pending.popleft().result()
                if media is not None:
                    merged.append(merge_frames([frames[n][k] for n in rendered_output_names], merge_type))
        for p in pending:
            p.result()
    if media is not None:
        media.write_video(output_filename, merged, fps=len(merged) / seconds)


# ---------------------------------------------------------------------------------------------------------------------------------
# camera paths (nerfstudio/cameras/camera_paths.py and render_mesh.py:37-68), on the package's Cameras
# ---------------------------------------------------------------------------------------------------------------------------------
def three_js_perspective_camera_focal_length(fov: Optional[float], image_height: int):
    """The focal length in pixels of a three.js perspective camera with vertical field of view ``fov`` degrees (50 when fov is None)."""
    if fov is None:
        print("Warning: fov is None, using default value")
        return 50
    return (image_height / 2.0) / np.tan(fov * (np.pi / 180.0) / 2.0)


def _unit(x: torch.Tensor) -> torch.Tensor:
    return x / torch.linalg.norm(x)


def _look(lookat: torch.Tensor, up: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
    """[3,4] camera-to-world whose z axis is along ``lookat`` (camera_utils.viewmatrix)."""
    z = _unit(lookat)
    x = _unit(torch.cross(_unit(up), z, dim=-1))
    y = _unit(torch.cross(z, x, dim=-1))
    return torch.stack([x, y, z, pos], 1)


def _homogeneous(m: torch.Tensor) -> torch.Tensor:
    bottom = torch.zeros_like(m[..., :1, :])
    bottom[..., :, 3] = 1
    return torch.cat([m, bottom], dim=-2)


def get_spiral_path(camera: Cameras, steps: int = 30, radius: Optional[float] = None, radiuses: Optional[Tuple[float]] = None, rots: int = 2,
                    zrate: float = 0.5) -> Cameras:
    """camera_paths.get_spiral_path: ``steps`` cameras on a spiral around the first camera's focal point, in fp32 on the host as the
    reference computes them.  The image is int(2 cx) x int(2 cy), as for the reference's Cameras built without a size."""
    if (radius is None) == (radiuses is None):
        raise ValueError("Only one of radius or radiuses must be specified.")
    rad = torch.tensor([radius] * 3 if radius is not None else list(radiuses))
    c2w0 = camera.camera_to_worlds[0].cpu()
    fx, fy, cx, cy = (t[0].cpu() for t in (camera.fx, camera.fy, camera.cx, camera.cy))
    up = c2w0[:3, 2]
    target = torch.tensor([0.0, 0.0, -float(torch.min(fx, fy))])
    glob = _homogeneous(c2w0)
    c2ws = []
    for theta in torch.linspace(0.0, 2.0 * torch.pi * rots, steps + 1)[:-1]:
        centre = torch.tensor([torch.cos(theta), -torch.sin(theta), -torch.sin(theta * zrate)]) * rad
        c2ws.append(torch.matmul(glob, _homogeneous(_look(centre - target, up, centre)))[:3, :4])
    return Cameras(torch.stack(c2ws), fx, fy, cx, cy, int((cx * 2).to(torch.int64)), int((cy * 2).to(torch.int64)), device=camera.device)


def get_path_from_json(camera_path: Dict[str, Any]) -> Cameras:
    """camera_paths.get_path_from_json: the viewer's camera path (per-frame camera_to_world and vertical fov) at render_width x
    render_height."""
    h, w = camera_path["render_height"], camera_path["render_width"]
    c2ws = torch.stack([torch.tensor(c["camera_to_world"]).view(4, 4)[:3] for c in camera_path["camera_path"]])
    focal = torch.tensor([three_js_perspective_camera_focal_length(c["fov"], h) for c in camera_path["camera_path"]])
    return Cameras(c2ws, focal, focal, w / 2, h / 2, int(w / 2 * 2), int(h / 2 * 2))


def _np_unit(x):
    return x / np.linalg.norm(x)


def _np_look(lookdir, up, position):
    z = _np_unit(lookdir)
    x = _np_unit(np.cross(up, z))
    y = _np_unit(np.cross(z, x))
    return np.stack([x, y, z, position], axis=1)


def _first_camera_path(cameras: Cameras, c2ws: np.ndarray) -> Cameras:
    """Cameras along ``c2ws`` with the intrinsics, size and type of the first of ``cameras``."""
    return Cameras(torch.from_numpy(np.ascontiguousarray(c2ws[:, :3, :4])), cameras.fx[0], cameras.fy[0], cameras.cx[0], cameras.cy[0],
                   cameras.width, cameras.height, cameras.camera_type[0], device=cameras.device)


def generate_ellipse_path(cameras: Cameras, n_frames: int = 120, const_speed: bool = True, z_variation: float = 0.0,
                          z_phase: float = 0.0) -> Cameras:
    """camera_paths.generate_ellipse_path (multinerf's): ``n_frames`` cameras on an ellipse in the plane z = 0 around the point nearest
    to every camera's optical axis, looking at it, in float64 as the reference computes it.  const_speed=True raises
    NotImplementedError, as there."""
    poses = cameras.camera_to_worlds.cpu().numpy()
    dirs, origins = poses[:, :3, 2:3], poses[:, :3, 3:4]
    m = np.eye(3) - dirs * np.transpose(dirs, [0, 2, 1])
    mtm = np.transpose(m, [0, 2, 1]) @ m
    centre = np.linalg.inv(mtm.mean(0)) @ (mtm @ origins).mean(0)[:, 0]
    offset = np.array([centre[0], centre[1], 0])
    sc = np.percentile(np.abs(poses[:, :3, 3] - offset), 90, axis=0)
    low, high = -sc + offset, sc + offset
    z_low, z_high = np.percentile(poses[:, :3, 3], 10, axis=0), np.percentile(poses[:, :3, 3], 90, axis=0)
    theta = np.linspace(0, 2.0 * np.pi, n_frames + 1, endpoint=True)
    positions = np.stack([low[0] + (high - low)[0] * (np.cos(theta) * 0.5 + 0.5), low[1] + (high - low)[1] * (np.sin(theta) * 0.5 + 0.5),
                          z_variation * (z_low[2] + (z_high - z_low)[2] * (np.cos(theta + 2 * np.pi * z_phase) * 0.5 + 0.5))], -1)
    if const_speed:
        raise NotImplementedError
    positions = positions[:-1]
    avg_up = poses[:, :3, 1].mean(0)
    avg_up = avg_up / np.linalg.norm(avg_up)
    axis = np.argmax(np.abs(avg_up))
    up = np.eye(3)[axis] * np.sign(avg_up[axis])
    return _first_camera_path(cameras, np.stack([_np_look(p - centre, up, p) for p in positions]))


def interpolate_trajectory(cameras: Cameras, num_views: int = 300) -> Cameras:
    """render_mesh.py:37-68: ``num_views`` cameras at times i / num_views (len - 1), i < num_views, along the given cameras: rotations by
    scipy's Slerp, positions linearly interpolated (scipy, imported here as the reference's script imports it)."""
    from scipy.interpolate import interp1d
    from scipy.spatial.transform import Rotation, Slerp

    c2ws = cameras.camera_to_worlds.cpu().numpy()
    times = list(range(len(c2ws)))
    slerp = Slerp(times, Rotation.from_matrix(c2ws[:, :3, :3]))
    interp = interp1d(times, c2ws[:, :3, 3], axis=0)
    out = []
    for i in range(num_views):
        t = float(i) / num_views * (len(c2ws) - 1)
        c2w = np.eye(4)
        c2w[:3, :3] = slerp(t).as_matrix()
        c2w[:3, 3] = interp(t)
        out.append(c2w)
    return _first_camera_path(cameras, np.stack(out))


def render_mesh(meshfile: Path, cameras: Optional[Cameras] = None, output_path: Path = Path("renders/output.mp4"), traj: str = "spiral",
                rendered_output_names: Optional[List[str]] = None, downscale_factor: int = 1, camera_path_filename: Path = Path("camera_path.json"),
                seconds: float = 5.0, fps: int = 24, output_format: str = "video", merge_type: str = "half", num_views: int = 300) -> None:
    """RenderTrajectory.main (render_mesh.py:187-251) with the package's ``cameras`` in place of the dataparser's training cameras
    (needed for every ``traj`` but "filename").  The trajectory's length sets ``seconds`` as there: the JSON's "seconds" for
    "filename", num_views / 24 for "spiral" and "interpolate", num_views / fps for "ellipse".  Needs ffmpeg (through mediapy) only
    for ``output_format="video"``."""
    names = ["rgb", "normal"] if rendered_output_names is None else list(rendered_output_names)
    _check_render_args(names, output_path, output_format, merge_type)
    if traj not in ("spiral", "filename", "interpolate", "ellipse"):
        raise ValueError(f"traj must be 'spiral', 'filename', 'interpolate' or 'ellipse', not {traj!r}")
    if traj != "filename" and cameras is None:
        raise ValueError(f'traj="{traj}" needs the training cameras')
    if traj == "filename":
        with open(camera_path_filename, "r", encoding="utf-8") as fh:
            camera_path = json.load(fh)
        seconds = camera_path["seconds"]
        path = get_path_from_json(camera_path)
        if cameras is not None:
            path = Cameras(path.camera_to_worlds, path.fx, path.fy, path.cx, path.cy, path.width, path.height, device=cameras.device)
    elif traj == "interpolate":
        path = interpolate_trajectory(cameras, num_views=num_views)
        seconds = len(path) / 24
    elif traj == "spiral":
        path = get_spiral_path(cameras, steps=num_views, radius=1.0)
        seconds = len(path) / 24
    else:
        path = generate_ellipse_path(cameras, n_frames=num_views, const_speed=False)
        seconds = len(path) / fps
    render_trajectory_video(meshfile, path, output_filename=Path(output_path), rendered_output_names=names,
                            rendered_resolution_scaling_factor=1.0 / downscale_factor, seconds=seconds, output_format=output_format,
                            merge_type=merge_type)
