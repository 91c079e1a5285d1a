"""Ray generation for batches of pinhole / fisheye cameras -- the part of ``nerfstudio.cameras.cameras.Cameras``
(cameras/cameras.py:300-457 ``generate_rays``, :459-695 ``_generate_rays_from_coords``) that feeds the render path.
One kernel (sdfb200_generate_rays) per call; distortion parameters, equirectangular cameras and camera-optimizer deltas are not
handled here (use the reference ``Cameras`` for those -- its RayBundle is accepted by every module of this package).
"""
from typing import Optional, Union

import torch

from . import _lib
from .rays import RayBundle

PERSPECTIVE, FISHEYE = _lib.CAMERA_PERSPECTIVE, _lib.CAMERA_FISHEYE


class Cameras:
    """Flat batch of C cameras.  camera_to_worlds [C,3,4]; fx, fy, cx, cy scalars or [C]; camera_type int or [C]."""

    def __init__(self, camera_to_worlds, fx, fy, cx, cy, width: int, height: int, camera_type: Union[int, torch.Tensor] = PERSPECTIVE,
                 device: Optional[torch.device] = None):
        c2w = torch.as_tensor(camera_to_worlds, dtype=torch.float32)
        if c2w.dim() == 2:
            c2w = c2w[None]
        n = c2w.shape[0]
        dev = device if device is not None else c2w.device
        self.camera_to_worlds = c2w[:, :3, :4].contiguous().to(dev)

        def per_cam(v, dtype=torch.float32):
            t = torch.as_tensor(v, dtype=dtype).reshape(-1)
            return (t.expand(n) if t.numel() == 1 else t).contiguous().to(dev)

        self.fx, self.fy, self.cx, self.cy = per_cam(fx), per_cam(fy), per_cam(cx), per_cam(cy)
        self.camera_type = per_cam(camera_type, torch.int32)
        self.width, self.height = int(width), int(height)
        self.device = dev

    def __len__(self):
        return self.camera_to_worlds.shape[0]

    def get_intrinsics_matrices(self) -> torch.Tensor:
        """[C,3,3] fp32 pinhole intrinsics (cameras/cameras.py:733-745)."""
        K = torch.zeros((len(self), 3, 3), dtype=torch.float32, device=self.device)
        K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = self.fx, self.fy, self.cx, self.cy, 1.0
        return K

    def rescale_output_resolution(self, scaling_factor: Union[float, int]) -> None:
        """Scales fx, fy, cx, cy (fp32 products) and the image size (cameras/cameras.py:747-771); height and width are truncated as
        ``.to(torch.int64)`` truncates the fp32 product.  The cameras share one image size, so the factor is one number."""
        if not isinstance(scaling_factor, (float, int)):
            raise ValueError("Scaling factor must be a float or an int (the cameras share one image size).")
        s = torch.tensor([scaling_factor], dtype=torch.float32, device=self.device)
        self.fx, self.fy, self.cx, self.cy = self.fx * s, self.fy * s, self.cx * s, self.cy * s
        self.height = int((torch.tensor([self.height]) * s.cpu()).to(torch.int64))
        self.width = int((torch.tensor([self.width]) * s.cpu()).to(torch.int64))

    def get_image_coords(self, pixel_offset: float = 0.5) -> torch.Tensor:
        """[H, W, 2] (y, x) pixel centres (cameras/cameras.py:268-293)."""
        ys = torch.arange(self.height, device=self.device, dtype=torch.float32) + pixel_offset
        xs = torch.arange(self.width, device=self.device, dtype=torch.float32) + pixel_offset
        return torch.stack(torch.meshgrid(ys, xs, indexing="ij"), dim=-1)

    def generate_rays(self, camera_indices, coords: Optional[torch.Tensor] = None) -> RayBundle:
        """camera_indices: int (whole image) or [N] / [N,1] tensor with coords [N,2] = (y, x).  Returns a RayBundle of shape
        [N] (or [H*W] for a whole image, row-major; reshape with ``.reshape(H, W, ...)`` as needed)."""
        lib = _lib.load()
        if isinstance(camera_indices, int):
            if coords is None:
                coords = self.get_image_coords().reshape(-1, 2)
            camera_indices = torch.full((coords.shape[0],), camera_indices, dtype=torch.int32, device=self.device)
        idx = camera_indices.reshape(-1).to(device=self.device, dtype=torch.int32).contiguous()
        coords = _lib.f32c(coords.reshape(-1, 2).to(self.device))
        n = idx.shape[0]
        if coords.shape[0] != n:
            raise ValueError("camera_indices and coords disagree on the number of rays")
        o = torch.empty(n, 3, device=self.device)
        d = torch.empty(n, 3, device=self.device)
        area = torch.empty(n, 1, device=self.device)
        dnorm = torch.empty(n, 1, device=self.device)
        _lib.check(lib.sdfb200_generate_rays(_lib.ptr(self.fx), _lib.ptr(self.fy), _lib.ptr(self.cx), _lib.ptr(self.cy), _lib.ptr(self.camera_type),
                                             _lib.ptr(self.camera_to_worlds), len(self), _lib.ptr(idx), _lib.ptr(coords), n, _lib.ptr(o), _lib.ptr(d),
                                             _lib.ptr(area), _lib.ptr(dnorm), _lib.stream_ptr()), "sdfb200_generate_rays")
        return RayBundle(origins=o, directions=d, pixel_area=area, directions_norm=dnorm, camera_indices=idx.view(n, 1).long())
