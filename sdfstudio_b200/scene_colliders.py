"""H100-native drop-ins for ``nerfstudio.model_components.scene_colliders`` (:30-163): set ``nears`` / ``fars`` on a RayBundle.
One kernel launch (sdfb200_collide) instead of ~20 ATen elementwise ops."""
import ctypes as C

import torch
from torch import nn

from . import _lib


def _collide(ray_bundle, ctype: int, params, near_plane: float = 0.0):
    lib = _lib.load()
    o, d = _lib.f32c(ray_bundle.origins.reshape(-1, 3)), _lib.f32c(ray_bundle.directions.reshape(-1, 3))
    n = o.shape[0]
    nears = torch.empty(n, device=o.device, dtype=torch.float32)
    fars = torch.empty_like(nears)
    arr = (C.c_float * len(params))(*[float(p) for p in params])
    _lib.check(lib.sdfb200_collide(_lib.ptr(o), _lib.ptr(d), n, ctype, arr, float(near_plane), _lib.ptr(nears), _lib.ptr(fars), _lib.stream_ptr()),
               "sdfb200_collide")
    shape = ray_bundle.origins.shape[:-1]
    ray_bundle.nears = nears.view(*shape, 1)
    ray_bundle.fars = fars.view(*shape, 1)
    return ray_bundle


class SceneCollider(nn.Module):
    """scene_colliders.py:30-47."""

    def __init__(self, **kwargs) -> None:
        self.kwargs = kwargs
        super().__init__()

    def set_nears_and_fars(self, ray_bundle):
        raise NotImplementedError

    def forward(self, ray_bundle):
        if ray_bundle.nears is not None and ray_bundle.fars is not None:
            return ray_bundle
        return self.set_nears_and_fars(ray_bundle)


class AABBBoxCollider(SceneCollider):
    """scene_colliders.py:50-113.  ``scene_box`` needs an ``aabb`` [2,3] attribute (the reference SceneBox works as is)."""

    def __init__(self, scene_box, near_plane: float = 0.0, **kwargs) -> None:
        super().__init__(**kwargs)
        self.scene_box = scene_box
        self.near_plane = near_plane

    def set_nears_and_fars(self, ray_bundle):
        aabb = torch.as_tensor(self.scene_box.aabb, dtype=torch.float32).reshape(6).tolist()
        return _collide(ray_bundle, _lib.COLLIDER_AABB, aabb, self.near_plane if self.training else 0.0)


class NearFarCollider(SceneCollider):
    """scene_colliders.py:116-134."""

    def __init__(self, near_plane: float, far_plane: float, **kwargs) -> None:
        self.near_plane = near_plane
        self.far_plane = far_plane
        super().__init__(**kwargs)

    def set_nears_and_fars(self, ray_bundle):
        return _collide(ray_bundle, _lib.COLLIDER_NEAR_FAR, [self.near_plane, self.far_plane])


class SphereCollider(SceneCollider):
    """scene_colliders.py:137-163 (note: like the reference it overrides ``forward`` and always recomputes)."""

    def __init__(self, radius: float = 1.0, soft_intersection=False, **kwargs) -> None:
        self.radius = radius
        self.soft_intersection = soft_intersection
        super().__init__(**kwargs)

    def forward(self, ray_bundle):
        return _collide(ray_bundle, _lib.COLLIDER_SPHERE, [self.radius, 1.0 if self.soft_intersection else 0.0, float(self.radius) ** 2])
