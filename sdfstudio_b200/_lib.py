"""ctypes binding of libsdfb200.so (the C-ABI declared in include/sdfb200.h).

The product path has NO fallback: if the shared library is missing or a call fails, an exception is raised.
"""
import ctypes as C
import os
import threading

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libsdfb200.so")

MAX_LEVELS = 32
MAX_LAYERS = 12

GRID_TORCH, GRID_TCNN = 0, 1
DT_F32, DT_F16 = 0, 1
CONTRACT_NONE, CONTRACT_LINF, CONTRACT_L2 = 0, 1, 2
SPACING = {"uniform": 0, "lindisp": 1, "sqrt": 2, "log": 3, "piecewise": 4, "identity": 5}
BG_COLOR, BG_LAST_SAMPLE, BG_PER_RAY = 0, 1, 2
CAMERA_PERSPECTIVE, CAMERA_FISHEYE = 1, 2
COLLIDER_AABB, COLLIDER_NEAR_FAR, COLLIDER_SPHERE = 0, 1, 2
PRECISION = {"fp32": 0, "bf16x3": 1, "bf16": 2}


class GridDesc(C.Structure):
    _fields_ = [
        ("layout", C.c_int32), ("n_levels", C.c_int32), ("n_features", C.c_int32), ("log2_hashmap_size", C.c_int32),
        ("smoothstep", C.c_int32), ("active_levels", C.c_int32), ("table_dtype", C.c_int32), ("reserved", C.c_int32),
        ("scale", C.c_float * MAX_LEVELS), ("resolution", C.c_uint32 * MAX_LEVELS), ("size", C.c_uint32 * MAX_LEVELS),
        ("offset", C.c_uint64 * MAX_LEVELS), ("hashed", C.c_uint8 * MAX_LEVELS),
    ]  # fmt: skip


class FieldDesc(C.Structure):
    _fields_ = [
        ("grid", GridDesc), ("use_grid_feature", C.c_int32), ("pe_degree", C.c_int32), ("use_position_encoding", C.c_int32),
        ("off_axis", C.c_int32), ("contraction", C.c_int32), ("n_geo_linear", C.c_int32),
        ("geo_dims", C.c_int32 * (MAX_LAYERS + 1)), ("geo_skip_layer", C.c_int32), ("n_color_linear", C.c_int32),
        ("color_dims", C.c_int32 * (MAX_LAYERS + 1)), ("appearance_dim", C.c_int32), ("use_diffuse_color", C.c_int32),
        ("use_specular_tint", C.c_int32), ("use_reflections", C.c_int32), ("use_n_dot_v", C.c_int32),
        ("use_numerical_gradients", C.c_int32), ("rgb_padding", C.c_float), ("precision", C.c_int32),
    ]  # fmt: skip


class FieldParams(C.Structure):
    _fields_ = [
        ("geo_weight_v", C.c_void_p * MAX_LAYERS), ("geo_weight_g", C.c_void_p * MAX_LAYERS), ("geo_bias", C.c_void_p * MAX_LAYERS),
        ("color_weight_v", C.c_void_p * MAX_LAYERS), ("color_weight_g", C.c_void_p * MAX_LAYERS), ("color_bias", C.c_void_p * MAX_LAYERS),
        ("diffuse_weight", C.c_void_p), ("diffuse_bias", C.c_void_p), ("tint_weight", C.c_void_p), ("tint_bias", C.c_void_p),
    ]  # fmt: skip


class FieldIn(C.Structure):
    _fields_ = [
        ("n_rays", C.c_int64), ("n_samples", C.c_int32), ("apply_contraction", C.c_int32), ("origins", C.c_void_p),
        ("directions", C.c_void_p), ("bins", C.c_void_p), ("appearance", C.c_void_p), ("variance", C.c_void_p), ("beta", C.c_void_p),
        ("beta_min", C.c_void_p), ("cos_anneal_ratio", C.c_float), ("numerical_delta", C.c_float),
    ]  # fmt: skip


class FieldOut(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("sdf", "geo_feature", "gradients", "normals", "rgb", "density", "alpha", "occupancy",
                                          "points_norm", "sampled_sdf", "points")]  # fmt: skip


class RenderOut(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("rgb", "depth", "normal", "accumulation", "steps_minmax")]


class FieldRender(C.Structure):
    _fields_ = [("from_density", C.c_int32), ("bg_mode", C.c_int32), ("clamp01", C.c_int32), ("clip_depth", C.c_int32), ("bg", C.c_void_p),
                ("weights", C.c_void_p), ("bg_transmittance", C.c_void_p), ("out", RenderOut)]


_lib = None
_lock = threading.Lock()

_i32, _i64, _f32, _vp, _sz = C.c_int32, C.c_int64, C.c_float, C.c_void_p, C.c_size_t
_PROTOS = {
    "sdfb200_version": (C.c_int, []),
    "sdfb200_last_error_string": (C.c_char_p, []),
    "sdfb200_launch_count": (_i64, []),
    "sdfb200_struct_size": (_sz, [_i32]),
    "sdfb200_grid_encode": (C.c_int, [C.POINTER(GridDesc), _vp, _vp, _i64, _vp, _i64, _vp, _vp]),
    "sdfb200_grid_encode_backward": (C.c_int, [C.POINTER(GridDesc), _vp, _vp, _vp, _i64, _vp, _vp, _vp]),
    "sdfb200_grid_encode_grouped": (C.c_int, [C.POINTER(GridDesc), _vp, _vp, _i64, _i32, _vp, _i64, _vp]),
    "sdfb200_grid_encode_backward_grouped": (C.c_int, [C.POINTER(GridDesc), _vp, _vp, _i64, _i32, _vp, _vp]),
    "sdfb200_grid_encode_backward_backward": (C.c_int, [C.POINTER(GridDesc), _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp]),
    "sdfb200_render_backward": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i32, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "sdfb200_weights_backward": (C.c_int, [_vp, _vp, _i32, _i64, _i32, _vp, _vp, _i32, _vp, _vp]),
    "sdfb200_generate_rays": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "sdfb200_collide": (C.c_int, [_vp, _vp, _i64, _i32, C.POINTER(C.c_float), _f32, _vp, _vp, _vp]),
    "sdfb200_lattice_points": (C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int32), _i64, _i64, _vp, _vp]),
    "sdfb200_field_packed_bytes": (_sz, [C.POINTER(FieldDesc)]),
    "sdfb200_field_pack": (C.c_int, [C.POINTER(FieldDesc), C.POINTER(FieldParams), _vp, _vp]),
    "sdfb200_field_workspace_bytes": (_sz, [C.POINTER(FieldDesc), _i64]),
    "sdfb200_field_forward": (C.c_int, [C.POINTER(FieldDesc), _vp, _vp, C.POINTER(FieldIn), C.POINTER(FieldOut), _vp, _sz, _vp]),
    "sdfb200_density_field_forward": (C.c_int, [C.POINTER(GridDesc), _vp, _vp, _i32, _i32, _i32, _vp, _vp, _i64, _vp, _vp, _vp]),
    "sdfb200_spaced_bins": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i64, _i32, _i32, _vp, _vp, _vp]),
    "sdfb200_bins_to_euclid": (C.c_int, [_vp, _vp, _vp, _i64, _i32, _i32, _vp, _vp]),
    "sdfb200_pdf_sample": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i64, _i32, _i32, _f32, _f32, _i32, _vp, _vp, _vp]),
    "sdfb200_merge_bins": (C.c_int, [_vp, _vp, _i64, _i32, _i32, _vp, _vp, _vp]),
    "sdfb200_merge_gather": (C.c_int, [_vp, _vp, _vp, _i64, _i32, _i32, _vp, _vp]),
    "sdfb200_neus_upsample_weights": (C.c_int, [_vp, _vp, _i64, _i32, _f32, _vp, _vp]),
    "sdfb200_volsdf_step": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _f32, _i32, _vp, _vp, _vp]),
    "sdfb200_volsdf_init_beta": (C.c_int, [_vp, _i64, _i32, _f32, _vp, _vp]),
    "sdfb200_unisurf_interval": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _f32, _vp, _vp, _vp, _vp, _vp]),
    "sdfb200_weights_from_alphas": (C.c_int, [_vp, _i64, _i32, _vp, _vp, _vp]),
    "sdfb200_weights_from_density": (C.c_int, [_vp, _vp, _i64, _i32, _vp, _vp, _vp]),
    "sdfb200_render": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i64, _i32, C.POINTER(RenderOut), _vp]),
    "sdfb200_render_alphas": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i64, _i32, _vp, _vp, C.POINTER(RenderOut), _vp]),
    "sdfb200_depth_clip": (C.c_int, [_vp, _vp, _i64, _vp]),
    "sdfb200_render_packed": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _i32, _i32, C.POINTER(RenderOut), _vp, _sz, _vp]),
    "sdfb200_gemm_workspace_bytes": (_sz, []),
    "sdfb200_gemm_nt": (C.c_int, [_i32, _vp, _i64, _vp, _i64, _i32, _i32, _vp, _i32, _vp, _i64, _i64, _vp, _sz, _vp]),
    "sdfb200_gemm_nn": (C.c_int, [_i32, _vp, _i64, _vp, _i64, _i32, _i32, _vp, _i64, _i64, _vp, _sz, _vp]),
    "sdfb200_gemm_tn": (C.c_int, [_i32, _vp, _i64, _vp, _i64, _vp, _i64, _i64, _i32, _i32, _vp, _sz, _vp]),
    "sdfb200_field_render_workspace_bytes": (_sz, [C.POINTER(FieldDesc), _i64, _i32]),
    "sdfb200_field_render": (C.c_int, [C.POINTER(FieldDesc), _vp, _vp, C.POINTER(FieldIn), C.POINTER(FieldOut), C.POINTER(FieldRender), _vp, _sz, _vp]),
}
EXPORTED_SYMBOLS = tuple(_PROTOS)
# validation hooks of the tensor-core building blocks: libsdfb200_dbg.so only (include/sdfb200_debug.h), never loaded by the product
_DEBUG_PROTOS = {
    "sdfb200_debug_tc_linear": (C.c_int, [_i32, _i32, _vp, _i32, _vp, _vp, _vp, _i32, _i64, _i32, _i32, _vp, _i32, _i32, _vp, _vp]),
    "sdfb200_debug_tc_gemm": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
}
_dbg = None


def load_debug():
    """libsdfb200_dbg.so = the product objects + the building-block test hooks (tests/test_gpu_tc.py)."""
    global _dbg
    if _dbg is None:
        path = os.path.join(HERE, "libsdfb200_dbg.so")
        if not os.path.exists(path):
            from . import build as _build

            _build.build(force=True)
        lib = C.CDLL(path)
        for name, (res, args) in _DEBUG_PROTOS.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        lib.sdfb200_last_error_string.restype = C.c_char_p
        _dbg = lib
    return _dbg


class Sdfb200Error(RuntimeError):
    pass


def load():
    """Load (building first if the sources are newer and nvcc exists).  Raises when unavailable -- never falls back."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            from . import build as _build

            _build.build()
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _PROTOS.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        for which, st in enumerate((GridDesc, FieldDesc, FieldParams, FieldIn, FieldOut, RenderOut, FieldRender)):
            if lib.sdfb200_struct_size(which) != C.sizeof(st):
                raise Sdfb200Error(f"ABI mismatch: sizeof({st.__name__}) = {C.sizeof(st)} but the library says {lib.sdfb200_struct_size(which)}")
        _lib = lib
    return _lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().sdfb200_last_error_string().decode(errors="replace")
        raise Sdfb200Error(f"{what or 'sdfb200 call'} failed with code {rc}: {msg}")


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    """device pointer of a tensor (None -> NULL).  The tensor must be contiguous."""
    if t is None:
        return None
    assert t.is_cuda, "sdfb200 kernels need CUDA tensors (there is no CPU path)"
    assert t.is_contiguous(), "sdfb200 kernels need contiguous tensors"
    return t.data_ptr()


def f32c(t):
    """contiguous fp32 view/copy (handles the reference's stride-0 expanded TensorDataclass fields)."""
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def launch_count() -> int:
    return int(load().sdfb200_launch_count())
