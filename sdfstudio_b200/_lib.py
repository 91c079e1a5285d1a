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
INTERLEVEL_OUTER, INTERLEVEL_ZIP = 0, 1


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


class NerfactoDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("hidden_dim", "n_hidden_layers", "hidden_dim_color", "n_hidden_layers_color", "geo_feat_dim",
                                         "appearance_dim", "contraction", "n_samples")]  # fmt: skip


NERF_MAX_FREQS = 10


class NerfFieldDesc(C.Structure):
    _fields_ = [
        ("base_layers", C.c_int32), ("base_width", C.c_int32), ("skip_layer", C.c_int32), ("head_layers", C.c_int32), ("head_width", C.c_int32),
        ("pe_frequencies", C.c_int32), ("pe_include_input", C.c_int32), ("pe_freqs", C.c_float * NERF_MAX_FREQS),
        ("dir_frequencies", C.c_int32), ("dir_include_input", C.c_int32), ("dir_freqs", C.c_float * NERF_MAX_FREQS),
        ("contraction", C.c_int32), ("n_samples", C.c_int32), ("precision", C.c_int32),
    ]  # fmt: skip


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
    "sdfb200_render_packed_backward": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                                 _vp]),
    "sdfb200_weights_backward": (C.c_int, [_vp, _vp, _i32, _i64, _i32, _vp, _vp, _i32, _vp, _vp]),
    "sdfb200_interlevel_loss": (C.c_int, [_vp, _vp, _i32, _vp, _vp, _i32, _i64, _i32, _f32, _vp, _vp, _vp, _vp]),
    "sdfb200_generate_rays": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "sdfb200_collide": (C.c_int, [_vp, _vp, _i64, _i32, C.POINTER(C.c_float), _f32, _vp, _vp, _vp]),
    "sdfb200_lattice_points": (C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int32), _i64, _i64, _vp, _vp]),
    "sdfb200_marching_cubes_workspace_bytes": (_sz, [C.POINTER(C.c_int64)]),
    "sdfb200_marching_cubes": (C.c_int, [_vp, C.POINTER(C.c_int64), _f32, _vp, C.POINTER(C.c_float), C.POINTER(C.c_float), _vp, _vp, _vp, _vp, _vp,
                                         _vp]),
    "sdfb200_uv_rasterize": (C.c_int, [_vp, _i64, _i32, _vp, _i32, _vp, _i32, _vp, _vp, _vp]),
    "sdfb200_uv_unwrap_grid": (C.c_int, [_vp, _vp, _i64, _i32, _i32, _vp, _i32, _vp, _i32, _vp, _vp, _vp, _vp]),
    "sdfb200_uv_texel_rays": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp]),
    "sdfb200_tsdf_integrate": (C.c_int, [_vp, _i64, _vp, _i32, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "sdfb200_knn": (C.c_int, [_vp, _vp, _i64, _vp, C.POINTER(C.c_float), _i32, _i32, _vp, _vp, _vp]),
    "sdfb200_point_normals": (C.c_int, [_vp, _i64, _vp, _i32, _vp, _vp]),
    "sdfb200_mesh_rasterize": (C.c_int, [_vp, _vp, _i64, _vp, _i32, _i32, _i32, _f32, _vp, _vp]),
    "sdfb200_mesh_shade": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _i64, _vp, _vp, C.POINTER(C.c_float), _vp, _vp, _vp]),
    "sdfb200_poisson_cells": (C.c_int, [_vp, _vp, _vp, _i64, _vp, _vp, _i32, C.POINTER(C.c_double), C.c_double, _vp, _vp, _vp, _vp]),
    "sdfb200_poisson_coarsen": (C.c_int, [_i32, _vp, _vp, _i64, _vp, _vp, _vp]),
    "sdfb200_poisson_gather": (C.c_int, [_i32, _vp, _vp, _i32, _i32, _i32, _vp, _vp]),
    "sdfb200_poisson_sample": (C.c_int, [_vp, _i64, _i32, C.POINTER(C.c_double), C.c_double, _vp, _i32, _vp, _vp]),
    "sdfb200_poisson_apply": (C.c_int, [_i32, C.c_double, _vp, _vp, C.c_double, _vp, _vp, _vp]),
    "sdfb200_poisson_workspace_bytes": (_sz, [_i32]),
    "sdfb200_poisson_solve": (C.c_int, [_i32, C.c_double, C.POINTER(_vp), C.POINTER(_vp), C.c_double, _vp, _vp, _i32, C.c_double, _vp, _sz,
                                        C.POINTER(C.c_int32), C.POINTER(C.c_double), _vp]),
    "sdfb200_poisson_sum": (C.c_int, [_vp, _i64, _vp, _vp, _vp]),
    "sdfb200_field_packed_bytes": (_sz, [C.POINTER(FieldDesc)]),
    "sdfb200_field_pack": (C.c_int, [C.POINTER(FieldDesc), C.POINTER(FieldParams), _vp, _vp]),
    "sdfb200_field_workspace_bytes": (_sz, [C.POINTER(FieldDesc), _i64]),
    "sdfb200_field_forward": (C.c_int, [C.POINTER(FieldDesc), _vp, _vp, C.POINTER(FieldIn), C.POINTER(FieldOut), _vp, _sz, _vp]),
    "sdfb200_density_field_forward": (C.c_int, [C.POINTER(GridDesc), _vp, _vp, _i32, _i32, _i32, _vp, _vp, _i64, _vp, _vp, _vp]),
    "sdfb200_nerfacto_field_forward": (C.c_int, [C.POINTER(GridDesc), C.POINTER(NerfactoDesc), _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _i64,
                                                 _vp, _vp, _vp, _vp, _vp]),
    "sdfb200_nerf_field_in_family": (C.c_int, [C.POINTER(NerfFieldDesc)]),
    "sdfb200_nerf_field_packed_bytes": (_sz, [C.POINTER(NerfFieldDesc)]),
    "sdfb200_nerf_field_pack": (C.c_int, [C.POINTER(NerfFieldDesc), C.POINTER(_vp), C.POINTER(_vp), _vp, _vp]),
    "sdfb200_nerf_field_forward": (C.c_int, [C.POINTER(NerfFieldDesc), _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp]),
    "sdfb200_spaced_bins":(C.c_int, [_vp, _vp, _vp, _vp, _i32, _i64, _i32, _i32, _vp, _vp, _vp]),
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
    "sdfb200_packed_weights": (C.c_int, [_vp, _vp, _i64, _vp, _vp]),
    "sdfb200_packed_accumulate": (C.c_int, [_vp, _vp, _i32, _vp, _i64, _vp, _vp]),
    "sdfb200_packed_weights_backward": (C.c_int, [_vp, _vp, _i64, _vp, _vp, _vp]),
    "sdfb200_packed_accumulate_backward": (C.c_int, [_vp, _vp, _i32, _vp, _i64, _vp, _vp, _vp, _vp]),
    "sdfb200_occupancy_prune": (C.c_int, [_vp, _vp, _i64, _f32, _f32, _vp, _f32, _vp, _vp]),
    "sdfb200_occupancy_march": (C.c_int, [_vp, _vp, _vp, _vp, _i64, C.POINTER(C.c_float), _vp, _i32, _f32, _vp, _vp, _vp, _vp, _vp, _vp]),
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
    "sdfb200_debug_mesh_rasterize": (C.c_int, [_vp, _vp, _i64, _vp, _i32, _i32, _i32, _f32, _vp, _i64, _vp]),
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
        for which, st in enumerate((GridDesc, FieldDesc, FieldParams, FieldIn, FieldOut, RenderOut, FieldRender, NerfactoDesc, NerfFieldDesc)):
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


def require_cuda(dev, what: str):
    if dev.type != "cuda":
        raise RuntimeError(f"sdfstudio_b200.{what} runs on CUDA only (there is no CPU path)")


def render_out(rgb=None, depth=None, normal=None, accumulation=None, steps_minmax=None) -> RenderOut:
    """sdfb200_render_out_t over the given tensors (None -> NULL: that output is not written)."""
    return RenderOut(ptr(rgb), ptr(depth), ptr(normal), ptr(accumulation), ptr(steps_minmax))


_MINMAX_SEED = {}


def steps_minmax_seed(dev):
    """{+inf, -inf}, the start value of steps_minmax, cached on `dev` so that a call makes no host->device copy.  Shared: clone it or
    copy it into the output, never write into it."""
    t = _MINMAX_SEED.get(str(dev))
    if t is None:
        t = _MINMAX_SEED[str(dev)] = torch.tensor([float("inf"), float("-inf")], device=dev, dtype=torch.float32)
    return t


def packed_key(params, precision):
    """Cache key of a blob packed from `params`: it changes when a parameter is reallocated or modified in place."""
    return tuple((p.data_ptr(), p._version) for p in params), precision


def launch_count() -> int:
    return int(load().sdfb200_launch_count())
