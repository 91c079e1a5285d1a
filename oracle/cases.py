"""TEST INFRASTRUCTURE -- the named parity cases shared by ``make_golden.py`` (reference side) and ``tests/`` (oracle and
CUDA side).  Every case is fully determined by a seed: parameters come from ``oracle.field.init_params`` (a torch CPU
generator is bit-reproducible across machines), rays from ``synthetic_rays``.
"""
import math
from dataclasses import replace
from typing import Dict, Tuple

import torch

from .field import FieldSpec

# name -> (FieldSpec, dict(R, S, near, far, init kwargs, extras))
CASES: Dict[str, Tuple[FieldSpec, dict]] = {
    # BASELINE.json configs[0]: neus-facto SDFField, 256 rays x 32 samples, torch-layout HashEncoding
    "neusfacto_c1": (
        FieldSpec(num_layers=2, num_layers_color=2, hidden_dim=256, use_grid_feature=True),
        dict(R=256, S=32, near=0.5, far=4.5, bias=0.5, beta_init=0.3, perturb=0.02, hash_init_scale=0.05, seed=1),
    ),
    # same shape, pure geometric init (hash / PE columns of glin0 are exactly zero)
    "neusfacto_c1_init": (
        FieldSpec(num_layers=2, num_layers_color=2, hidden_dim=256, use_grid_feature=True),
        dict(R=64, S=16, near=0.5, far=4.5, bias=0.5, beta_init=0.3, perturb=0.0, hash_init_scale=1e-3, seed=2),
    ),
    # neus-facto-angelo shaped (method_configs.py:404-432), reduced table: numerical gradients, F=8, linear interp,
    # 1 hidden geo layer, 4 colour layers, PE zeroed, progressive mask at level 6 of 8
    "angelo_small": (
        FieldSpec(num_layers=1, num_layers_color=4, hidden_dim=256, use_grid_feature=True, use_appearance_embedding=True,
                  use_numerical_gradients=True, base_res=16, max_res=512, num_levels=8, log2_hashmap_size=15,
                  hash_features_per_level=8, hash_smoothstep=False, use_position_encoding=False),
        dict(R=64, S=16, near=0.5, far=4.5, bias=0.5, beta_init=0.3, perturb=0.02, hash_init_scale=0.05, seed=3, mask_level=6,
             num_grad_delta=0.002),
    ),
    # bakedsdf shaped (method_configs.py:265-292), reduced table: L-inf contraction, off-axis PE deg 8, ref-nerf heads
    "bakedsdf_small": (
        FieldSpec(num_layers=2, num_layers_color=2, hidden_dim=256, use_grid_feature=True, position_encoding_max_degree=8,
                  use_diffuse_color=True, use_specular_tint=True, use_reflections=True, use_n_dot_v=True, off_axis=True,
                  log2_hashmap_size=15, contraction="linf"),
        dict(R=64, S=24, near=0.2, far=30.0, bias=0.05, beta_init=0.1, perturb=0.02, hash_init_scale=0.05, seed=4, spacing="piecewise"),
    ),
    # stock volsdf preset (method_configs.py:635 + sdf_field.py defaults): 8x256 MLP, no grid, skip connection at 4
    "volsdf_stock": (
        FieldSpec(num_layers=8, num_layers_color=4, hidden_dim=256, use_grid_feature=False),
        dict(R=64, S=16, near=0.5, far=4.5, bias=0.8, beta_init=0.1, perturb=0.01, seed=5, inside_outside=True),
    ),
}

# cases pinned on the CPU side only (oracle vs reference golden): they widen what the oracle is pinned on without adding GPU test shapes
CPU_CASES: Dict[str, Tuple[FieldSpec, dict]] = {
    # neus-facto shape behind the default (L2) SceneContraction (spatial_distortions.py:66-73, order=None), unbounded far plane
    "neusfacto_l2": (
        FieldSpec(num_layers=2, num_layers_color=2, hidden_dim=256, use_grid_feature=True, log2_hashmap_size=15, contraction="l2"),
        dict(R=64, S=24, near=0.2, far=30.0, bias=0.5, beta_init=0.3, perturb=0.02, hash_init_scale=0.05, seed=6, spacing="piecewise"),
    ),
    # branches of get_colors / the grid no other case combines (sdf_field.py:532-612): reflections + n.v WITHOUT the diffuse / tint heads,
    # appearance embedding on, narrower MLPs (128 / 192 / 96), 3 colour layers, F = 4 linear hash grid, inside_outside geometry
    "mixed_heads": (
        FieldSpec(num_layers=2, num_layers_color=3, hidden_dim=128, hidden_dim_color=192, geo_feat_dim=96, use_grid_feature=True, num_levels=8, max_res=256,
                  log2_hashmap_size=14, hash_features_per_level=4, hash_smoothstep=False, use_appearance_embedding=True, use_reflections=True, use_n_dot_v=True,
                  position_encoding_max_degree=4),
        dict(R=48, S=20, near=0.5, far=4.5, bias=0.6, beta_init=0.2, perturb=0.02, hash_init_scale=0.05, seed=7, inside_outside=True, spacing="lindisp"),
    ),
}

# the training-mode sampler golden (make_golden_samplers_train.py): the first TRAIN_SAMPLER_RAYS rays of this case (its
# sdf crosses zero on most of them, so UniSurf finds surfaces).  The ErrorBoundedSampler runs at beta0 = TRAIN_SAMPLER_BETA0
# in place of the field's beta: small enough that it does not converge and runs all of max_total_iters = 5 iterations.
TRAIN_SAMPLER_CASE = "neusfacto_c1_init"
TRAIN_SAMPLER_RAYS = 32
TRAIN_SAMPLER_BETA0 = 0.005


def proposal_density(positions, level: int):
    """Analytic density [..., 1] for the proposal levels of the training-mode sampler golden: a shell of radius 0.5 (the
    case's sphere), sharper at the second level.  Plain torch ops, so the reference, the oracle and the GPU tests (on CPU
    copies of the positions) evaluate it to the same bits."""
    r = positions.norm(dim=-1, keepdim=True)
    width = 0.05 if level == 0 else 0.02
    return 50.0 * torch.exp(-(((r - 0.5) / width) ** 2)) + 0.1


def synthetic_rays(R: int, seed: int, radius: float = 2.7, dtype=torch.float32):
    """DTU-shaped synthetic rays (SURVEY.md section 8d config 2): cameras on a sphere of radius ~2.7 looking at the origin
    through a 384x384 pinhole (fx~925), uniformly random pixels.  Returns origins, unit directions, camera_indices."""
    g = torch.Generator().manual_seed(seed)
    n_views = 49
    cam = torch.randn(n_views, 3, generator=g)
    cam = cam / cam.norm(dim=-1, keepdim=True) * radius
    idx = torch.randint(0, n_views, (R,), generator=g)
    o = cam[idx]
    fwd = -o / o.norm(dim=-1, keepdim=True)
    up = torch.tensor([0.0, 0.0, 1.0]).expand_as(fwd)
    right = torch.linalg.cross(fwd, up)
    right = right / right.norm(dim=-1, keepdim=True).clamp_min(1e-6)
    up2 = torch.linalg.cross(right, fwd)
    px = torch.rand(R, 2, generator=g) * 384.0
    x = (px[:, 0:1] - 199.4) / 925.5
    y = (px[:, 1:2] - 198.1) / 922.6
    d = fwd + x * right + y * up2
    d = d / d.norm(dim=-1, keepdim=True)
    return o.to(dtype).contiguous(), d.to(dtype).contiguous(), idx


def case_inputs(name: str):
    spec, kw = CASES[name] if name in CASES else CPU_CASES[name]
    o, d, cam = synthetic_rays(kw["R"], kw["seed"] + 1000)
    nears = torch.full((kw["R"], 1), kw["near"])
    fars = torch.full((kw["R"], 1), kw["far"])
    return spec, kw, o, d, cam, nears, fars


def init_kwargs(kw: dict):
    return dict(bias=kw["bias"], beta_init=kw["beta_init"], perturb=kw.get("perturb", 0.0), seed=kw["seed"],
                hash_init_scale=kw.get("hash_init_scale", 1e-3), inside_outside=kw.get("inside_outside", False))
