"""H100-native drop-in for ``nerfstudio.fields.density_fields.HashMLPDensityField`` (the proposal networks of
neus-facto / bakedsdf, density_fields.py:40-121): same constructor, ``get_density``, ``density_fn``.  The reference builds a
``tcnn.NetworkWithInputEncoding`` (HashGrid + FullyFusedMLP, ReLU, no biases, output activation None) and applies
``trunc_exp``; here one fused kernel (sdfb200_density_field_forward) does lookup + MLP + exp.

Parameters: ``mlp_base.params`` is ONE flat fp32 tensor like tcnn's ``NetworkWithInputEncoding``: network weights first (row-major
[hidden, in_pad], (n_hidden - 1) x [hidden, hidden], output matrix [16, hidden] = the single output neuron padded to tcnn's 16-row
granularity, row 0 live; in_pad = L*F rounded up to 16), then the grid table in tcnn level layout -- so the element count equals a
reference ``proposal_networks.{i}.mlp_base.params`` and ``checkpoint.load_density_field_checkpoint`` can load it.  tiny-cuda-nn is not
vendored in the reference, so the ORDERING inside that vector is restated from tcnn's published layout and is UNPINNED (DESIGN.md section 4).
"""
import math
from typing import Optional

import numpy as np
import torch
from torch import nn

from . import _lib
from .autograd_ops import training_step
from .encoding import _GridFn, make_grid_desc
from .spatial_distortions import contraction_code


class _TruncExp(torch.autograd.Function):
    """field_components/activations.py:24-38: exp forward, gradient g * exp(clamp(x, -15, 15))."""

    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return torch.exp(x)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return g * torch.exp(x.clamp(-15, 15))


def fully_fused_weights(g: torch.Generator, in_dim: int, hidden_dim: int, n_hidden_layers: int, n_output_dims: int) -> torch.Tensor:
    """Initial weights of a tcnn FullyFusedMLP (ReLU, no biases) as one flat vector: xavier-uniform [hidden, in_pad] (padded input
    columns zero) | (n_hidden_layers - 1) x [hidden, hidden] | [16, hidden] (the output padded to 16 rows, rows >= n_output_dims zero)."""
    in_pad = (in_dim + 15) // 16 * 16
    w0 = (torch.rand(hidden_dim, in_pad, generator=g) * 2 - 1) * math.sqrt(6.0 / (in_pad + hidden_dim))
    w0[:, in_dim:] = 0.0
    ws = [w0.reshape(-1)]
    for _ in range(n_hidden_layers - 1):
        ws.append(((torch.rand(hidden_dim, hidden_dim, generator=g) * 2 - 1) * math.sqrt(6.0 / (2 * hidden_dim))).reshape(-1))
    wo = torch.zeros(16, hidden_dim)
    wo[:n_output_dims] = (torch.rand(n_output_dims, hidden_dim, generator=g) * 2 - 1) * math.sqrt(6.0 / (hidden_dim + 16))
    ws.append(wo.reshape(-1))
    return torch.cat(ws)


def fully_fused_mlp(x: torch.Tensor, w: torch.Tensor, in_dim: int, in_pad: int, hidden_dim: int, n_hidden_layers: int, n_output_dims: int):
    """A FullyFusedMLP over the flat weights `w` (layout of fully_fused_weights), through ATen on views of `w` so that autograd reaches
    it: [N, in_dim] -> the live output rows [N, n_output_dims] (no output activation)."""
    o = hidden_dim * in_pad
    h = torch.relu(x @ w[:o].view(hidden_dim, in_pad)[:, :in_dim].t())
    for _ in range(n_hidden_layers - 1):
        h = torch.relu(h @ w[o: o + hidden_dim * hidden_dim].view(hidden_dim, hidden_dim).t())
        o += hidden_dim * hidden_dim
    return h @ w[o: o + 16 * hidden_dim].view(16, hidden_dim)[:n_output_dims].t()


def normalized_positions(positions: torch.Tensor, aabb: torch.Tensor, spatial_distortion) -> torch.Tensor:
    """Positions -> the grid's unit cube: SceneContraction then (x + 2) / 4 when there is a spatial distortion, else
    SceneBox.get_normalized_positions."""
    if spatial_distortion is not None:
        return (spatial_distortion(positions) + 2.0) / 4.0
    return (positions - aabb[0]) / (aabb[1] - aabb[0])


def kernel_aabb(aabb: torch.Tensor, code: int) -> Optional[torch.Tensor]:
    """The aabb of a field kernel call with contraction `code`: the kernels normalise with it only when there is no contraction."""
    return _lib.f32c(aabb.detach()) if code == _lib.CONTRACT_NONE else None


class _NetworkWithInputEncoding(nn.Module):
    """tcnn.NetworkWithInputEncoding(HashGrid, FullyFusedMLP with ReLU and no biases) as one flat parameter vector: network weights
    ([hidden, in_pad] | (n_hidden - 1) x [hidden, hidden] | [16, hidden], rows 0..n_output_dims-1 of the output matrix live), then the
    grid table.  The proposal networks use one output, the nerfacto field 1 + geo_feat_dim."""

    def __init__(self, n_levels, n_features, log2_hashmap_size, base_res, per_level_scale, hidden_dim, n_hidden_layers, seed=1337, n_output_dims=1):
        super().__init__()
        if not 1 <= n_output_dims <= 16:
            raise NotImplementedError("n_output_dims must be 1..16 (one padded output block)")
        self.hidden_dim, self.n_hidden_layers, self.n_output_dims = hidden_dim, n_hidden_layers, n_output_dims
        self.in_dim = n_levels * n_features
        self.in_pad = (self.in_dim + 15) // 16 * 16
        self.desc = make_grid_desc("tcnn", n_levels, n_features, log2_hashmap_size, base_res, per_level_scale, False)
        self.n_out_pad = 16                                   # tcnn pads the output layer to 16 neurons
        self.n_net = hidden_dim * self.in_pad + (n_hidden_layers - 1) * hidden_dim * hidden_dim + self.n_out_pad * hidden_dim
        self.n_grid = self.desc._total_entries * n_features
        g = torch.Generator().manual_seed(seed)
        w = fully_fused_weights(g, self.in_dim, hidden_dim, n_hidden_layers, n_output_dims)
        grid = (torch.rand(self.n_grid, generator=g) * 2 - 1) * 1e-4   # tcnn: U(-1e-4, 1e-4) grid
        self.params = nn.Parameter(torch.cat([w, grid]))

    @property
    def weights(self):
        return self.params[: self.n_net]

    @property
    def table(self):
        return self.params[self.n_net:]

    def kernel_desc(self) -> "_lib.GridDesc":
        """The grid descriptor of a kernel call on this network's table: every level active, fp32."""
        self.desc.active_levels, self.desc.table_dtype = self.desc.n_levels, _lib.DT_F32
        return self.desc

    def forward(self, x01: torch.Tensor) -> torch.Tensor:
        """The differentiable pass: [N, 3] in [0, 1] -> [N, n_output_dims] (no output activation)."""
        feat = _GridFn.apply(x01, self.params, self)
        return fully_fused_mlp(feat, self.params[: self.n_net], self.in_dim, self.in_pad, self.hidden_dim, self.n_hidden_layers, self.n_output_dims)


class HashMLPDensityField(nn.Module):
    """density_fields.py:40-121."""

    def __init__(self, aabb, num_layers: int = 2, hidden_dim: int = 64, spatial_distortion=None, use_linear=False, num_levels=8, max_res=1024,
                 base_res=16, log2_hashmap_size=18, features_per_level=2) -> None:
        super().__init__()
        if use_linear:
            raise NotImplementedError("use_linear=True (encoding + nn.Linear) is not used by any SDF preset")
        if hidden_dim not in (16, 32, 64):
            raise NotImplementedError("hidden_dim must be 16, 32 or 64")
        if num_layers not in (2, 3, 4, 5):
            raise NotImplementedError("num_layers must be 2, 3, 4 or 5")
        if features_per_level not in (1, 2, 4, 8):
            raise NotImplementedError("features_per_level must be 1, 2, 4 or 8")
        self.aabb = nn.Parameter(torch.as_tensor(aabb, dtype=torch.float32), requires_grad=False)
        self.spatial_distortion = spatial_distortion
        self.use_linear = use_linear
        growth = float(np.exp((np.log(max_res) - np.log(base_res)) / (num_levels - 1)))
        self.mlp_base = _NetworkWithInputEncoding(num_levels, features_per_level, log2_hashmap_size, base_res, growth, hidden_dim, num_layers - 1)

    def density_from_positions(self, positions: torch.Tensor, return_pre_activation: bool = False):
        """positions [..., 3] -> density [..., 1] (fields/base_field.py:48-65 + density_fields.py:98-118)."""
        if training_step(self, (self.mlp_base.params,)):
            return self._density_differentiable(positions, return_pre_activation)
        lib = _lib.load()
        pos = _lib.f32c(positions.reshape(-1, 3))
        n = pos.shape[0]
        dens = torch.empty(n, device=pos.device, dtype=torch.float32)
        pre = torch.empty_like(dens) if return_pre_activation else None
        code = contraction_code(self.spatial_distortion)
        aabb = kernel_aabb(self.aabb, code)
        nb = self.mlp_base
        p = nb.params.detach()
        _lib.check(lib.sdfb200_density_field_forward(nb.kernel_desc(), p[nb.n_net:].data_ptr(), p.data_ptr(), nb.hidden_dim, nb.n_hidden_layers, code,
                                                     _lib.ptr(aabb), _lib.ptr(pos), n, _lib.ptr(dens), _lib.ptr(pre), _lib.stream_ptr()),
                   "sdfb200_density_field_forward")
        dens = dens.view(*positions.shape[:-1], 1)
        return (dens, pre.view(*positions.shape[:-1], 1)) if return_pre_activation else dens

    def _density_differentiable(self, positions, return_pre_activation=False):
        """Training path (the interlevel loss trains the proposal networks, models/neus_facto.py): the hash grid through this package's
        twice-differentiable operator (sdfb200_grid_encode / _backward), the width-16..64 ReLU MLP through ATen, trunc_exp with the
        reference's clipped backward (field_components/activations.py:24-42)."""
        x01 = normalized_positions(positions.reshape(-1, 3), self.aabb, self.spatial_distortion)
        pre = self.mlp_base(x01).view(*positions.shape[:-1], 1)
        dens = _TruncExp.apply(pre)
        return (dens, pre) if return_pre_activation else dens

    def density_fn(self, positions: torch.Tensor) -> torch.Tensor:
        return self.density_from_positions(positions)

    def get_density(self, ray_samples):
        return self.density_from_positions(ray_samples.frustums.get_positions()), None

    def get_outputs(self, ray_samples, density_embedding: Optional[torch.Tensor] = None):
        return {}

    def forward(self, ray_samples):
        density, _ = self.get_density(ray_samples)
        return {"density": density}
