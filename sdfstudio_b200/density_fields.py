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
from .encoding import make_grid_desc


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


class _GridFn(torch.autograd.Function):
    """hash-grid features of the flat tcnn-style parameter vector (grid table = its tail): forward / backward kernels of the
    Encoding operator, gradient scattered into the tail of d(params)."""

    @staticmethod
    def forward(ctx, x01, params, nb):
        lib = _lib.load()
        x = _lib.f32c(x01)
        n = x.shape[0]
        desc = nb.desc
        desc.active_levels, desc.table_dtype = desc.n_levels, _lib.DT_F32
        out = torch.empty(n, nb.in_dim, device=x.device, dtype=torch.float32)
        table = params.detach()[nb.n_net:]
        _lib.check(lib.sdfb200_grid_encode(desc, table.data_ptr(), _lib.ptr(x), n, _lib.ptr(out), nb.in_dim, None, _lib.stream_ptr()), "sdfb200_grid_encode")
        ctx.save_for_backward(x, params)
        ctx.nb = nb
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dout):
        lib = _lib.load()
        x, params = ctx.saved_tensors
        nb = ctx.nb
        dout = _lib.f32c(dout)
        dparams = torch.zeros_like(params, dtype=torch.float32)
        dx = torch.zeros_like(x) if ctx.needs_input_grad[0] else None
        table = params.detach()[nb.n_net:]
        _lib.check(lib.sdfb200_grid_encode_backward(nb.desc, table.data_ptr(), _lib.ptr(x), _lib.ptr(dout), x.shape[0], dparams[nb.n_net:].data_ptr(),
                                                    _lib.ptr(dx), _lib.stream_ptr()), "sdfb200_grid_encode_backward")
        return dx, dparams, None


class _NetworkWithInputEncoding(nn.Module):
    def __init__(self, n_levels, n_features, log2_hashmap_size, base_res, per_level_scale, hidden_dim, n_hidden_layers, seed=1337):
        super().__init__()
        self.hidden_dim, self.n_hidden_layers = hidden_dim, n_hidden_layers
        self.in_dim = n_levels * n_features
        self.in_pad = (self.in_dim + 15) // 16 * 16
        self.desc = make_grid_desc("tcnn", n_levels, n_features, log2_hashmap_size, base_res, per_level_scale, False)
        self.n_out_pad = 16                                   # tcnn pads the output layer to 16 neurons
        self.n_net = hidden_dim * self.in_pad + (n_hidden_layers - 1) * hidden_dim * hidden_dim + self.n_out_pad * hidden_dim
        self.n_grid = self.desc._total_entries * n_features
        g = torch.Generator().manual_seed(seed)
        # tcnn: xavier-uniform weights, U(-1e-4, 1e-4) grid
        w0 = (torch.rand(hidden_dim, self.in_pad, generator=g) * 2 - 1) * math.sqrt(6.0 / (self.in_pad + hidden_dim))
        w0[:, self.in_dim:] = 0.0
        ws = [w0.reshape(-1)]
        for _ in range(n_hidden_layers - 1):
            ws.append(((torch.rand(hidden_dim, hidden_dim, generator=g) * 2 - 1) * math.sqrt(6.0 / (2 * hidden_dim))).reshape(-1))
        wo = torch.zeros(self.n_out_pad, hidden_dim)
        wo[0] = (torch.rand(hidden_dim, generator=g) * 2 - 1) * math.sqrt(6.0 / (hidden_dim + 16))
        ws.append(wo.reshape(-1))
        grid = (torch.rand(self.n_grid, generator=g) * 2 - 1) * 1e-4
        self.params = nn.Parameter(torch.cat(ws + [grid]))

    @property
    def weights(self):
        return self.params[: self.n_net]

    @property
    def table(self):
        return self.params[self.n_net:]


class HashMLPDensityField(nn.Module):
    """density_fields.py:40-121."""

    def __init__(self, aabb, num_layers: int = 2, hidden_dim: int = 64, spatial_distortion=None, use_linear=False, num_levels=8, max_res=1024,
                 base_res=16, log2_hashmap_size=18, features_per_level=2) -> None:
        super().__init__()
        if use_linear:
            raise NotImplementedError("use_linear=True (encoding + nn.Linear) is not used by any SDF preset")
        if hidden_dim not in (16, 32, 64):
            raise NotImplementedError("hidden_dim must be 16, 32 or 64")
        self.aabb = nn.Parameter(torch.as_tensor(aabb, dtype=torch.float32), requires_grad=False)
        self.spatial_distortion = spatial_distortion
        self.use_linear = use_linear
        growth = float(np.exp((np.log(max_res) - np.log(base_res)) / (num_levels - 1)))
        self.mlp_base = _NetworkWithInputEncoding(num_levels, features_per_level, log2_hashmap_size, base_res, growth, hidden_dim, num_layers - 1)

    def _contraction_code(self):
        sd = self.spatial_distortion
        if sd is None:
            return None
        order = getattr(sd, "order", None)
        if order is None:
            return _lib.CONTRACT_L2
        if order == float("inf"):
            return _lib.CONTRACT_LINF
        raise NotImplementedError(f"SceneContraction order {order!r}")

    def density_from_positions(self, positions: torch.Tensor, return_pre_activation: bool = False):
        """positions [..., 3] -> density [..., 1] (fields/base_field.py:48-65 + density_fields.py:98-118)."""
        if torch.is_grad_enabled() and self.training and self.mlp_base.params.requires_grad:
            return self._density_differentiable(positions, return_pre_activation)
        lib = _lib.load()
        pos = _lib.f32c(positions.reshape(-1, 3))
        n = pos.shape[0]
        dens = torch.empty(n, device=pos.device, dtype=torch.float32)
        pre = torch.empty_like(dens) if return_pre_activation else None
        code = self._contraction_code()
        aabb = None if code is not None else _lib.f32c(self.aabb.detach())
        nb = self.mlp_base
        p = nb.params.detach()
        w, table = p[: nb.n_net], p[nb.n_net:]
        desc = nb.desc
        desc.active_levels = desc.n_levels
        desc.table_dtype = _lib.DT_F32
        _lib.check(lib.sdfb200_density_field_forward(desc, table.data_ptr(), w.data_ptr(), nb.hidden_dim, nb.n_hidden_layers, code or 0, _lib.ptr(aabb),
                                                     _lib.ptr(pos), n, _lib.ptr(dens), _lib.ptr(pre), _lib.stream_ptr()), "sdfb200_density_field_forward")
        dens = dens.view(*positions.shape[:-1], 1)
        return (dens, pre.view(*positions.shape[:-1], 1)) if return_pre_activation else dens

    def _density_differentiable(self, positions, return_pre_activation=False):
        """Training path (the interlevel loss trains the proposal networks, models/neus_facto.py): the hash grid through this package's
        twice-differentiable operator (sdfb200_grid_encode / _backward), the width-16..64 ReLU MLP through ATen, trunc_exp with the
        reference's clipped backward (field_components/activations.py:24-42)."""
        nb = self.mlp_base
        x = positions.reshape(-1, 3)
        if self.spatial_distortion is not None:
            x01 = (self.spatial_distortion(x) + 2.0) / 4.0
        else:
            x01 = (x - self.aabb[0]) / (self.aabb[1] - self.aabb[0])                  # SceneBox.get_normalized_positions
        feat = _GridFn.apply(x01, nb.params, nb)
        w = nb.params[: nb.n_net]
        o = nb.hidden_dim * nb.in_pad
        h = torch.relu(feat @ w[:o].view(nb.hidden_dim, nb.in_pad)[:, : nb.in_dim].t())
        for _ in range(nb.n_hidden_layers - 1):
            h = torch.relu(h @ w[o: o + nb.hidden_dim * nb.hidden_dim].view(nb.hidden_dim, nb.hidden_dim).t())
            o += nb.hidden_dim * nb.hidden_dim
        pre = (h @ w[o: o + nb.hidden_dim]).view(*positions.shape[:-1], 1)
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
