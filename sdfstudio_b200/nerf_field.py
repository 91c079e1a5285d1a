"""H100-native drop-in for ``nerfstudio.fields.vanilla_nerf_field.NeRFField`` (vanilla_nerf_field.py:37-114), the field behind
``background_model="mlp"``, the default background of the surface presets (models/base_surface_model.py:188-201).  Same constructor,
``get_density``, ``get_outputs``, ``density_fn`` and ``forward``, and the reference's parameter names (``mlp_base.layers.{i}``,
``mlp_head.layers.{i}``, ``field_output_density.net``, ``field_heads.0.net``), so a reference state dict loads with ``load_state_dict``.

Engines (``_engine``):
* eval forward (``torch.no_grad()`` or eval mode) at precision ``bf16x3`` / ``bf16`` for a shape in the fused kernel's family
  (``sdfb200_nerf_field_in_family``: 8 x 256 base with the skip at 4, 2 x 128 head, encodings of at most 10 frequencies): one launch of
  k_nerf_field_tc (csrc/nerf_field_tc.cu);
* training (autograd recording in train mode), ``get_density`` / ``get_outputs`` called on their own, or a shape outside the family: the
  differentiable composition on ``linear_ops.linear`` (ReLU in the GEMM epilogue, activations padded to 16 columns);
* precision ``fp32``: ATen matmuls, the reference's arithmetic.
There is no CPU path.

Not supported (``SurfaceModel`` uses none of them): ``compute_normals=True``, ``use_integrated_encoding=True``, field heads other than
the single ``RGBFieldHead``.
"""
import ctypes
import math
from typing import Optional, Tuple

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib
from . import linear_ops as _lo
from .autograd_ops import training_step
from .field_heads import FieldHeadNames
from .rays import point_or_ray_inputs
from .sdf_field_train import nerf_encoding, nerf_frequencies
from .spatial_distortions import contraction_code


class Identity(nn.Module):
    """encodings.py:48-62."""

    def __init__(self, in_dim: int) -> None:
        super().__init__()
        self.in_dim = in_dim

    def get_out_dim(self) -> int:
        return self.in_dim

    def forward(self, in_tensor):
        return in_tensor


class NeRFEncoding(nn.Module):
    """encodings.py:99-208 without the integrated (``covs``) form."""

    def __init__(self, in_dim: int, num_frequencies: int, min_freq_exp: float, max_freq_exp: float, include_input: bool = False,
                 off_axis: bool = False) -> None:
        super().__init__()
        self.in_dim = in_dim
        self.num_frequencies = num_frequencies
        self.min_freq = min_freq_exp
        self.max_freq = max_freq_exp
        self.include_input = include_input
        self.off_axis = off_axis

    def get_out_dim(self) -> int:
        return (21 if self.off_axis else self.in_dim) * self.num_frequencies * 2 + (self.in_dim if self.include_input else 0)

    def forward(self, in_tensor, covs=None):
        if covs is not None:
            raise NotImplementedError("integrated encodings are not supported")
        return nerf_encoding(in_tensor, self.num_frequencies, self.max_freq, self.include_input, self.off_axis, self.min_freq)


class _MLP(nn.Module):
    """field_components/mlp.py:27-99 with ReLU between the layers and as the output activation (how NeRFField builds both MLPs)."""

    def __init__(self, in_dim: int, num_layers: int, layer_width: int, skip_connections: Optional[Tuple[int]] = None) -> None:
        super().__init__()
        self.in_dim, self.num_layers, self.layer_width = in_dim, num_layers, layer_width
        self.out_dim = layer_width
        self.skip_connections = skip_connections
        self._skip_connections = set(skip_connections) if skip_connections else set()
        if 0 in self._skip_connections:
            raise ValueError("Skip connection at layer 0 doesn't make sense.")
        if num_layers == 1:
            layers = [nn.Linear(in_dim, layer_width)]
        else:
            layers = [nn.Linear(in_dim if i == 0 else layer_width + (in_dim if i in self._skip_connections else 0), layer_width)
                      for i in range(num_layers - 1)] + [nn.Linear(layer_width, layer_width)]
        self.layers = nn.ModuleList(layers)

    def get_out_dim(self) -> int:
        return self.out_dim


class RGBFieldHead(nn.Module):
    """field_heads.py:111-120: Linear(in_dim, 3) + sigmoid, its input width set by the field."""

    field_head_name = FieldHeadNames.RGB

    def __init__(self, in_dim: Optional[int] = None) -> None:
        super().__init__()
        self.in_dim = in_dim
        self.net = None
        if in_dim is not None:
            self.set_in_dim(in_dim)

    def set_in_dim(self, in_dim: int) -> None:
        self.in_dim = in_dim
        self.net = nn.Linear(in_dim, 3)


class _DensityFieldHead(nn.Module):
    """field_heads.py:99-108: Linear(in_dim, 1) + softplus."""

    def __init__(self, in_dim: int) -> None:
        super().__init__()
        self.net = nn.Linear(in_dim, 1)


_DEFAULT_HEADS = (RGBFieldHead(),)


def _encoding_shape(enc):
    """(in_dim, num_frequencies, min, max, include_input, off_axis) of a NeRFEncoding or Identity (the package's or the reference's)."""
    if not hasattr(enc, "num_frequencies"):
        if hasattr(enc, "in_dim") and type(enc).__name__ == "Identity":
            return enc.in_dim, 0, 0.0, 0.0, True, False
        raise NotImplementedError(f"encoding {type(enc).__name__} is not supported (NeRFEncoding or Identity)")
    return enc.in_dim, int(enc.num_frequencies), float(enc.min_freq), float(enc.max_freq), bool(enc.include_input), bool(getattr(enc, "off_axis", False))


class NeRFField(nn.Module):
    """vanilla_nerf_field.py:37-114."""

    def __init__(self, position_encoding: nn.Module = Identity(in_dim=3), direction_encoding: nn.Module = Identity(in_dim=3), base_mlp_num_layers: int = 8,
                 base_mlp_layer_width: int = 256, head_mlp_num_layers: int = 2, head_mlp_layer_width: int = 128, skip_connections: Tuple[int] = (4,),
                 field_heads: Tuple[nn.Module] = _DEFAULT_HEADS, use_integrated_encoding: bool = False, spatial_distortion=None, *,
                 precision: str = "bf16x3") -> None:
        super().__init__()
        if use_integrated_encoding:
            raise NotImplementedError("use_integrated_encoding=True is not supported (SurfaceModel does not use it)")
        if precision not in _lib.PRECISION:
            raise ValueError(f"precision must be one of {sorted(_lib.PRECISION)}")
        if field_heads is _DEFAULT_HEADS:         # the reference shares one default head between instances; each field gets its own
            field_heads = (RGBFieldHead(),)
        if len(field_heads) != 1 or type(field_heads[0]).__name__ != "RGBFieldHead":
            raise NotImplementedError("only the single RGBFieldHead is supported (SurfaceModel uses no other)")
        self.position_encoding = position_encoding
        self.direction_encoding = direction_encoding
        self.use_integrated_encoding = use_integrated_encoding
        self.spatial_distortion = spatial_distortion
        self.precision = precision
        self._pe = _encoding_shape(position_encoding)
        self._de = _encoding_shape(direction_encoding)
        self.mlp_base = _MLP(position_encoding.get_out_dim(), base_mlp_num_layers, base_mlp_layer_width, skip_connections)
        self.mlp_head = _MLP(self.mlp_base.get_out_dim() + direction_encoding.get_out_dim(), head_mlp_num_layers, head_mlp_layer_width)
        self.field_output_density = _DensityFieldHead(self.mlp_base.get_out_dim())
        self.field_heads = nn.ModuleList(field_heads)
        for field_head in self.field_heads:
            field_head.set_in_dim(self.mlp_head.get_out_dim())
        self._packed = None
        self._packed_key = None

    # ------------------------------------------------------------------ engine choice
    def _desc(self, n_samples: int = 0) -> "_lib.NerfFieldDesc":
        d = _lib.NerfFieldDesc()
        b, h = self.mlp_base, self.mlp_head
        d.base_layers, d.base_width = b.num_layers, b.layer_width
        skips = sorted(b._skip_connections)
        d.skip_layer = skips[0] if len(skips) == 1 else -1
        d.head_layers, d.head_width = h.num_layers, h.layer_width
        for enc, pre in ((self._pe, "pe"), (self._de, "dir")):
            in_dim, n, lo, hi, inc, off_axis = enc
            ok = in_dim == 3 and not off_axis and n <= _lib.NERF_MAX_FREQS
            setattr(d, pre + "_frequencies", n if ok else -1)
            setattr(d, pre + "_include_input", int(inc))
            if ok:
                getattr(d, pre + "_freqs")[:n] = nerf_frequencies(lo, hi, n).tolist()
        d.contraction = contraction_code(self.spatial_distortion)
        d.n_samples = n_samples
        d.precision = _lib.PRECISION[self.precision]
        return d

    def _engine(self) -> str:
        """'aten' (fp32), 'compose' (linear_ops GEMMs, differentiable) or 'kernel' (one fused launch) for a forward call."""
        if self.precision == "fp32":
            return "aten"
        if training_step(self, self.parameters()) or not _lib.load().sdfb200_nerf_field_in_family(self._desc()):
            return "compose"
        return "kernel"

    # ------------------------------------------------------------------ composition (training, and shapes outside the family)
    def _dense(self, lin, x, relu: bool):
        if self.precision == "fp32":
            y = F.linear(x, lin.weight, lin.bias)
            return torch.relu(y) if relu else y
        return _lo.linear(_lo.pad_cols(x), lin.weight, lin.bias, 2 if relu else 0, self.precision)[:, : lin.out_features]

    def _mlp(self, mlp, in_tensor):
        """field_components/mlp.py:80-99."""
        x = in_tensor
        for i, layer in enumerate(mlp.layers):
            if i in mlp._skip_connections:
                x = torch.cat([in_tensor, x], -1)
            x = self._dense(layer, x, True)
        return x

    def _density_from_positions(self, positions):
        _lib.require_cuda(positions.device, "NeRFField")
        if self.spatial_distortion is not None:
            positions = self.spatial_distortion(positions)
        shape = positions.shape[:-1]
        encoded_xyz = self.position_encoding(positions.reshape(-1, 3))
        base_mlp_out = self._mlp(self.mlp_base, encoded_xyz)
        density = F.softplus(self._dense(self.field_output_density.net, base_mlp_out, False))
        return density.view(*shape, 1), base_mlp_out.view(*shape, base_mlp_out.shape[-1])

    def get_density(self, ray_samples):
        """vanilla_nerf_field.py:91-104."""
        return self._density_from_positions(ray_samples.frustums.get_positions())

    def density_fn(self, positions: torch.Tensor) -> torch.Tensor:
        """fields/base_field.py:48-65: the density at `positions`."""
        return self._density_from_positions(positions)[0]

    def get_outputs(self, ray_samples, density_embedding: Optional[torch.Tensor] = None):
        """vanilla_nerf_field.py:106-114."""
        directions = ray_samples.frustums.directions
        _lib.require_cuda(directions.device, "NeRFField")
        shape = directions.shape[:-1]
        encoded_dir = self.direction_encoding(directions.reshape(-1, 3))
        mlp_out = self._mlp(self.mlp_head, torch.cat([encoded_dir, density_embedding.reshape(encoded_dir.shape[0], density_embedding.shape[-1])], dim=-1))
        rgb = torch.sigmoid(self._dense(self.field_heads[0].net, mlp_out, False))
        return {FieldHeadNames.RGB: rgb.view(*shape, 3)}

    # ------------------------------------------------------------------ forward
    def forward(self, ray_samples, compute_normals: bool = False):
        """fields/base_field.py:104-123."""
        if compute_normals:
            raise NotImplementedError("compute_normals=True is not supported by the NeRF background field")
        if self._engine() == "kernel":
            density, rgb = self._kernel_forward(ray_samples)
            return {FieldHeadNames.RGB: rgb, FieldHeadNames.DENSITY: density}
        density, density_embedding = self.get_density(ray_samples)
        outputs = self.get_outputs(ray_samples, density_embedding=density_embedding)
        outputs[FieldHeadNames.DENSITY] = density
        return outputs

    def _linears(self):
        return [*self.mlp_base.layers, *self.mlp_head.layers, self.field_output_density.net, self.field_heads[0].net]

    def _packed_weights(self, desc):
        """The weights in the fused kernel's layout (tc_pack); rebuilt only when a parameter changed."""
        lib = _lib.load()
        params = [p for lin in self._linears() for p in (lin.weight, lin.bias)]
        key = _lib.packed_key(params, desc.precision)
        if self._packed is not None and key == self._packed_key:
            return self._packed
        packed = torch.empty(lib.sdfb200_nerf_field_packed_bytes(desc), dtype=torch.uint8, device=params[0].device)
        ws = [_lib.f32c(lin.weight.detach()) for lin in self._linears()]
        bs = [_lib.f32c(lin.bias.detach()) for lin in self._linears()]
        w_ptrs = (ctypes.c_void_p * len(ws))(*[w.data_ptr() for w in ws])
        b_ptrs = (ctypes.c_void_p * len(bs))(*[b.data_ptr() for b in bs])
        _lib.check(lib.sdfb200_nerf_field_pack(desc, w_ptrs, b_ptrs, packed.data_ptr(), _lib.stream_ptr()), "sdfb200_nerf_field_pack")
        self._packed, self._packed_key = packed, key
        return packed

    def _kernel_forward(self, ray_samples):
        """One sdfb200_nerf_field_forward launch, in ray or point mode (rays.point_or_ray_inputs)."""
        lib = _lib.load()
        _lib.require_cuda(ray_samples.frustums.directions.device, "NeRFField")
        origins, directions, bins, n_rows, S, shape = point_or_ray_inputs(ray_samples)
        desc = self._desc(S)
        packed = self._packed_weights(desc)
        N = math.prod(shape)
        density = torch.empty(N, device=origins.device, dtype=torch.float32)
        rgb = torch.empty(N, 3, device=origins.device, dtype=torch.float32)
        _lib.check(lib.sdfb200_nerf_field_forward(desc, packed.data_ptr(), _lib.ptr(origins), _lib.ptr(directions), _lib.ptr(bins), n_rows,
                                                  density.data_ptr(), rgb.data_ptr(), _lib.stream_ptr()), "sdfb200_nerf_field_forward")
        return density.view(*shape, 1), rgb.view(*shape, 3)

