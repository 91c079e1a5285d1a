"""Drop-in for the ``tinycudann.Encoding`` operator used by SDFField (nerfstudio/fields/sdf_field.py:230-241, :386)
and for the reference's own ``HashEncoding`` (nerfstudio/field_components/encodings.py:269-403).

``Encoding(n_input_dims=3, encoding_config={...})`` keeps tcnn's constructor / ``n_output_dims`` / ``forward`` /
``.parameters()`` contract.  Two table layouts are supported behind ``layout=``:

* ``"tcnn"``  (default, what real sdfstudio checkpoints hold): coarse levels dense, per-level sizes rounded up to 8,
  single flat ``params`` tensor.
* ``"torch"`` : the reference ``HashEncoding(implementation="torch")`` layout, ``hash_table [L*T, F]``.

The arithmetic runs in libsdfb200.so (sdfb200_grid_encode / sdfb200_grid_encode_backward); there is no PyTorch path.
"""
import contextlib
import math
from typing import Optional

import numpy as np
import torch
from torch import nn
from torch.optim.optimizer import register_optimizer_step_post_hook

from . import _lib

# Bumped after every optimizer step.  A fused optimizer step (torch.optim.Adam(fused=True)) writes the parameters without bumping their
# version counter, so Encoding.compute_table keys its fp16 copy on this as well.
_optimizer_steps = [0]


def _count_optimizer_step(optimizer, args, kwargs):
    _optimizer_steps[0] += 1


register_optimizer_step_post_hook(_count_optimizer_step)


def growth_factor(num_levels: int, base_res: int, max_res: float) -> float:
    """sdf_field.py:226."""
    if num_levels <= 1:
        return 1.0
    return float(np.exp((np.log(max_res) - np.log(base_res)) / (num_levels - 1)))


def make_grid_desc(layout: str, n_levels: int, n_features: int, log2_hashmap_size: int, base_resolution: int, per_level_scale: float,
                   smoothstep: bool, table_dtype: torch.dtype = torch.float32) -> "_lib.GridDesc":
    """Fill the C descriptor (include/sdfb200.h: sdfb200_grid_t)."""
    if n_levels > _lib.MAX_LEVELS:
        raise ValueError(f"n_levels {n_levels} > {_lib.MAX_LEVELS}")
    if n_features not in (1, 2, 4, 8):
        raise ValueError("n_features_per_level must be 1, 2, 4 or 8")
    g = _lib.GridDesc()
    g.n_levels, g.n_features, g.log2_hashmap_size = n_levels, n_features, log2_hashmap_size
    g.smoothstep = int(bool(smoothstep))
    g.active_levels = n_levels
    g.table_dtype = _lib.DT_F16 if table_dtype == torch.float16 else _lib.DT_F32
    T = 1 << log2_hashmap_size
    total = 0
    if layout == "torch":
        g.layout = _lib.GRID_TORCH
        # encodings.py:301-303: floor(min_res * growth**level), growth recomputed from (min_res, max_res) in float64 and
        # evaluated by torch in float32.  max_res is what SDFField hands to the encoder: base * g**(L-1).
        max_res = base_resolution * per_level_scale ** (n_levels - 1)
        growth = np.exp((np.log(max_res) - np.log(base_resolution)) / (n_levels - 1)) if n_levels > 1 else 1.0
        scal = torch.floor(base_resolution * growth ** torch.arange(n_levels))
        for l in range(n_levels):
            g.scale[l] = float(scal[l])
            g.resolution[l] = int(scal[l]) + 1
            g.size[l] = T
            g.offset[l] = l * T
            g.hashed[l] = 1
        total = n_levels * T
    elif layout == "tcnn":
        g.layout = _lib.GRID_TCNN
        log2g = math.log2(per_level_scale)
        for l in range(n_levels):
            scale = float(np.float32(np.exp2(np.float32(l * log2g)) * np.float32(base_resolution) - np.float32(1.0)))
            res = int(math.ceil(scale)) + 1
            dense = res**3
            n = min(((dense + 7) // 8) * 8, T)
            g.scale[l] = scale
            g.resolution[l] = res
            g.size[l] = n
            g.offset[l] = total
            g.hashed[l] = 1 if dense > n else 0
            total += n
    else:
        raise ValueError(f"unknown grid layout {layout!r}")
    g._total_entries = total  # python-side attribute (not part of the C struct)
    return g


class _GridEncodeFn(torch.autograd.Function):
    """out = encode(x; table).  Differentiable twice: backward is itself an autograd Function (``_GridEncodeBwdFn``) so that
    ``autograd.grad(sdf, x, create_graph=True)`` (sdf_field.py:655-662) followed by the eikonal loss works like it does over tcnn."""

    @staticmethod
    def forward(ctx, x, table, enc):
        lib = _lib.load()
        x = _lib.f32c(x)
        n = x.shape[0]
        out = torch.empty(n, enc.n_output_dims, device=x.device, dtype=torch.float32)
        # Encoding.point_groups(G): the batch is G taps per sample (tap g of sample s at row g * n / G + s) that mostly share their table rows
        groups = enc._groups if enc._groups > 1 and n % enc._groups == 0 else 1
        if groups > 1:
            _lib.check(lib.sdfb200_grid_encode_grouped(enc._desc_ref(), _lib.ptr(enc.compute_table()), _lib.ptr(x), n, groups, _lib.ptr(out), enc.n_output_dims,
                                                       _lib.stream_ptr()), "sdfb200_grid_encode_grouped")
        else:
            _lib.check(lib.sdfb200_grid_encode(enc._desc_ref(), _lib.ptr(enc.compute_table()), _lib.ptr(x), n, _lib.ptr(out), enc.n_output_dims, None,
                                               _lib.stream_ptr()), "sdfb200_grid_encode")
        ctx.save_for_backward(x, table)
        ctx.enc = enc
        ctx.groups = groups
        return out

    @staticmethod
    def backward(ctx, dout):
        x, table = ctx.saved_tensors
        # inside Encoding.inputs_only_backward() (the autograd.grad(sdf, x) of SDFField) the table gradient is not requested:
        # skip its atomic scatter -- autograd cannot tell a Python Function which of its input gradients a call needs
        need_dtable = ctx.needs_input_grad[1] and not ctx.enc._inputs_only
        dx, dtable = _GridEncodeBwdFn.apply(dout, x, table, ctx.enc, ctx.needs_input_grad[0], need_dtable, ctx.groups)
        return dx, dtable, None


class _GridEncodeBwdFn(torch.autograd.Function):
    """(dx, dtable) = encode_backward(dout; x, table); its own backward is sdfb200_grid_encode_backward_backward."""

    @staticmethod
    def forward(ctx, dout, x, table, enc, need_dx, need_dtable, groups=1):
        lib = _lib.load()
        dout = _lib.f32c(dout)
        n = x.shape[0]
        dtable = torch.zeros(table.shape, device=table.device, dtype=torch.float32) if need_dtable else None
        dx = torch.zeros_like(x) if need_dx else None
        if dtable is None and dx is None:
            ctx.save_for_backward(dout, x, table)
            ctx.enc = enc
            return None, None
        if groups > 1 and dx is None:
            # table gradient of a grouped batch: taps that hit the same 8 rows of a level are summed in registers, one set of atomics per run
            _lib.check(lib.sdfb200_grid_encode_backward_grouped(enc._desc_ref(), _lib.ptr(x), _lib.ptr(dout), n, groups, _lib.ptr(dtable), _lib.stream_ptr()),
                       "sdfb200_grid_encode_backward_grouped")
        else:
            _lib.check(lib.sdfb200_grid_encode_backward(enc._desc_ref(), _lib.ptr(enc.compute_table()), _lib.ptr(x), _lib.ptr(dout), n, _lib.ptr(dtable),
                                                        _lib.ptr(dx), _lib.stream_ptr()), "sdfb200_grid_encode_backward")
        ctx.save_for_backward(dout, x, table)
        ctx.enc = enc
        dt = dtable.to(table.dtype) if dtable is not None else None
        if dt is not None:
            ctx.mark_non_differentiable(dt)
        return dx, dt

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_dx, g_dtable):
        if g_dx is None:
            return None, None, None, None, None, None, None
        lib = _lib.load()
        dout, x, table = ctx.saved_tensors
        enc = ctx.enc
        g_dx = _lib.f32c(g_dx)
        n = x.shape[0]
        g_dout = torch.empty_like(dout) if ctx.needs_input_grad[0] else None
        g_x = torch.zeros_like(x) if ctx.needs_input_grad[1] else None
        g_table = torch.zeros(table.shape, device=table.device, dtype=torch.float32) if ctx.needs_input_grad[2] else None
        _lib.check(lib.sdfb200_grid_encode_backward_backward(enc._desc_ref(), _lib.ptr(enc.compute_table()), _lib.ptr(x), _lib.ptr(dout), _lib.ptr(g_dx), n,
                                                             _lib.ptr(g_dout), _lib.ptr(g_table), _lib.ptr(g_x), _lib.stream_ptr()),
                   "sdfb200_grid_encode_backward_backward")
        return g_dout, g_x, (g_table.to(table.dtype) if g_table is not None else None), None, None, None, None


class _GridFn(torch.autograd.Function):
    """hash-grid features of the flat parameter vector of a tiny-cuda-nn NetworkWithInputEncoding (grid table = its tail, `nb` the
    module that owns it: density_fields._NetworkWithInputEncoding): forward / backward kernels of the Encoding operator, gradient
    scattered into the tail of d(params).  The training path of the proposal and nerfacto fields."""

    @staticmethod
    def forward(ctx, x01, params, nb):
        lib = _lib.load()
        x = _lib.f32c(x01)
        n = x.shape[0]
        out = torch.empty(n, nb.in_dim, device=x.device, dtype=torch.float32)
        table = params.detach()[nb.n_net:]
        _lib.check(lib.sdfb200_grid_encode(nb.kernel_desc(), table.data_ptr(), _lib.ptr(x), n, _lib.ptr(out), nb.in_dim, None, _lib.stream_ptr()), "sdfb200_grid_encode")
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


class Encoding(nn.Module):
    """``tinycudann.Encoding`` look-alike (HashGrid / DenseGrid otypes)."""

    def __init__(self, n_input_dims: int, encoding_config: dict, seed: int = 1337, dtype: Optional[torch.dtype] = None,
                 layout: str = "tcnn", device: Optional[torch.device] = None, table_dtype: str = "fp32"):
        super().__init__()
        if table_dtype not in ("fp32", "fp16"):
            raise ValueError("table_dtype must be 'fp32' or 'fp16'")
        # "fp16": the kernels gather from a half-precision copy of the (fp32 master) parameters, which is what tiny-cuda-nn
        # itself does (fp16 compute params + fp32 master); the copy is refreshed whenever the parameter changes
        self.table_dtype = table_dtype
        self._inputs_only = False
        self._groups = 1
        self._half_cache = None
        self._half_key = None
        if n_input_dims != 3:
            raise ValueError("only 3-D grids are supported")
        otype = encoding_config.get("otype", "HashGrid")
        if otype not in ("HashGrid", "DenseGrid", "Grid"):
            raise ValueError(f"unsupported encoding otype {otype!r}")
        self.encoding_config = dict(encoding_config)
        self.layout = layout
        self.n_input_dims = 3
        self.n_levels = int(encoding_config.get("n_levels", 16))
        self.n_features_per_level = int(encoding_config.get("n_features_per_level", 2))
        self.log2_hashmap_size = int(encoding_config.get("log2_hashmap_size", 19))
        self.base_resolution = int(encoding_config.get("base_resolution", 16))
        self.per_level_scale = float(encoding_config.get("per_level_scale", 2.0))
        self.interpolation = encoding_config.get("interpolation", "Linear")
        if self.interpolation not in ("Linear", "Smoothstep"):
            raise ValueError(f"unsupported interpolation {self.interpolation!r}")
        self.n_output_dims = self.n_levels * self.n_features_per_level
        self.active_levels = self.n_levels
        self._desc = make_grid_desc(layout, self.n_levels, self.n_features_per_level, self.log2_hashmap_size, self.base_resolution,
                                    self.per_level_scale, self.interpolation == "Smoothstep")
        total = self._desc._total_entries
        g = torch.Generator().manual_seed(seed)
        if layout == "torch":
            # encodings.py:306-308: U(-1,1) * 1e-3
            table = (torch.rand(total, self.n_features_per_level, generator=g) * 2 - 1) * 1e-3
            self.hash_table = nn.Parameter(table.to(device) if device is not None else table)
        else:
            # tcnn initialises grids with U(-1e-4, 1e-4); parameters are exposed as one flat fp32 tensor
            table = (torch.rand(total * self.n_features_per_level, generator=g) * 2 - 1) * 1e-4
            self.params = nn.Parameter(table.to(device) if device is not None else table)

    @property
    def table(self) -> torch.Tensor:
        return self.hash_table if self.layout == "torch" else self.params

    def compute_table(self) -> torch.Tensor:
        """the tensor the kernels gather from (the parameter itself, or its cached fp16 copy).

        The fp16 copy is rebuilt when the parameter is reallocated, written in place (its version counter: optimizer steps with
        ``foreach``, ``load_state_dict``, ``copy_`` under ``no_grad``) or after any optimizer step (fused steps do not bump the version
        counter).  A write through ``.data`` is NOT seen: ``.data`` has a version counter of its own, so the kernels keep gathering the
        old values until one of the events above.  Write under ``torch.no_grad()`` instead."""
        t = self.table
        if self.table_dtype == "fp32" or t.dtype == torch.float16:
            return t.detach()
        key = (t.data_ptr(), t._version, str(t.device), _optimizer_steps[0])
        if self._half_key != key:
            self._half_cache = t.detach().to(torch.float16)
            self._half_key = key
        return self._half_cache

    def _desc_ref(self):
        self._desc.active_levels = int(self.active_levels)
        half = self.table_dtype == "fp16" or self.table.dtype == torch.float16
        self._desc.table_dtype = _lib.DT_F16 if half else _lib.DT_F32
        return self._desc

    @contextlib.contextmanager
    def inputs_only_backward(self):
        """Backward passes started inside this context compute d/dx only (no table-gradient scatter).  For
        ``torch.autograd.grad(sdf, x, create_graph=True)``-style calls whose `inputs` do not include the table."""
        prev, self._inputs_only = self._inputs_only, True
        try:
            yield
        finally:
            self._inputs_only = prev

    @contextlib.contextmanager
    def point_groups(self, groups: int):
        """Calls inside this context pass batches of `groups` taps per sample (tap g of sample s at row g * n / groups + s), e.g. a sample and its
        six +-delta taps of the numerical gradient (sdf_field.py:424-452).  Taps that hit the same table rows share their gathers / atomics."""
        prev, self._groups = self._groups, max(1, int(groups))
        try:
            yield
        finally:
            self._groups = prev

    def set_active_levels(self, levels: int):
        """levels >= `levels` output zeros (fused form of SDFField.update_mask, sdf_field.py:376-378)."""
        self.active_levels = max(0, min(int(levels), self.n_levels))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        shape = x.shape[:-1]
        out = _GridEncodeFn.apply(x.reshape(-1, 3), self.table, self)
        return out.view(*shape, self.n_output_dims)

    def extra_repr(self):
        return f"layout={self.layout}, L={self.n_levels}, F={self.n_features_per_level}, T=2^{self.log2_hashmap_size}, {self.interpolation}"


class HashEncoding(Encoding):
    """nerfstudio ``HashEncoding`` look-alike (field_components/encodings.py:283-335): torch-layout table."""

    def __init__(self, num_levels: int = 16, min_res: int = 16, max_res: int = 1024, log2_hashmap_size: int = 19, features_per_level: int = 2,
                 hash_init_scale: float = 0.001, implementation: str = "torch", interpolation: Optional[str] = None, seed: int = 1337):
        cfg = {
            "otype": "HashGrid", "n_levels": num_levels, "n_features_per_level": features_per_level, "log2_hashmap_size": log2_hashmap_size,
            "base_resolution": min_res, "per_level_scale": growth_factor(num_levels, min_res, max_res), "interpolation": interpolation or "Linear",
        }  # fmt: skip
        super().__init__(3, cfg, seed=seed, layout="torch" if implementation == "torch" else "tcnn")
        if self.layout == "torch" and hash_init_scale != 0.001:
            with torch.no_grad():
                self.hash_table.mul_(hash_init_scale / 0.001)

    def get_out_dim(self) -> int:
        return self.n_output_dims
