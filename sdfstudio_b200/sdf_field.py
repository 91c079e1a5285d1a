"""H100-native drop-in for ``nerfstudio.fields.sdf_field`` (SDFField, SDFFieldConfig, LaplaceDensity,
SingleVarianceNetwork).  Same constructor, same methods, same parameter names/shapes (``glin{l}.weight_g/weight_v/bias``,
``clin{l}.*``, ``laplace_density.beta``, ``deviation_network.variance``, ``embedding_appearance.embedding.weight``) so a
reference state_dict loads directly; the arithmetic runs in libsdfb200.so through sdfb200_field_forward.

Swap-in under ns-train: ``SDFFieldConfig._target`` of this module (see INTEGRATION.md).
"""
import itertools
import math
import warnings
from dataclasses import dataclass, field
from typing import Dict, Optional, Type

import numpy as np
import torch
from torch import nn

from . import _lib
from . import sdf_field_train as _train
from .autograd_ops import training_step
from .encoding import Encoding, growth_factor
from .field_heads import FieldHeadNames
from .rays import bins_of, rays_of, sample_geometry
from .renderers import _background
from .spatial_distortions import contraction_code


class LaplaceDensity(nn.Module):
    """sdf_field.py:49-71.  Callable on arbitrary tensors (used as ``density_fn`` by ErrorBoundedSampler)."""

    def __init__(self, init_val, beta_min=0.0001):
        super().__init__()
        self.register_parameter("beta_min", nn.Parameter(beta_min * torch.ones(1), requires_grad=False))
        self.register_parameter("beta", nn.Parameter(init_val * torch.ones(1), requires_grad=True))

    def forward(self, sdf, beta=None):
        if beta is None:
            beta = self.get_beta()
        alpha = 1.0 / beta
        return alpha * (0.5 + 0.5 * sdf.sign() * torch.expm1(-sdf.abs() / beta))

    def get_beta(self):
        return self.beta.abs() + self.beta_min


class SingleVarianceNetwork(nn.Module):
    """sdf_field.py:101-118."""

    def __init__(self, init_val):
        super().__init__()
        self.register_parameter("variance", nn.Parameter(init_val * torch.ones(1), requires_grad=True))

    def forward(self, x):
        return torch.ones([len(x), 1], device=x.device) * torch.exp(self.variance * 10.0)

    def get_variance(self):
        return torch.exp(self.variance * 10.0).clip(1e-6, 1e6)


class _Embedding(nn.Module):
    """field_components/embedding.py:26-54."""

    def __init__(self, in_dim, out_dim):
        super().__init__()
        self.in_dim, self.out_dim = in_dim, out_dim
        self.embedding = nn.Embedding(in_dim, out_dim)

    def get_out_dim(self):
        return self.out_dim

    def mean(self, dim=0):
        return self.embedding.weight.mean(dim)

    def forward(self, x):
        return self.embedding(x)


class _EncodingInfo:
    """Shape-only stand-in for NeRFEncoding (the sin/cos features are produced inside the fused kernel)."""

    def __init__(self, in_dim, num_frequencies, include_input, off_axis=False):
        self.in_dim, self.num_frequencies, self.include_input, self.off_axis = in_dim, num_frequencies, include_input, off_axis

    def get_out_dim(self):
        d = (21 if self.off_axis else self.in_dim) * self.num_frequencies * 2
        return d + (self.in_dim if self.include_input else 0)


@dataclass
class SDFFieldConfig:
    """Field-for-field copy of the reference config (sdf_field.py:121-185) + two knobs of this package at the end."""

    _target: Type = field(default_factory=lambda: SDFField)
    num_layers: int = 8
    hidden_dim: int = 256
    geo_feat_dim: int = 256
    num_layers_color: int = 4
    hidden_dim_color: int = 256
    appearance_embedding_dim: int = 32
    use_appearance_embedding: bool = False
    bias: float = 0.8
    geometric_init: bool = True
    inside_outside: bool = True
    weight_norm: bool = True
    use_grid_feature: bool = False
    divide_factor: float = 2.0
    beta_init: float = 0.1
    encoding_type: str = "hash"
    position_encoding_max_degree: int = 6
    use_diffuse_color: bool = False
    use_specular_tint: bool = False
    use_reflections: bool = False
    use_n_dot_v: bool = False
    rgb_padding: float = 0.001
    off_axis: bool = False
    use_numerical_gradients: bool = False
    num_levels: int = 16
    max_res: int = 2048
    base_res: int = 16
    log2_hashmap_size: int = 19
    hash_features_per_level: int = 2
    hash_smoothstep: bool = True
    use_position_encoding: bool = True
    # ---- knobs of this package (not in the reference) ----
    grid_layout: str = "tcnn"      # "tcnn" (checkpoint compatible) | "torch" (reference HashEncoding layout)
    precision: str = "fp32"        # "fp32" | "bf16x3" | "bf16"   (include/sdfb200.h SDFB200_PRECISION_*)
    table_dtype: str = "fp32"      # "fp32" | "fp16": gather from an fp16 copy of the table (tiny-cuda-nn's own storage precision)
    train_gemm: str = "auto"       # training-mode dense layers: "auto" = tensor-core GEMMs (linear_ops.py) unless precision == "fp32"; "aten" | "tc"

    def setup(self, **kwargs):
        return self._target(self, **kwargs)


class SDFField(nn.Module):
    """Drop-in for ``nerfstudio.fields.sdf_field.SDFField`` (sdf_field.py:188-698)."""

    def __init__(self, config: SDFFieldConfig, aabb, num_images: int, use_average_appearance_embedding: bool = False, spatial_distortion=None):
        super().__init__()
        self.config = config
        self.aabb = nn.Parameter(torch.as_tensor(aabb, dtype=torch.float32), requires_grad=False)
        self.spatial_distortion = spatial_distortion
        self.num_images = num_images
        self.embedding_appearance = _Embedding(num_images, config.appearance_embedding_dim)
        self.use_average_appearance_embedding = use_average_appearance_embedding
        self.use_grid_feature = config.use_grid_feature
        self.divide_factor = config.divide_factor
        self.num_levels, self.max_res, self.base_res = config.num_levels, config.max_res, config.base_res
        self.log2_hashmap_size, self.features_per_level = config.log2_hashmap_size, config.hash_features_per_level
        self.growth_factor = growth_factor(self.num_levels, self.base_res, self.max_res)
        if config.encoding_type != "hash":
            raise NotImplementedError("only encoding_type='hash' is supported (the periodic / tensorf_vm branches of the reference "
                                      "crash when use_grid_feature=True, sdf_field.py:242-245,388)")
        self.encoding = Encoding(
            n_input_dims=3,
            encoding_config={
                "otype": "HashGrid", "n_levels": self.num_levels, "n_features_per_level": self.features_per_level,
                "log2_hashmap_size": self.log2_hashmap_size, "base_resolution": self.base_res, "per_level_scale": self.growth_factor,
                "interpolation": "Smoothstep" if config.hash_smoothstep else "Linear",
            },  # fmt: skip
            layout=getattr(config, "grid_layout", "tcnn"),
            table_dtype=getattr(config, "table_dtype", "fp32"),
        )
        self.hash_encoding_mask = torch.ones(self.num_levels * self.features_per_level, dtype=torch.float32)
        self._active_levels = self.num_levels
        self.position_encoding = _EncodingInfo(3, config.position_encoding_max_degree, False, config.off_axis)
        self.direction_encoding = _EncodingInfo(3, 4, True)

        # ---- geometric network, geometric init (sdf_field.py:277-315) ----
        dims = [config.hidden_dim for _ in range(config.num_layers)]
        in_dim = 3 + self.position_encoding.get_out_dim() + self.encoding.n_output_dims
        dims = [in_dim] + dims + [1 + config.geo_feat_dim]
        self.num_layers = len(dims)
        self.skip_in = [4]
        self._geo_dims = dims
        for l in range(0, self.num_layers - 1):
            out_dim = dims[l + 1] - dims[0] if l + 1 in self.skip_in else dims[l + 1]
            lin = nn.Linear(dims[l], out_dim)
            if config.geometric_init:
                if l == self.num_layers - 2:
                    mean = np.sqrt(np.pi) / np.sqrt(dims[l])
                    if not config.inside_outside:
                        torch.nn.init.normal_(lin.weight, mean=mean, std=0.0001)
                        torch.nn.init.constant_(lin.bias, -config.bias)
                    else:
                        torch.nn.init.normal_(lin.weight, mean=-mean, std=0.0001)
                        torch.nn.init.constant_(lin.bias, config.bias)
                elif l == 0:
                    torch.nn.init.constant_(lin.bias, 0.0)
                    torch.nn.init.constant_(lin.weight[:, 3:], 0.0)
                    torch.nn.init.normal_(lin.weight[:, :3], 0.0, np.sqrt(2) / np.sqrt(out_dim))
                elif l in self.skip_in:
                    torch.nn.init.constant_(lin.bias, 0.0)
                    torch.nn.init.normal_(lin.weight, 0.0, np.sqrt(2) / np.sqrt(out_dim))
                    torch.nn.init.constant_(lin.weight[:, -(dims[0] - 3):], 0.0)
                else:
                    torch.nn.init.constant_(lin.bias, 0.0)
                    torch.nn.init.normal_(lin.weight, 0.0, np.sqrt(2) / np.sqrt(out_dim))
            if config.weight_norm:
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    lin = nn.utils.weight_norm(lin)
            setattr(self, "glin" + str(l), lin)

        self.laplace_density = LaplaceDensity(init_val=config.beta_init)
        self.deviation_network = SingleVarianceNetwork(init_val=config.beta_init)
        if config.use_diffuse_color:
            self.diffuse_color_pred = nn.Linear(config.geo_feat_dim, 3)
        if config.use_specular_tint:
            self.specular_tint_pred = nn.Linear(config.geo_feat_dim, 3)

        # ---- colour network (sdf_field.py:331-363) ----
        dims = [config.hidden_dim_color for _ in range(config.num_layers_color)]
        if config.use_diffuse_color:
            in_dim = self.direction_encoding.get_out_dim() + config.geo_feat_dim + self.embedding_appearance.get_out_dim()
        else:
            in_dim = 3 + self.direction_encoding.get_out_dim() + 3 + config.geo_feat_dim + self.embedding_appearance.get_out_dim()
        if config.use_n_dot_v:
            in_dim += 1
        dims = [in_dim] + dims + [3]
        self.num_layers_color = len(dims)
        self._color_dims = dims
        for l in range(0, self.num_layers_color - 1):
            lin = nn.Linear(dims[l], dims[l + 1])
            torch.nn.init.kaiming_uniform_(lin.weight.data)
            torch.nn.init.zeros_(lin.bias.data)
            if config.weight_norm:
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    lin = nn.utils.weight_norm(lin)
            setattr(self, "clin" + str(l), lin)

        self._cos_anneal_ratio = 1.0
        self.numerical_gradients_delta = 0.0001
        self._packed = None
        self._packed_key = None
        self._workspace = None

    # ------------------------------------------------------------------ small reference API
    def set_cos_anneal_ratio(self, anneal: float) -> None:
        self._cos_anneal_ratio = anneal

    def update_mask(self, level: int):
        """sdf_field.py:376-378.  The mask is applied inside the kernel by skipping the masked levels' gathers."""
        self.hash_encoding_mask[:] = 1.0
        self.hash_encoding_mask[level * self.features_per_level:] = 0
        self._active_levels = max(0, min(int(level), self.num_levels))

    def set_numerical_gradients_delta(self, delta: float) -> None:
        self.numerical_gradients_delta = delta

    def get_occupancy(self, sdf):
        return torch.sigmoid(-10.0 * sdf)

    # ------------------------------------------------------------------ descriptor / packed weights
    def _field_desc(self) -> "_lib.FieldDesc":
        c = self.config
        d = _lib.FieldDesc()
        g = self.encoding._desc_ref()
        g.active_levels = self._active_levels
        d.grid = g
        d.use_grid_feature = int(c.use_grid_feature)
        d.pe_degree = c.position_encoding_max_degree
        d.use_position_encoding = int(c.use_position_encoding)
        d.off_axis = int(c.off_axis)
        d.contraction = contraction_code(self.spatial_distortion)
        n_geo = self.num_layers - 1
        if n_geo > _lib.MAX_LAYERS or self.num_layers_color - 1 > _lib.MAX_LAYERS:
            raise NotImplementedError("too many layers")
        d.n_geo_linear = n_geo
        for i, v in enumerate(self._geo_dims):
            d.geo_dims[i] = v
        skip = 4 if n_geo > 4 else -1
        d.geo_skip_layer = skip
        d.n_color_linear = self.num_layers_color - 1
        for i, v in enumerate(self._color_dims):
            d.color_dims[i] = v
        # the packing reads every layer at the [N, K] the descriptor implies (make_field_plan, csrc/field_plan.h): the layer feeding the
        # skip concat is narrower.  With num_layers = 3 the reference's skip_in = [4] narrows the LAST layer instead, which the descriptor
        # cannot express, and a layer replaced by one of another shape would be read out of bounds just the same
        gd, cd = self._geo_dims, self._color_dims
        for l in range(n_geo):
            self._check_layer_shape(f"glin{l}", gd[l + 1] - gd[0] if l + 1 == skip else gd[l + 1], gd[l])
        for l in range(self.num_layers_color - 1):
            self._check_layer_shape(f"clin{l}", cd[l + 1], cd[l])
        d.appearance_dim = c.appearance_embedding_dim
        d.use_diffuse_color, d.use_specular_tint = int(c.use_diffuse_color), int(c.use_specular_tint)
        d.use_reflections, d.use_n_dot_v = int(c.use_reflections), int(c.use_n_dot_v)
        d.use_numerical_gradients = int(c.use_numerical_gradients)
        d.rgb_padding = c.rgb_padding
        d.precision = _lib.PRECISION[getattr(c, "precision", "fp32")]
        return d

    def _check_layer_shape(self, name: str, n: int, k: int) -> None:
        """ValueError unless Linear `name` holds an [n, k] weight (weight-normed: weight_v [n, k], weight_g [n, 1]) and an [n] bias.  Reads
        the registered parameters directly: this runs on every call."""
        p = self._modules[name]._parameters
        v = p.get("weight_v")
        if (p["weight"] if v is None else v).shape == (n, k) and p["bias"].shape == (n,) and (v is None or p["weight_g"].shape == (n, 1)):
            return
        have = (("weight", (n, k)),) if v is None else (("weight_v", (n, k)), ("weight_g", (n, 1)))
        what, want = next((w, s) for w, s in have + (("bias", (n,)),) if p[w].shape != s)
        raise ValueError(f"SDFField: {name}.{what} is {list(p[what].shape)}, but the field's layer dims make it {list(want)}"
                         + (" (num_layers = 3 puts the reference's skip connection after the last geometric layer, which neither the "
                            "reference nor this field can evaluate)" if self.num_layers == 5 and name == "glin3" else ""))

    def _mlp_params(self):
        """The MLPs' parameters, lazily (so that the engine choice touches none of them outside a training step)."""
        for l in range(self.num_layers - 1):
            yield from getattr(self, f"glin{l}").parameters()
        for l in range(self.num_layers_color - 1):
            yield from getattr(self, f"clin{l}").parameters()
        for n in ("diffuse_color_pred", "specular_tint_pred"):
            if hasattr(self, n):
                yield from getattr(self, n).parameters()

    def _packed_weights(self, desc):
        """Fold weight-norm and lay the weights out for the kernels; redone only when a parameter changed."""
        lib = _lib.load()
        params = list(self._mlp_params())
        key = _lib.packed_key(params, desc.precision)
        if self._packed is not None and key == self._packed_key:
            return self._packed
        nbytes = lib.sdfb200_field_packed_bytes(desc)
        if nbytes == 0:
            _lib.check(-1, "sdfb200_field_packed_bytes")
        if self._packed is None or self._packed.numel() != nbytes or self._packed.device != params[0].device:
            self._packed = torch.empty(nbytes, dtype=torch.uint8, device=params[0].device)
        fp = _lib.FieldParams()
        keep = []

        def dev(t):
            t = _lib.f32c(t.detach())
            keep.append(t)
            return t.data_ptr()

        def fill(prefix, n, wv, wg, b):
            for l in range(n):
                lin = getattr(self, f"{prefix}{l}")
                if hasattr(lin, "weight_v"):
                    wv[l], wg[l] = dev(lin.weight_v), dev(lin.weight_g)
                else:
                    wv[l], wg[l] = dev(lin.weight), None
                b[l] = dev(lin.bias)

        fill("glin", self.num_layers - 1, fp.geo_weight_v, fp.geo_weight_g, fp.geo_bias)
        fill("clin", self.num_layers_color - 1, fp.color_weight_v, fp.color_weight_g, fp.color_bias)
        if hasattr(self, "diffuse_color_pred"):
            fp.diffuse_weight, fp.diffuse_bias = dev(self.diffuse_color_pred.weight), dev(self.diffuse_color_pred.bias)
        if hasattr(self, "specular_tint_pred"):
            fp.tint_weight, fp.tint_bias = dev(self.specular_tint_pred.weight), dev(self.specular_tint_pred.bias)
        _lib.check(lib.sdfb200_field_pack(desc, fp, _lib.ptr(self._packed), _lib.stream_ptr()), "sdfb200_field_pack")
        self._packed_key = key
        return self._packed

    def _workspace_of(self, nbytes: int, query: str, dev):
        """The shared workspace on `dev`, grown to at least `nbytes` (the result of the size query `query`; 0 = refused)."""
        if nbytes == 0:
            _lib.check(-1, query)
        if self._workspace is None or self._workspace.numel() < nbytes or self._workspace.device != dev:
            self._workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        return self._workspace

    def _field_in(self, origins, directions, bins, n_samples: int, apply_contraction: bool, appearance):
        """sdfb200_field_in_t of one call: pointers only, so the caller keeps the tensors alive until the call is made."""
        fin = _lib.FieldIn()
        fin.n_rays, fin.n_samples, fin.apply_contraction = origins.shape[0], n_samples, int(apply_contraction)
        fin.origins, fin.directions, fin.bins = _lib.ptr(origins), _lib.ptr(directions), _lib.ptr(bins)
        fin.appearance = _lib.ptr(appearance)
        fin.variance = _lib.ptr(self.deviation_network.variance.detach())
        fin.beta = _lib.ptr(self.laplace_density.beta.detach())
        fin.beta_min = _lib.ptr(self.laplace_density.beta_min.detach())
        fin.cos_anneal_ratio = float(self._cos_anneal_ratio)
        fin.numerical_delta = float(self.numerical_gradients_delta)
        return fin

    # ------------------------------------------------------------------ the kernel call
    def _run(self, origins, directions, bins, n_samples: int, wants, apply_contraction: bool, appearance=None,
             analytic_gradients: bool = False) -> Dict[str, torch.Tensor]:
        """origins [R,3] (or points [N,3] in point mode), directions [R,3] | None, bins [R,S+1] | None.
        `wants`: iterable of output names of sdfb200_field_out_t.  `analytic_gradients`: differentiate the network even when the field
        uses numerical gradients.  Returns flat tensors ([N] / [N,k])."""
        lib = _lib.load()
        dev = self.aabb.device
        _lib.require_cuda(dev, "SDFField")
        R = origins.shape[0]
        N = R * n_samples
        desc = self._field_desc()
        packed = self._packed_weights(desc)
        if analytic_gradients and desc.use_numerical_gradients:
            # a numerical-gradient field runs the exact-fp32 engine at every precision, and its packed weights are the fp32 section alone:
            # the fp32 descriptor without numerical gradients evaluates the same network on the same blob
            desc.use_numerical_gradients = 0
            desc.precision = _lib.PRECISION["fp32"]
        ws = self._workspace_of(lib.sdfb200_field_workspace_bytes(desc, N), "sdfb200_field_workspace_bytes", dev)
        gf = self.config.geo_feat_dim
        shapes = {"sdf": (N,), "geo_feature": (N, gf), "gradients": (N, 3), "normals": (N, 3), "rgb": (N, 3), "density": (N,), "alpha": (N,),
                  "occupancy": (N,), "points_norm": (N,), "sampled_sdf": (N, 6), "points": (N, 3)}
        outs = {k: torch.empty(shapes[k], device=dev, dtype=torch.float32) for k in wants}
        fin = self._field_in(origins, directions, bins, n_samples, apply_contraction, appearance)
        fout = _lib.FieldOut()
        for k, t in outs.items():
            setattr(fout, k, t.data_ptr())
        table = self.encoding.compute_table() if self.use_grid_feature else None
        _lib.check(lib.sdfb200_field_forward(desc, _lib.ptr(packed), _lib.ptr(table), fin, fout, _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
                   "sdfb200_field_forward")
        return outs

    _SAMPLE_SHAPES = {"sdf": 1, "gradients": 3, "normals": 3, "rgb": 3, "density": 1, "alpha": 1, "occupancy": 1, "points_norm": 1, "points": 3}

    @torch.no_grad()
    def render(self, ray_samples, background, from_density: bool = False, training: bool = False, want_weights: bool = True,
               sample_outputs=(), clip_depth: bool = True) -> Dict[str, torch.Tensor]:
        """``get_outputs`` + weights + RGB / expected-depth / normal / accumulation renderers in ONE library call
        (sdfb200_field_render): what ``SurfaceModel.get_outputs`` computes between the sampler and the losses
        (models/base_surface_model.py:292-365; NeuS alphas, models/neus.py:85-116, or ``from_density`` = VolSDF's Laplace
        density weights, models/volsdf.py:62-87).  On the fused tensor-core path the per-sample heads never touch HBM unless they
        are asked for through ``sample_outputs`` (names of sdfb200_field_out_t).  Inference only (no autograd).
        Returns rgb [R,3], depth [R,1], normal [R,3], accumulation [R,1], bg_transmittance [R,1] (+ weights [R,S,1], + per-sample heads)."""
        if ray_samples.camera_indices is None:
            raise AttributeError("Camera indices are not provided.")
        lib = _lib.load()
        origins, directions = rays_of(ray_samples)
        bins = bins_of(ray_samples)
        R, S = origins.shape[0], bins.shape[1] - 1
        N = R * S
        dev = origins.device
        _lib.require_cuda(dev, "SDFField")
        desc = self._field_desc()
        packed = self._packed_weights(desc)
        ws = self._workspace_of(lib.sdfb200_field_render_workspace_bytes(desc, R, S), "sdfb200_field_render_workspace_bytes", dev)
        # one flat output allocation: per-ray block [R, 9] = rgb(3) depth normal(3) accumulation bg_transmittance | minmax(2) | per-sample blocks
        widths = [self._SAMPLE_SHAPES[k] for k in sample_outputs]
        flat = torch.empty(R * 9 + 2 + N * (sum(widths) + (1 if want_weights else 0)), device=dev, dtype=torch.float32)
        mm = flat[R * 9: R * 9 + 2]
        mm.copy_(_lib.steps_minmax_seed(dev))
        off = R * 9 + 2
        fout = _lib.FieldOut()
        res = {}
        for k, w_ in zip(sample_outputs, widths):
            t = flat[off: off + N * w_]
            off += N * w_
            setattr(fout, k, t.data_ptr())
            res[k] = t.view(R, S, w_)
        rnd = _lib.FieldRender()
        rnd.from_density, rnd.clamp01, rnd.clip_depth = int(from_density), int(not training), int(clip_depth)
        rnd.bg_mode, bg_t = _background(background, R, dev)
        rnd.bg = _lib.ptr(bg_t)
        if want_weights:
            wt = flat[off: off + N]
            rnd.weights = wt.data_ptr()
            res["weights"] = wt.view(R, S, 1)
        # per-ray outputs are stored planar ([3,R] etc. would not match the ABI) -> carve row-major [R,3] blocks instead
        rgb = flat[: R * 3].view(R, 3)
        nrm = flat[R * 3: R * 6].view(R, 3)
        depth, acc, bgT = flat[R * 6: R * 7], flat[R * 7: R * 8], flat[R * 8: R * 9]
        rnd.bg_transmittance = bgT.data_ptr()
        rnd.out = _lib.render_out(rgb, depth, nrm, acc, mm)
        app = self._appearance(ray_samples.camera_indices, R, dev)
        fin = self._field_in(origins, directions, bins, S, True, app)
        table = self.encoding.compute_table() if self.use_grid_feature else None
        _lib.check(lib.sdfb200_field_render(desc, _lib.ptr(packed), _lib.ptr(table), fin, fout, rnd, _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
                   "sdfb200_field_render")
        res.update({"rgb": rgb, "depth": depth[:, None], "normal": nrm, "accumulation": acc[:, None], "bg_transmittance": bgT[:, None]})
        return res

    def _differentiable(self) -> bool:
        """True when autograd is recording a training step: the methods below then return graph-carrying tensors from the
        autograd composition in sdf_field_train.py (grid operator = this package's kernels incl. double backward).  Everything
        under torch.no_grad() -- samplers, evaluation, meshing -- and eval mode runs the fused kernels."""
        return training_step(self, itertools.chain((self.encoding.table,), self._mlp_params()))

    # ------------------------------------------------------------------ reference methods
    def forward_geonetwork(self, inputs):
        """sdf_field.py:380-410: [N,3] -> [N, 1+geo_feat_dim]."""
        if self._differentiable():
            return _train.forward_geonetwork(self, inputs)
        pts = _lib.f32c(inputs.reshape(-1, 3))
        o = self._run(pts, None, None, 1, ("sdf", "geo_feature"), apply_contraction=False)
        return torch.cat([o["sdf"][:, None], o["geo_feature"]], dim=-1)

    def get_sdf(self, ray_samples):
        """sdf_field.py:412-418 (NOTE: un-contracted start positions, like the reference)."""
        if self._differentiable():
            pos = ray_samples.frustums.get_start_positions()
            h = _train.forward_geonetwork(self, pos.reshape(-1, 3)).view(*ray_samples.frustums.shape, -1)
            return h[..., :1]
        origins, directions, bins, shape = sample_geometry(ray_samples)
        o = self._run(origins, directions, bins, bins.shape[1] - 1, ("sdf",), apply_contraction=False)
        return o["sdf"].view(*shape, 1)

    def gradient(self, x, skip_spatial_distortion=False, return_sdf=False):
        """sdf_field.py:424-465."""
        if self._differentiable():
            return _train.gradient(self, x, skip_spatial_distortion, return_sdf)
        pts = _lib.f32c(x.reshape(-1, 3))
        wants = ["gradients"] + (["sampled_sdf"] if return_sdf and self.config.use_numerical_gradients else [])
        o = self._run(pts, None, None, 1, wants, apply_contraction=not skip_spatial_distortion)
        g = o["gradients"].view(*x.shape)
        if not return_sdf:
            return g
        pts_sdf = o["sampled_sdf"].t().reshape(6, *x.shape[:-1]) if "sampled_sdf" in o else None
        return g, pts_sdf

    def get_density(self, ray_samples):
        """sdf_field.py:467-474."""
        if self._differentiable():
            pos = ray_samples.frustums.get_start_positions()
            h = _train.forward_geonetwork(self, pos.reshape(-1, 3)).view(*ray_samples.frustums.shape, -1)
            return self.laplace_density(h[..., :1]), h[..., 1:]
        origins, directions, bins, shape = sample_geometry(ray_samples)
        o = self._run(origins, directions, bins, bins.shape[1] - 1, ("density", "geo_feature"), apply_contraction=False)
        return o["density"].view(*shape, 1), o["geo_feature"].view(*shape, -1)

    def get_alpha(self, ray_samples, sdf=None, gradients=None):
        """sdf_field.py:476-525."""
        if self._differentiable():
            if sdf is None or gradients is None:
                inputs = ray_samples.frustums.get_start_positions().reshape(-1, 3)
                inputs.requires_grad_(True)
                with torch.enable_grad():
                    sdf = _train.forward_geonetwork(self, inputs)[:, :1]
                with self.encoding.inputs_only_backward():
                    gradients = torch.autograd.grad(sdf, inputs, torch.ones_like(sdf), create_graph=True, retain_graph=True, only_inputs=True)[0]
                sdf = sdf.view(*ray_samples.frustums.shape, -1)
                gradients = gradients.view(*ray_samples.frustums.shape, -1)
            return _train.get_alpha(self, ray_samples, sdf, gradients)
        if sdf is None or gradients is None:
            # like the reference (and the training path), the gradient is autograd's at the un-contracted start positions, also when the
            # field uses numerical gradients elsewhere
            origins, directions, bins, shape = sample_geometry(ray_samples)
            o = self._run(origins, directions, bins, bins.shape[1] - 1, ("alpha",), apply_contraction=False, analytic_gradients=True)
            return o["alpha"].view(*shape, 1)
        return _train.get_alpha(self, ray_samples, sdf, gradients)

    def _appearance(self, camera_indices, R, device):
        c = self.config
        if self.training:
            if not c.use_appearance_embedding or camera_indices is None:
                return None
            idx = camera_indices.reshape(camera_indices.shape[0], -1)[:, 0].long()
            return _lib.f32c(self.embedding_appearance(idx).detach())
        if self.use_average_appearance_embedding:
            return _lib.f32c(self.embedding_appearance.mean(dim=0).detach()[None, :].expand(R, -1))
        return None

    def get_outputs(self, ray_samples, return_alphas=False, return_occupancy=False):
        """sdf_field.py:614-689."""
        if ray_samples.camera_indices is None:
            raise AttributeError("Camera indices are not provided.")
        if self._differentiable():
            return _train.get_outputs(self, ray_samples, return_alphas=return_alphas, return_occupancy=return_occupancy)
        origins, directions, bins, shape = sample_geometry(ray_samples)
        R, S = origins.shape[0], bins.shape[1] - 1
        wants = ["rgb", "density", "sdf", "normals", "gradients", "points_norm"]
        if self.config.use_numerical_gradients:
            wants.append("sampled_sdf")
        if return_alphas:
            wants.append("alpha")
        if return_occupancy:
            wants.append("occupancy")
        app = self._appearance(ray_samples.camera_indices, R, origins.device)
        o = self._run(origins, directions, bins, S, wants, apply_contraction=True, appearance=app)
        outputs = {
            FieldHeadNames.RGB: o["rgb"].view(*shape, 3),
            FieldHeadNames.DENSITY: o["density"].view(*shape, 1),
            FieldHeadNames.SDF: o["sdf"].view(*shape, 1),
            FieldHeadNames.NORMAL: o["normals"].view(*shape, 3),
            FieldHeadNames.GRADIENT: o["gradients"].view(*shape, 3),
            "points_norm": o["points_norm"].view(*shape, 1),
            "sampled_sdf": o["sampled_sdf"].view(*shape, 6) if "sampled_sdf" in o else None,
        }
        if return_alphas:
            outputs[FieldHeadNames.ALPHA] = o["alpha"].view(*shape, 1)
        if return_occupancy:
            outputs[FieldHeadNames.OCCUPANCY] = o["occupancy"].view(*shape, 1)
        return outputs

    def forward(self, ray_samples, return_alphas=False, return_occupancy=False):
        return self.get_outputs(ray_samples, return_alphas=return_alphas, return_occupancy=return_occupancy)
