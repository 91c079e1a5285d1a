"""H100-native drop-in for ``nerfstudio.fields.nerfacto_field.TCNNNerfactoField`` (nerfacto_field.py:67-318), the field behind
``background_model="grid"`` of neus-facto-angelo and bakedangelo (models/base_surface_model.py:181-187), which the reference builds
from four tiny-cuda-nn modules.  Same constructor, ``get_density``, ``get_outputs``, ``density_fn`` and ``forward``.

* Evaluation (``torch.no_grad()`` or eval mode): ``forward`` is one kernel launch (sdfb200_nerfacto_field_forward): hash grid ->
  ReLU MLP -> exp for the density, tcnn SphericalHarmonics(4) + geometry feature + appearance -> ReLU MLP -> sigmoid for the colour.
* Training (autograd recording in train mode), and ``get_density`` / ``get_outputs`` / ``density_fn`` called on their own: the
  differentiable composition of this package's grid operator, ATen matmuls on views of the flat parameters, SH-4 in torch,
  ``trunc_exp`` and ``nn.Embedding``.

Parameters keep the reference's names: ``mlp_base.params`` (network weights, then the grid table: the proposal networks' layout
with an output of 1 + geo_feat_dim), ``mlp_head.params`` ([HC, pad16(16 + geo + app)] | (n - 1) x [HC, HC] | [16, HC]),
``embedding_appearance.embedding.weight``, ``aabb`` and the empty ``direction_encoding.params`` / ``position_encoding.params``, so
``checkpoint.load_background_field_checkpoint`` loads a reference checkpoint.

tiny-cuda-nn is not vendored in the reference, so these points restate its published behaviour and are UNPINNED (DESIGN.md section 4):
* SH signs: tcnn's SH uses the Condon-Shortley phase, i.e. nerfstudio's ``components_from_spherical_harmonics`` (utils/math.py:46-70)
  with components 1, 3, 5, 7, 9, 11, 13 and 15 negated;
* the padded input columns of ``mlp_head`` (64 for the default shape) contribute nothing, as for the proposal networks;
* network weights come before the encoding's parameters inside ``NetworkWithInputEncoding.params``;
* parameter-free encodings register a zero-length ``params`` (they appear in the state dict);
* tcnn computes in fp16; this package computes in fp32.

Not supported (``SurfaceModel`` uses none of them): ``compute_normals=True``, transient embeddings, semantics, predicted normals.
"""
import math
from typing import Optional

import numpy as np
import torch
from torch import nn

from . import _lib
from .autograd_ops import training_step
from .density_fields import _NetworkWithInputEncoding, _TruncExp, fully_fused_mlp, fully_fused_weights, kernel_aabb, normalized_positions
from .field_heads import FieldHeadNames
from .rays import point_or_ray_inputs
from .sdf_field import _Embedding
from .spatial_distortions import contraction_code

BASE_RES, FEATURES_PER_LEVEL = 16, 2   # fixed by the reference constructor (nerfacto_field.py:126-127)
SH_DIM = 16                            # tcnn SphericalHarmonics, degree 4


def sh4(x: torch.Tensor) -> torch.Tensor:
    """tcnn SphericalHarmonics degree 4 of x in [-1,1]^3 ([..., 3] -> [..., 16])."""
    x_, y, z = x[..., 0], x[..., 1], x[..., 2]
    xx, yy, zz = x_ * x_, y * y, z * z
    return torch.stack([
        torch.full_like(x_, 0.28209479177387814), -0.4886025119029199 * y, 0.4886025119029199 * z, -0.4886025119029199 * x_,
        1.0925484305920792 * x_ * y, -1.0925484305920792 * y * z, 0.9461746957575601 * zz - 0.31539156525251999, -1.0925484305920792 * x_ * z,
        0.5462742152960396 * (xx - yy), -0.5900435899266435 * y * (3 * xx - yy), 2.890611442640554 * x_ * y * z, -0.4570457994644658 * y * (5 * zz - 1),
        0.3731763325901154 * z * (5 * zz - 3), -0.4570457994644658 * x_ * (5 * zz - 1), 1.445305721320277 * z * (xx - yy), -0.5900435899266435 * x_ * (xx - 3 * yy),
    ], dim=-1)  # fmt: skip


class _ParamFreeEncoding(nn.Module):
    """tcnn.Encoding without parameters (SphericalHarmonics, Frequency): tcnn registers a zero-length ``params`` even then.  The
    encodings themselves are evaluated inside the kernel / by ``sh4``."""

    def __init__(self, n_output_dims: int):
        super().__init__()
        self.n_output_dims = n_output_dims
        self.params = nn.Parameter(torch.zeros(0))


class _Network(nn.Module):
    """tcnn.Network(FullyFusedMLP, ReLU, no biases) as one flat parameter vector: [hidden, in_pad] | (n_hidden - 1) x [hidden, hidden] |
    [16, hidden], in_pad = n_input_dims rounded up to 16, rows 0..n_output_dims-1 of the output matrix live."""

    def __init__(self, n_input_dims, n_output_dims, hidden_dim, n_hidden_layers, seed=1337):
        super().__init__()
        self.in_dim, self.in_pad = n_input_dims, (n_input_dims + 15) // 16 * 16
        self.hidden_dim, self.n_hidden_layers, self.n_output_dims = hidden_dim, n_hidden_layers, n_output_dims
        g = torch.Generator().manual_seed(seed)
        self.params = nn.Parameter(fully_fused_weights(g, n_input_dims, hidden_dim, n_hidden_layers, n_output_dims))

    def forward(self, x):
        """[N, in_dim] -> [N, n_output_dims] (no output activation)."""
        return fully_fused_mlp(x, self.params, self.in_dim, self.in_pad, self.hidden_dim, self.n_hidden_layers, self.n_output_dims)


class TCNNNerfactoField(nn.Module):
    """nerfacto_field.py:67-318."""

    def __init__(self, aabb, num_images: int, num_layers: int = 2, hidden_dim: int = 64, geo_feat_dim: int = 15, num_levels: int = 16,
                 max_res: int = 1024, log2_hashmap_size: int = 19, num_layers_color: int = 3, num_layers_transient: int = 2,
                 hidden_dim_color: int = 64, hidden_dim_transient: int = 64, appearance_embedding_dim: int = 32, transient_embedding_dim: int = 16,
                 use_transient_embedding: bool = False, use_semantics: bool = False, num_semantic_classes: int = 100, use_pred_normals: bool = False,
                 use_average_appearance_embedding: bool = False, spatial_distortion=None) -> None:
        super().__init__()
        if use_transient_embedding or use_semantics or use_pred_normals:
            raise NotImplementedError("transient embeddings, semantics and predicted normals are not supported (SurfaceModel uses none of them)")
        if hidden_dim not in (16, 32, 64) or hidden_dim_color not in (16, 32, 64):
            raise NotImplementedError("hidden_dim and hidden_dim_color must be 16, 32 or 64")
        if num_layers not in (2, 3, 4) or num_layers_color not in (2, 3, 4):
            raise NotImplementedError("num_layers and num_layers_color must be 2, 3 or 4")
        if not 0 <= geo_feat_dim <= 15 or appearance_embedding_dim < 0 or SH_DIM + geo_feat_dim + appearance_embedding_dim > 64:
            raise NotImplementedError("needs geo_feat_dim <= 15 and 16 + geo_feat_dim + appearance_embedding_dim <= 64")
        self.aabb = nn.Parameter(torch.as_tensor(aabb, dtype=torch.float32), requires_grad=False)
        self.geo_feat_dim = geo_feat_dim
        self.spatial_distortion = spatial_distortion
        self.num_images = num_images
        self.appearance_embedding_dim = appearance_embedding_dim
        self.embedding_appearance = _Embedding(num_images, appearance_embedding_dim)
        self.use_average_appearance_embedding = use_average_appearance_embedding
        self.use_transient_embedding, self.use_semantics, self.use_pred_normals = use_transient_embedding, use_semantics, use_pred_normals
        growth = float(np.exp((np.log(max_res) - np.log(BASE_RES)) / (num_levels - 1)))
        self.direction_encoding = _ParamFreeEncoding(SH_DIM)
        self.position_encoding = _ParamFreeEncoding(3 * 2 * 2)   # Frequency, n_frequencies = 2
        self.mlp_base = _NetworkWithInputEncoding(num_levels, FEATURES_PER_LEVEL, log2_hashmap_size, BASE_RES, growth, hidden_dim, num_layers - 1,
                                                  n_output_dims=1 + geo_feat_dim)
        self.mlp_head = _Network(SH_DIM + geo_feat_dim + appearance_embedding_dim, 3, hidden_dim_color, num_layers_color - 1)
        self._density_before_activation = None
        self._locations = None
        self._positions_of_last_call = None

    # ------------------------------------------------------------------ reference attributes
    @property
    def _sample_locations(self):
        """Normalised positions of the last evaluation (Field._sample_locations).  The kernel path does not materialise them: it keeps the
        last call's ``frustums.get_positions`` (and through it that call's frustum tensors, until the next call) and normalises on first
        access.  The composition path stores them like the reference."""
        if self._locations is None and self._positions_of_last_call is not None:
            with torch.no_grad():
                self._locations = normalized_positions(self._positions_of_last_call(), self.aabb, self.spatial_distortion)
        return self._locations

    def _contraction_code(self) -> int:
        return contraction_code(self.spatial_distortion)

    # ------------------------------------------------------------------ differentiable composition
    def _density_from_positions(self, positions):
        x01 = normalized_positions(positions, self.aabb, self.spatial_distortion)
        self._locations, self._positions_of_last_call = x01, None
        h = self.mlp_base(x01.reshape(-1, 3)).view(*positions.shape[:-1], -1)
        density_before_activation, base_mlp_out = torch.split(h, [1, self.geo_feat_dim], dim=-1)
        self._density_before_activation = density_before_activation
        return _TruncExp.apply(density_before_activation), base_mlp_out

    def get_density(self, ray_samples):
        """nerfacto_field.py:223-243."""
        return self._density_from_positions(ray_samples.frustums.get_positions())

    def density_fn(self, positions: torch.Tensor) -> torch.Tensor:
        """fields/base_field.py:48-65: the density at `positions` (a zero-length frustum there)."""
        return self._density_from_positions(positions)[0]

    def _appearance_mode(self):
        if self.training:
            return "camera"
        return "mean" if self.use_average_appearance_embedding else "zeros"

    def get_outputs(self, ray_samples, density_embedding: Optional[torch.Tensor] = None):
        """nerfacto_field.py:245-318 without transients, semantics and predicted normals."""
        assert density_embedding is not None
        if ray_samples.camera_indices is None:
            raise AttributeError("Camera indices are not provided.")
        directions = (ray_samples.frustums.directions + 1.0) / 2.0          # get_normalized_directions
        shape = directions.shape[:-1]
        d = sh4(directions.reshape(-1, 3) * 2.0 - 1.0)                      # tcnn maps its [0,1] input back with 2x - 1
        mode = self._appearance_mode()
        A = self.appearance_embedding_dim
        if mode == "camera" and A > 0:
            app = self.embedding_appearance(ray_samples.camera_indices.squeeze())
        elif mode == "camera":
            # no lookup into an empty embedding: the CUDA backward of nn.Embedding with embedding_dim = 0 takes the weight's row stride (1)
            # as its feature count and reads and writes one element per index out of bounds
            app = torch.zeros((*shape, 0), device=directions.device)
        elif mode == "mean":
            app = torch.ones((*shape, A), device=directions.device) * self.embedding_appearance.mean(dim=0)
        else:
            app = torch.zeros((*shape, A), device=directions.device)
        n = d.shape[0]   # explicit row counts: geo_feat_dim or A may be 0, and reshape(-1, 0) cannot infer the rows
        h = torch.cat([d, density_embedding.reshape(n, self.geo_feat_dim), app.reshape(n, A)], dim=-1)
        rgb = torch.sigmoid(self.mlp_head(h)).view(*shape, -1)
        return {FieldHeadNames.RGB: rgb}

    # ------------------------------------------------------------------ forward
    def forward(self, ray_samples, compute_normals: bool = False):
        """fields/base_field.py:104-123."""
        if compute_normals:
            raise NotImplementedError("compute_normals=True is not supported by the nerfacto background field")
        if training_step(self, self.parameters()):
            density, density_embedding = self.get_density(ray_samples)
            outputs = self.get_outputs(ray_samples, density_embedding=density_embedding)
            outputs[FieldHeadNames.DENSITY] = density
            return outputs
        if ray_samples.camera_indices is None:
            raise AttributeError("Camera indices are not provided.")
        density, rgb = self._kernel_forward(ray_samples)
        return {FieldHeadNames.RGB: rgb, FieldHeadNames.DENSITY: density}

    def _kernel_forward(self, ray_samples):
        """One sdfb200_nerfacto_field_forward launch, in ray or point mode (rays.point_or_ray_inputs)."""
        lib = _lib.load()
        dev = self.aabb.device
        _lib.require_cuda(dev, "TCNNNerfactoField")
        origins, directions, bins, n_rows, S, shape = point_or_ray_inputs(ray_samples)
        cams = ray_samples.camera_indices
        cam_rows = cams.reshape(n_rows, -1)[:, 0] if bins is not None else cams.reshape(-1)
        N = math.prod(shape)
        mode = self._appearance_mode()
        stride = self.appearance_embedding_dim
        if mode == "camera":
            app = _lib.f32c(self.embedding_appearance(cam_rows.long()).detach())
        elif mode == "mean":
            app, stride = _lib.f32c(self.embedding_appearance.mean(dim=0).detach()), 0
        else:
            app = None
        density = torch.empty(N, device=dev, dtype=torch.float32)
        rgb = torch.empty(N, 3, device=dev, dtype=torch.float32)
        pre = torch.empty(N, device=dev, dtype=torch.float32)
        nb, nh = self.mlp_base, self.mlp_head
        p = nb.params.detach()
        nd = self._desc(S)
        aabb = kernel_aabb(self.aabb, nd.contraction)
        _lib.check(lib.sdfb200_nerfacto_field_forward(nb.kernel_desc(), nd, p[nb.n_net:].data_ptr(), p.data_ptr(), nh.params.detach().data_ptr(),
                                                      _lib.ptr(aabb), _lib.ptr(origins), _lib.ptr(directions), _lib.ptr(bins), n_rows, _lib.ptr(app),
                                                      stride, density.data_ptr(), rgb.data_ptr(), pre.data_ptr(), None, _lib.stream_ptr()),
                   "sdfb200_nerfacto_field_forward")
        self._density_before_activation = pre.view(*shape, 1)
        self._locations, self._positions_of_last_call = None, ray_samples.frustums.get_positions
        return density.view(*shape, 1), rgb.view(*shape, 3)

    def _desc(self, n_samples: int) -> "_lib.NerfactoDesc":
        d = _lib.NerfactoDesc()
        nb, nh = self.mlp_base, self.mlp_head
        d.hidden_dim, d.n_hidden_layers = nb.hidden_dim, nb.n_hidden_layers
        d.hidden_dim_color, d.n_hidden_layers_color = nh.hidden_dim, nh.n_hidden_layers
        d.geo_feat_dim, d.appearance_dim = self.geo_feat_dim, self.appearance_embedding_dim
        d.contraction, d.n_samples = self._contraction_code(), n_samples
        return d
