"""Differentiable (training) path of SDFField.

What trains in the reference is ATen autograd over ``nn.Linear`` layers plus the ``tinycudann.Encoding`` operator
(nerfstudio/fields/sdf_field.py:380-410, :614-689).  This module is that composition over this package's kernels: the grid operator
(forward, backward, second-order backward for the eikonal term: sdfb200_grid_encode / _backward / _backward_backward, and their grouped
forms for the seven taps of a numerical-gradient sample) and, at precision bf16x3 / bf16, the dense layers on the tensor-core GEMMs of
linear_ops.py (closed under differentiation); precision "fp32" keeps ATen matmuls, the reference's exact arithmetic.
The fused tensor-core kernel (csrc/field_tc_kernel.cuh) is the rendering / sampling path (everything under ``torch.no_grad``: the NeuS /
error-bounded / UniSurf samplers, evaluation, mesh extraction).

Functions take the SDFField module as first argument; SDFField dispatches here when autograd is recording in training mode.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import linear_ops as _lo
from .field_heads import FieldHeadNames

# 21 icosahedron directions of the off-axis encoding (field_components/encodings.py:129-153), [3, 21]
_OFF_AXIS = [
    [0.8506508, 0, 0.5257311], [0.809017, 0.5, 0.309017], [0.5257311, 0.8506508, 0], [1, 0, 0], [0.809017, 0.5, -0.309017],
    [0.8506508, 0, -0.5257311], [0.309017, 0.809017, -0.5], [0, 0.5257311, -0.8506508], [0.5, 0.309017, -0.809017], [0, 1, 0],
    [-0.5257311, 0.8506508, 0], [-0.309017, 0.809017, -0.5], [0, 0.5257311, 0.8506508], [-0.309017, 0.809017, 0.5],
    [0.309017, 0.809017, 0.5], [0.5, 0.309017, 0.809017], [0.5, -0.309017, 0.809017], [0, 0, 1], [-0.5, 0.309017, 0.809017],
    [-0.809017, 0.5, 0.309017], [-0.809017, 0.5, -0.309017],
]  # fmt: skip


def nerf_encoding(x, num_frequencies: int, max_exp: float, include_input: bool, off_axis: bool = False):
    """NeRFEncoding.forward (encodings.py:167-208), min_freq_exp = 0."""
    freqs = 2 ** torch.linspace(0.0, max_exp, num_frequencies, device=x.device)
    base = x @ torch.tensor(_OFF_AXIS, device=x.device, dtype=x.dtype).T if off_axis else x
    scaled = (base[..., None] * freqs).reshape(*base.shape[:-1], -1)
    enc = torch.sin(torch.cat([scaled, scaled + torch.pi / 2.0], dim=-1))
    return torch.cat([enc, x], dim=-1) if include_input else enc


def _gemm_precision(field):
    """None -> ATen matmuls (precision "fp32": exact reference arithmetic); otherwise the tensor-core GEMMs of linear_ops at that precision."""
    mode = getattr(field.config, "train_gemm", "auto")
    prec = getattr(field.config, "precision", "fp32")
    if mode == "aten" or (mode == "auto" and prec == "fp32"):
        return None
    return "bf16" if prec == "bf16" else "bf16x3"


def _weight_of(lin):
    """the effective weight of a (weight-normed) nn.Linear, with autograd history to weight_g / weight_v (sdf_field.py:312-313)"""
    if hasattr(lin, "weight_v"):
        return torch._weight_norm(lin.weight_v, lin.weight_g, 0)
    return lin.weight


def _dense(field, lin, x, act: int = 0):
    """act(lin(x)) with act 0 none / 1 softplus(beta=100) / 2 relu.  x may carry zero padding columns beyond lin.in_features; on the
    tensor-core path the result is padded to a multiple of 16 columns (callers slice what they need)."""
    prec = _gemm_precision(field)
    k, n = lin.in_features, lin.out_features
    if prec is None:
        y = lin(x[:, :k] if x.shape[1] != k else x)
        return F.softplus(y, beta=100) if act == 1 else (torch.relu(y) if act == 2 else y)
    kp = _lo.pad16(k)
    if x.shape[1] < kp:
        x = F.pad(x, (0, kp - x.shape[1]))
    elif x.shape[1] > kp:
        x = x[:, :kp]
    return _lo.linear(x, _weight_of(lin), lin.bias, act, prec)


def forward_geonetwork(field, inputs):
    """sdf_field.py:380-410."""
    c = field.config
    if field.use_grid_feature:
        positions = (inputs + 2.0) / 4.0
        feature = field.encoding(positions)
        feature = feature * field.hash_encoding_mask.to(feature.device)
    else:
        feature = torch.zeros_like(inputs[:, :1].repeat(1, field.encoding.n_output_dims))
    if c.use_position_encoding:
        pe = nerf_encoding(inputs, c.position_encoding_max_degree, c.position_encoding_max_degree - 1, False, c.off_axis)
    else:                                                  # zeros of the encoding's shape (sdf_field.py:393-394) without evaluating it first
        pe = inputs.new_zeros(inputs.shape[0], (21 if c.off_axis else 3) * 2 * c.position_encoding_max_degree)
    parts = [inputs, pe, feature]
    width = sum(t.shape[1] for t in parts)
    if _gemm_precision(field) is not None and width % 16 != 0:
        parts.append(inputs.new_zeros(inputs.shape[0], _lo.pad16(width) - width))     # the GEMMs' K padding, written by the same concatenation
    x = torch.cat(parts, dim=-1)
    inputs = x[:, :width]
    for l in range(0, field.num_layers - 1):
        lin = getattr(field, "glin" + str(l))
        if l in field.skip_in:
            x = torch.cat([x[:, : lin.in_features - inputs.shape[1]], inputs], 1) / np.sqrt(2)
        x = _dense(field, lin, x, 1 if l < field.num_layers - 2 else 0)
    return x[:, : lin.out_features] if x.shape[1] != lin.out_features else x


def gradient(field, x, skip_spatial_distortion=False, return_sdf=False):
    """sdf_field.py:424-465."""
    if field.spatial_distortion is not None and not skip_spatial_distortion:
        x = field.spatial_distortion(x)
    points_sdf = None
    if field.config.use_numerical_gradients:
        delta = field.numerical_gradients_delta
        offs = torch.tensor([[delta, 0, 0], [-delta, 0, 0], [0, delta, 0], [0, -delta, 0], [0, 0, delta], [0, 0, -delta]], device=x.device, dtype=x.dtype)
        points = x[None] + offs.view(6, *([1] * (x.dim() - 1)), 3)
        with field.encoding.point_groups(6):               # the six taps of a sample share their table rows at all but the finest levels
            points_sdf = forward_geonetwork(field, points.view(-1, 3))[..., 0].view(6, *x.shape[:-1])
        gradients = torch.stack([0.5 * (points_sdf[0] - points_sdf[1]) / delta, 0.5 * (points_sdf[2] - points_sdf[3]) / delta,
                                 0.5 * (points_sdf[4] - points_sdf[5]) / delta], dim=-1)
    else:
        with torch.enable_grad():
            if not x.requires_grad:
                x.requires_grad_(True)
            y = forward_geonetwork(field, x)[:, :1]
            with field.encoding.inputs_only_backward():
                gradients = torch.autograd.grad(outputs=y, inputs=x, grad_outputs=torch.ones_like(y), create_graph=True, retain_graph=True, only_inputs=True)[0]
    return (gradients, points_sdf) if return_sdf else gradients


def get_colors(field, points, directions, gradients, geo_features, camera_indices):
    """sdf_field.py:532-612."""
    c = field.config
    gf = geo_features.view(-1, c.geo_feat_dim)
    if c.use_diffuse_color:
        raw_rgb_diffuse = field.diffuse_color_pred(gf)
    if c.use_specular_tint:
        tint = torch.sigmoid(field.specular_tint_pred(gf))
    normals = F.normalize(gradients, p=2, dim=-1)
    if c.use_reflections:
        refdirs = 2.0 * torch.sum(normals * -directions, dim=-1, keepdim=True) * normals + directions
        d = nerf_encoding(refdirs, 4, 3.0, True)
    else:
        d = nerf_encoding(directions, 4, 3.0, True)
    if field.training:
        emb = field.embedding_appearance(camera_indices)
        if not c.use_appearance_embedding:
            emb = torch.zeros_like(emb)
    elif field.use_average_appearance_embedding:
        emb = torch.ones((*directions.shape[:-1], c.appearance_embedding_dim), device=directions.device) * field.embedding_appearance.mean(dim=0)
    else:
        emb = torch.zeros((*directions.shape[:-1], c.appearance_embedding_dim), device=directions.device)
    emb = emb.view(-1, c.appearance_embedding_dim)
    h = [d, gf, emb] if c.use_diffuse_color else [points, d, gradients, gf, emb]
    if c.use_n_dot_v:
        h.append(torch.sum(normals * directions, dim=-1, keepdim=True))
    h = torch.cat(h, dim=-1)
    for l in range(0, field.num_layers_color - 1):
        h = _dense(field, getattr(field, "clin" + str(l)), h, 2 if l < field.num_layers_color - 2 else 0)
    rgb = torch.sigmoid(h[:, :3])
    if c.use_diffuse_color:
        diffuse_linear = torch.sigmoid(raw_rgb_diffuse - math.log(3.0))
        specular_linear = tint * rgb if c.use_specular_tint else 0.5 * rgb
        rgb = torch.clamp(specular_linear + diffuse_linear, 0.0, 1.0)
    return rgb * (1 + 2 * c.rgb_padding) - c.rgb_padding


def get_alpha(field, ray_samples, sdf, gradients):
    """sdf_field.py:476-525."""
    inv_s = field.deviation_network.get_variance()
    true_cos = (ray_samples.frustums.directions * gradients).sum(-1, keepdim=True)
    r = field._cos_anneal_ratio
    iter_cos = -(F.relu(-true_cos * 0.5 + 0.5) * (1.0 - r) + F.relu(-true_cos) * r)
    deltas = ray_samples.deltas
    prev_cdf = torch.sigmoid((sdf - iter_cos * deltas * 0.5) * inv_s)
    next_cdf = torch.sigmoid((sdf + iter_cos * deltas * 0.5) * inv_s)
    return ((prev_cdf - next_cdf + 1e-5) / (prev_cdf + 1e-5)).clip(0.0, 1.0)


def get_outputs(field, ray_samples, return_alphas=False, return_occupancy=False):
    """sdf_field.py:614-689."""
    if ray_samples.camera_indices is None:
        raise AttributeError("Camera indices are not provided.")
    c = field.config
    shape = ray_samples.frustums.directions.shape[:-1]
    camera_indices = ray_samples.camera_indices.squeeze()
    inputs = ray_samples.frustums.get_start_positions().reshape(-1, 3)
    directions_flat = ray_samples.frustums.directions.reshape(-1, 3)
    if field.spatial_distortion is not None:
        inputs = field.spatial_distortion(inputs)
    points_norm = inputs.norm(dim=-1)
    if c.use_numerical_gradients:
        # sdf_field.py:640-645 evaluates the geo network at x and (inside gradient()) at x +- delta e_i: row-wise independent, so the seven
        # evaluations run as ONE batch [7, N] here -- same values, and the grid operator merges the taps of a sample (Encoding.point_groups).
        # The positions need no gradient in this mode (the reference sets requires_grad and never uses it).
        delta = field.numerical_gradients_delta
        offs = torch.tensor([[0, 0, 0], [delta, 0, 0], [-delta, 0, 0], [0, delta, 0], [0, -delta, 0], [0, 0, delta], [0, 0, -delta]], device=inputs.device,
                            dtype=inputs.dtype)
        n = inputs.shape[0]
        with torch.enable_grad(), field.encoding.point_groups(7):
            h_all = forward_geonetwork(field, (inputs[None] + offs[:, None, :]).view(-1, 3))
        h = h_all[:n]
        sdf, geo_feature = torch.split(h, [1, c.geo_feat_dim], dim=-1)
        ps = h_all[n:, 0].view(6, n)
        gradients = torch.stack([0.5 * (ps[0] - ps[1]) / delta, 0.5 * (ps[2] - ps[3]) / delta, 0.5 * (ps[4] - ps[5]) / delta], dim=-1)
        sampled_sdf = ps.view(-1, *shape).permute(1, 2, 0).contiguous()
    else:
        if not inputs.requires_grad:
            inputs.requires_grad_(True)
        with torch.enable_grad():
            h = forward_geonetwork(field, inputs)
            sdf, geo_feature = torch.split(h, [1, c.geo_feat_dim], dim=-1)
        with field.encoding.inputs_only_backward():
            gradients = torch.autograd.grad(outputs=sdf, inputs=inputs, grad_outputs=torch.ones_like(sdf), create_graph=True, retain_graph=True,
                                            only_inputs=True)[0]
        sampled_sdf = None
    rgb = get_colors(field, inputs, directions_flat, gradients, geo_feature, camera_indices)
    density = field.laplace_density(sdf)
    rgb, sdf, density = rgb.view(*shape, -1), sdf.view(*shape, -1), density.view(*shape, -1)
    gradients = gradients.view(*shape, -1)
    outputs = {
        FieldHeadNames.RGB: rgb,
        FieldHeadNames.DENSITY: density,
        FieldHeadNames.SDF: sdf,
        FieldHeadNames.NORMAL: F.normalize(gradients, p=2, dim=-1),
        FieldHeadNames.GRADIENT: gradients,
        "points_norm": points_norm.view(*shape, -1),
        "sampled_sdf": sampled_sdf,
    }
    if return_alphas:
        outputs[FieldHeadNames.ALPHA] = get_alpha(field, ray_samples, sdf, gradients)
    if return_occupancy:
        outputs[FieldHeadNames.OCCUPANCY] = field.get_occupancy(sdf)
    return outputs
