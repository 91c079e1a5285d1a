"""TEST INFRASTRUCTURE -- CPU restatement of the nerfacto background field (TCNNNerfactoField, nerfstudio/fields/nerfacto_field.py:67-318,
through Field.forward, fields/base_field.py:104-123) and of SurfaceModel.forward_background_field_and_merge
(models/base_surface_model.py:257-290).  Functional, in the dtype of its inputs (fp32 or fp64).

The composition (normalisation, the [1, geo] split, trunc_exp, direction normalisation, concat order, appearance modes, sigmoid) is pinned
against the unmodified reference by tests/golden/nerfacto_field.npz (oracle/make_golden_nerfacto.py).  What tiny-cuda-nn computes inside
its modules (SH signs, padded columns, parameter order, fp16 arithmetic) is restated from its published behaviour: PARITY UNPINNED.
"""
import torch

from . import hashgrid
from .field import scene_contraction

BASE_RES, FEATURES_PER_LEVEL, SH_DIM = 16, 2, 16


def sh4_tcnn(x):
    """tcnn SphericalHarmonics degree 4 of x in [-1,1]^3: nerfstudio's components_from_spherical_harmonics (utils/math.py:46-70, levels = 4)
    with tcnn's Condon-Shortley signs (components 1, 3, 5, 7, 9, 11, 13, 15 negated)."""
    x_, y, z = x[..., 0], x[..., 1], x[..., 2]
    xx, yy, zz = x_**2, y**2, z**2
    c = [
        torch.full_like(x_, 0.28209479177387814),
        0.4886025119029199 * y, 0.4886025119029199 * z, 0.4886025119029199 * x_,
        1.0925484305920792 * x_ * y, 1.0925484305920792 * y * z, 0.9461746957575601 * zz - 0.31539156525251999, 1.0925484305920792 * x_ * z,
        0.5462742152960396 * (xx - yy),
        0.5900435899266435 * y * (3 * xx - yy), 2.890611442640554 * x_ * y * z, 0.4570457994644658 * y * (5 * zz - 1),
        0.3731763325901154 * z * (5 * zz - 3), 0.4570457994644658 * x_ * (5 * zz - 1), 1.445305721320277 * z * (xx - yy),
        0.5900435899266435 * x_ * (xx - 3 * yy),
    ]  # fmt: skip
    for k in (1, 3, 5, 7, 9, 11, 13, 15):
        c[k] = -c[k]
    return torch.stack(c, dim=-1)


def mlp(x, weights, in_dim, hidden, n_hidden, n_out):
    """tcnn FullyFusedMLP (ReLU, no biases, no output activation) over the flat weights [hidden, in_pad] | (n_hidden-1) x [hidden, hidden] |
    [16, hidden]: the layer walk of oracle.density with an output of n_out rows."""
    in_pad = (in_dim + 15) // 16 * 16
    o = hidden * in_pad
    h = torch.relu(x @ weights[:o].view(hidden, in_pad)[:, :in_dim].t())
    for _ in range(n_hidden - 1):
        h = torch.relu(h @ weights[o: o + hidden * hidden].view(hidden, hidden).t())
        o += hidden * hidden
    return h @ weights[o: o + 16 * hidden].view(16, hidden)[:n_out].t()


def normalize(positions, aabb=None, contraction=None):
    """get_density's normalisation (nerfacto_field.py:225-231): SceneContraction then (x + 2) / 4, or SceneBox.get_normalized_positions."""
    if contraction is not None:
        return (scene_contraction(positions, contraction) + 2.0) / 4.0
    return (positions - aabb[0]) / (aabb[1] - aabb[0])


def midpoints(origins, directions, starts, ends):
    """Frustums.get_positions (cameras/rays.py): origins + directions * (starts + ends) / 2, per sample."""
    return origins + directions * (starts + ends) / 2


class NerfactoSpec:
    def __init__(self, num_levels=16, max_res=1024, log2_hashmap_size=19, hidden_dim=64, num_layers=2, geo_feat_dim=15, hidden_dim_color=64,
                 num_layers_color=3, appearance_embedding_dim=32):
        self.num_levels, self.max_res, self.log2_hashmap_size = num_levels, max_res, log2_hashmap_size
        self.hidden_dim, self.num_layers, self.geo_feat_dim = hidden_dim, num_layers, geo_feat_dim
        self.hidden_dim_color, self.num_layers_color, self.appearance_embedding_dim = hidden_dim_color, num_layers_color, appearance_embedding_dim

    @property
    def growth(self):
        import numpy as np

        return float(np.exp((np.log(self.max_res) - np.log(BASE_RES)) / (self.num_levels - 1)))

    def meta(self):
        return hashgrid.tcnn_grid_meta(self.num_levels, FEATURES_PER_LEVEL, self.log2_hashmap_size, BASE_RES, self.growth)

    def n_base_net(self):
        in_pad = (self.num_levels * FEATURES_PER_LEVEL + 15) // 16 * 16
        H = self.hidden_dim
        return H * in_pad + (self.num_layers - 2) * H * H + 16 * H


def density(x01, base_params, spec: NerfactoSpec):
    """mlp_base on normalised positions [N,3] -> (density [N], pre-activation [N], geometry feature [N, geo])."""
    n_net = spec.n_base_net()
    feat = hashgrid.encode_tcnn_layout(x01, base_params[n_net:].view(-1, FEATURES_PER_LEVEL), spec.meta(), FEATURES_PER_LEVEL, False)
    h = mlp(feat, base_params[:n_net], spec.num_levels * FEATURES_PER_LEVEL, spec.hidden_dim, spec.num_layers - 1, 1 + spec.geo_feat_dim)
    pre = h[:, 0]
    return torch.exp(pre), pre, h[:, 1:]


def rgb(directions, geo, appearance, head_params, spec: NerfactoSpec):
    """get_outputs (nerfacto_field.py:245-318): directions [N,3], geo [N, geo], appearance [N, A] -> rgb [N,3]."""
    d01 = (directions + 1.0) / 2.0                        # get_normalized_directions
    sh = sh4_tcnn(d01 * 2 - 1)                           # tcnn maps its input back with 2x - 1
    h = torch.cat([sh, geo, appearance], dim=-1)
    out = mlp(h, head_params, SH_DIM + spec.geo_feat_dim + spec.appearance_embedding_dim, spec.hidden_dim_color, spec.num_layers_color - 1, 3)
    return torch.sigmoid(out)


def field(positions, directions, appearance, base_params, head_params, spec: NerfactoSpec, aabb=None, contraction=None):
    """positions / directions [N,3], appearance [N, A] -> dict(density [N], pre [N], geo [N, geo], rgb [N,3], x01 [N,3])."""
    x01 = normalize(positions, aabb, contraction)
    dens, pre, geo = density(x01, base_params, spec)
    return {"density": dens, "pre": pre, "geo": geo, "rgb": rgb(directions, geo, appearance, head_params, spec), "x01": x01}


def merge_background(alpha, rgb_fg, start_positions, deltas, density_bg, rgb_bg):
    """forward_background_field_and_merge (base_surface_model.py:257-290): inside mask on |start position| < 1, background alpha =
    RaySamples.get_alphas = 1 - exp(-density * delta).  alpha / density_bg / deltas [..., 1], rgb [..., 3]."""
    inside = (start_positions.norm(dim=-1, keepdim=True) < 1.0).to(alpha.dtype)
    alpha_bg = 1 - torch.exp(-(deltas * density_bg))
    return alpha * inside + (1.0 - inside) * alpha_bg, rgb_fg * inside + (1.0 - inside) * rgb_bg
