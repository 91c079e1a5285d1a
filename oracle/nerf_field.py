"""TEST INFRASTRUCTURE -- CPU restatement of the vanilla NeRF background field and of the background branch of SurfaceModel.

* ``field``: NeRFField.get_density + get_outputs (nerfstudio/fields/vanilla_nerf_field.py:91-114): positions (frustum midpoints,
  cameras/rays.py:93-106) -> SceneContraction (spatial_distortions.py:66-73) -> NeRFEncoding (encodings.py:167-208) -> mlp_base
  (field_components/mlp.py:80-99, ReLU between the layers and as out_activation, skip = cat([encoding, x])) -> density = softplus of
  field_output_density (field_heads.py:99-108); rgb = sigmoid of field_heads.0 (field_heads.py:111-120) on mlp_head(cat([dir-enc, base])).
* ``background_branch``: base_surface_model.py:313-329: nears <- fars, fars <- far_plane_bg, LinearDisparitySampler (ray_samplers.py:154-175,
  eval: no jitter), the field, get_weights (rays.py:146-192), RGBRenderer (renderers.py:53-118) and rgb + bg_transmittance * rgb_bg.

Parameters are a state dict with the reference's names.  Runs in the dtype of its inputs (fp32 or fp64).
"""
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch

from . import render, samplers
from .field import nerf_encoding, scene_contraction


@dataclass
class NerfSpec:
    pe: Tuple[int, float, float, bool] = (10, 0.0, 9.0, True)     # num_frequencies, min_freq_exp, max_freq_exp, include_input
    de: Tuple[int, float, float, bool] = (4, 0.0, 3.0, True)
    base_layers: int = 8
    head_layers: int = 2
    skips: Tuple[int, ...] = (4,)
    contraction: Optional[str] = "linf"                            # None | 'linf' | 'l2'


def midpoints(origins, directions, starts, ends):
    """Frustums.get_positions: origins + directions * (starts + ends) / 2 (rays.py:93-106)."""
    return origins + directions * (starts + ends) / 2


def _linear(x, params, name):
    return x @ params[name + ".weight"].to(x.dtype).T + params[name + ".bias"].to(x.dtype)


def mlp(in_tensor, params, prefix, num_layers, skips=()):
    x = in_tensor
    for i in range(num_layers):
        if i in skips:
            x = torch.cat([in_tensor, x], -1)
        x = torch.relu(_linear(x, params, f"{prefix}.layers.{i}"))
    return x


def encode(x, enc):
    n, lo, hi, inc = enc
    return nerf_encoding(x, n, lo, hi, inc)


def field(positions, directions, params: Dict[str, torch.Tensor], spec: NerfSpec, contracted: bool = False):
    """positions / directions [..., 3] -> {contracted, encoding, density [..., 1], embedding [..., 256], rgb [..., 3]}.  With ``contracted``
    the positions are taken as already contracted."""
    x = positions if contracted else scene_contraction(positions, spec.contraction)
    pe = encode(x, spec.pe)
    base = mlp(pe, params, "mlp_base", spec.base_layers, spec.skips)
    density = torch.nn.functional.softplus(_linear(base, params, "field_output_density.net"))
    de = encode(directions, spec.de)
    head = mlp(torch.cat([de, base], dim=-1), params, "mlp_head", spec.head_layers)
    rgb = torch.sigmoid(_linear(head, params, "field_heads.0.net"))
    return {"contracted": x, "encoding": pe, "dir_encoding": de, "density": density, "embedding": base, "rgb": rgb}


def background_branch(origins, directions, fars, bg_transmittance, rgb_fg, params, spec: NerfSpec, background, num_samples: int = 32,
                      far_plane_bg: float = 1000.0):
    """origins / directions [R,3], fars [R,1] (the foreground's far plane), bg_transmittance [R,1], rgb_fg [R,3] (the rendered foreground),
    background [3] -> {bins [R,S+1], weights [R,S], rgb_bg [R,3], rgb [R,3]} in eval mode."""
    bins = samplers.spaced_sampler(fars, torch.ones_like(fars) * far_plane_bg, num_samples, "lindisp")
    eu = bins.euclid
    R, S = eu.shape[0], num_samples
    pos = midpoints(origins[:, None, :], directions[:, None, :], eu[:, :-1, None], eu[:, 1:, None])
    fo = field(pos, directions[:, None, :].expand(R, S, 3), params, spec)
    weights, _ = samplers.weights_from_density(bins.deltas, fo["density"][..., 0])
    rgb_bg = render.render_rgb(fo["rgb"], weights[..., None], background)
    return {"bins": eu, "weights": weights, "rgb_bg": rgb_bg, "rgb": rgb_fg + bg_transmittance * rgb_bg, "field": fo}
