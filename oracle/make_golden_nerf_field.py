"""TEST INFRASTRUCTURE -- mints tests/golden/nerf_field.npz + nerf_field.json from the UNMODIFIED reference NeRFField
(nerfstudio/fields/vanilla_nerf_field.py:37-114) and the background branch of SurfaceModel.get_outputs (models/base_surface_model.py:313-329),
run on CPU (build container only):

* the constructor signatures of NeRFField and NeRFEncoding, the state-dict names / shapes at SurfaceModel's shape (:188-201);
* for seeded parameters (``seeded_params``) and a seeded case (4 rays x 32 background samples from the reference LinearDisparitySampler
  between the far plane and 1000, plus 64 points), under the L-inf and L2 SceneContraction and none: the contracted positions, the
  position encoding, density, density embedding and rgb;
* the reference's own eval-mode background-branch outputs for a fixed bg_transmittance and foreground rgb: bins, weights, rgb_bg and the
  merged rgb.

    python -m oracle.make_golden_nerf_field
"""
import inspect
import json
import os
import warnings

import numpy as np
import torch

from . import ref_import

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
R, S, NPTS = 4, 32, 64
FAR_PLANE_BG = 1000.0
NORMS = ("linf", "l2", "none")
BACKGROUND = [0.2, 0.5, 0.9]


def default_repr(v):
    """A constructor default as JSON: plain values as they are, objects by their type name (tuples of objects element-wise)."""
    if v is inspect.Parameter.empty:
        return "<required>"
    if v is None or isinstance(v, (bool, int, float, str)):
        return v
    if isinstance(v, tuple):
        return [default_repr(x) for x in v]
    return type(v).__name__


def signature(fn):
    return [[n, default_repr(p.default)] for n, p in inspect.signature(fn).parameters.items() if n != "self"]


def seeded_params(shapes, seed=3):
    """{name: shape} -> parameters with He-scaled weights and spread biases, so that the ReLUs stay alive and every output varies."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, shape in shapes.items():
        if name.endswith(".weight"):
            out[name] = torch.randn(*shape, generator=g) * (2.0 / shape[1]) ** 0.5
        else:
            out[name] = torch.randn(*shape, generator=g) * 0.2
    return out


def seeded_inputs(seed=0):
    """4 rays from inside the unit sphere region outwards (fars 1.5-3.5) and 64 points spread over [-60, 60]^3 (contracted and not)."""
    g = torch.Generator().manual_seed(seed)
    o = torch.randn(R, 3, generator=g) * 0.3
    d = torch.randn(R, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True)
    fars = 1.5 + 2.0 * torch.rand(R, 1, generator=g)
    pts = torch.randn(NPTS, 3, generator=g) * torch.logspace(-1, 1.8, NPTS)[:, None]
    pdirs = torch.randn(NPTS, 3, generator=g)
    pdirs = pdirs / pdirs.norm(dim=-1, keepdim=True)
    bg_t = torch.rand(R, 1, generator=g)
    rgb_fg = torch.rand(R, 3, generator=g) * (1 - bg_t)
    return o, d, fars, pts, pdirs, bg_t, rgb_fg


def main():
    ref_import.install_shims()
    warnings.simplefilter("ignore")
    from nerfstudio.cameras.rays import Frustums, RayBundle, RaySamples
    from nerfstudio.field_components.encodings import NeRFEncoding
    from nerfstudio.field_components.field_heads import FieldHeadNames
    from nerfstudio.field_components.spatial_distortions import SceneContraction
    from nerfstudio.fields.vanilla_nerf_field import NeRFField
    from nerfstudio.model_components.ray_samplers import LinearDisparitySampler
    from nerfstudio.model_components.renderers import RGBRenderer

    def make(norm):
        pe = NeRFEncoding(in_dim=3, num_frequencies=10, min_freq_exp=0.0, max_freq_exp=9.0, include_input=True)
        de = NeRFEncoding(in_dim=3, num_frequencies=4, min_freq_exp=0.0, max_freq_exp=3.0, include_input=True)
        sd = None if norm == "none" else SceneContraction(order=float("inf") if norm == "linf" else None)
        return NeRFField(position_encoding=pe, direction_encoding=de, spatial_distortion=sd)

    f = make("linf")
    shapes = {k: list(v.shape) for k, v in f.state_dict().items()}
    params = seeded_params(shapes)
    o, d, fars, pts, pdirs, bg_t, rgb_fg = seeded_inputs()
    out = {"origins": o, "directions": d, "fars": fars, "points": pts, "point_directions": pdirs, "bg_transmittance": bg_t, "rgb_fg": rgb_fg}
    bundle = RayBundle(origins=o, directions=d, pixel_area=torch.ones(R, 1), camera_indices=torch.zeros(R, 1, dtype=torch.long),
                       nears=fars, fars=torch.ones_like(fars) * FAR_PLANE_BG)
    sampler = LinearDisparitySampler(num_samples=S).eval()
    rs = sampler(bundle)
    out["bins"] = torch.cat([rs.frustums.starts[..., 0], rs.frustums.ends[..., -1:, 0]], dim=-1)
    pfr = Frustums(origins=pts, directions=pdirs, starts=torch.zeros(NPTS, 1), ends=torch.zeros(NPTS, 1), pixel_area=torch.ones(NPTS, 1))
    prs = RaySamples(frustums=pfr, camera_indices=torch.zeros(NPTS, 1, dtype=torch.long))
    for norm in NORMS:
        f = make(norm).eval()
        f.load_state_dict(params)
        for tag, samples in (("ray", rs), ("pt", prs)):
            with torch.no_grad():
                pos = samples.frustums.get_positions()
                out[f"contracted_{norm}_{tag}"] = pos if f.spatial_distortion is None else f.spatial_distortion(pos)
                out[f"encoding_{norm}_{tag}"] = f.position_encoding(out[f"contracted_{norm}_{tag}"])
                density, emb = f.get_density(samples)
                fo = f(samples)
            out[f"density_{norm}_{tag}"], out[f"embedding_{norm}_{tag}"] = density, emb
            out[f"rgb_{norm}_{tag}"] = fo[FieldHeadNames.RGB]
            assert torch.equal(fo[FieldHeadNames.DENSITY], density)
        if norm == "linf":   # the background branch, base_surface_model.py:317-329, eval mode
            renderer = RGBRenderer(background_color=torch.tensor(BACKGROUND)).eval()
            with torch.no_grad():
                fo = f(rs)
                weights_bg = rs.get_weights(fo[FieldHeadNames.DENSITY])
                rgb_bg = renderer(rgb=fo[FieldHeadNames.RGB], weights=weights_bg)
            out["bg_weights"], out["bg_rgb_bg"], out["bg_rgb"] = weights_bg[..., 0], rgb_bg, rgb_fg + bg_t * rgb_bg
    np.savez_compressed(os.path.join(GOLDEN_DIR, "nerf_field.npz"), **{k: v.detach().cpu().numpy() for k, v in out.items()})
    meta = {"signature": signature(NeRFField.__init__), "encoding_signature": signature(NeRFEncoding.__init__), "state_dict": shapes,
            "rays": R, "samples": S, "points": NPTS, "far_plane_bg": FAR_PLANE_BG, "norms": NORMS, "background": BACKGROUND, "param_seed": 3}
    with open(os.path.join(GOLDEN_DIR, "nerf_field.json"), "w") as fh:
        json.dump(meta, fh, indent=1)
    print("wrote", GOLDEN_DIR, {k: tuple(v.shape) for k, v in out.items()})


if __name__ == "__main__":
    main()
