"""TEST INFRASTRUCTURE -- mints tests/golden/nerfacto_field.npz + nerfacto_field.json from the UNMODIFIED reference TCNNNerfactoField
(nerfstudio/fields/nerfacto_field.py:67-318) run on CPU (build container only):

* the constructor signature, the state-dict names / shapes of the default field and the flat tcnn parameter counts;
* for a seeded case (8 rays x 48 samples, 5 images, small grid): density, pre-activation, geometry feature, rgb and the normalised positions
  the reference handed to ``mlp_base``, in train mode with camera indices, eval with zeros and eval with the mean embedding, under the
  L-inf and L2 SceneContraction and the aabb normalisation.

This pins the reference's own composition around tiny-cuda-nn (normalisation, the [1, geo] split, trunc_exp, direction normalisation,
concat order, appearance modes, sigmoid).  tiny-cuda-nn is not vendored: its ``NetworkWithInputEncoding``, ``Network`` and
``Encoding("SphericalHarmonics" | "Frequency")`` are stood in for by oracle/nerfacto.py's restatements, patched into the reference module
only (the stand-in installed by ref_import.py is left as it is).

    python -m oracle.make_golden_nerfacto
"""
import inspect
import json
import os
import types
import warnings

import numpy as np
import torch
from torch import nn

from . import hashgrid, nerfacto, ref_import

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
CASE = {"num_images": 5, "hidden_dim": 16, "hidden_dim_color": 16, "log2_hashmap_size": 6}
R, S = 8, 48
AABB = [[-3.0, -3.0, -3.0], [3.0, 3.0, 3.0]]
RUNS = [("linf", "train"), ("l2", "train"), ("aabb", "train"), ("linf", "eval_zeros"), ("linf", "eval_mean")]


def _pad16(n):
    return (n + 15) // 16 * 16


def _net_size(n_in, n_out, cfg):
    H, n_hidden = cfg["n_neurons"], cfg["n_hidden_layers"]
    return H * _pad16(n_in) + (n_hidden - 1) * H * H + _pad16(n_out) * H


def tcnn_standin(seen):
    """tinycudann look-alike built from oracle/nerfacto.py (fp32; tcnn itself computes in fp16).  `seen` collects mlp_base's inputs."""

    class NetworkWithInputEncoding(nn.Module):
        def __init__(self, n_input_dims, n_output_dims, encoding_config, network_config, seed=1337):
            super().__init__()
            enc = encoding_config
            self.F, self.n_out, self.cfg = enc["n_features_per_level"], n_output_dims, network_config
            self.meta = hashgrid.tcnn_grid_meta(enc["n_levels"], self.F, enc["log2_hashmap_size"], enc["base_resolution"], enc["per_level_scale"])
            self.in_dim = enc["n_levels"] * self.F
            self.n_net = _net_size(self.in_dim, n_output_dims, network_config)
            self.params = nn.Parameter(torch.zeros(self.n_net + self.meta["total"] * self.F))
            self.n_output_dims = n_output_dims

        def forward(self, x):
            seen.append(x.detach().clone())
            feat = hashgrid.encode_tcnn_layout(x, self.params[self.n_net:].view(-1, self.F), self.meta, self.F, False)
            return nerfacto.mlp(feat, self.params[: self.n_net], self.in_dim, self.cfg["n_neurons"], self.cfg["n_hidden_layers"], self.n_out)

    class Network(nn.Module):
        def __init__(self, n_input_dims, n_output_dims, network_config, seed=1337):
            super().__init__()
            self.in_dim, self.n_out, self.cfg = n_input_dims, n_output_dims, network_config
            self.params = nn.Parameter(torch.zeros(_net_size(n_input_dims, n_output_dims, network_config)))
            self.n_output_dims = n_output_dims

        def forward(self, x):
            out = nerfacto.mlp(x, self.params, self.in_dim, self.cfg["n_neurons"], self.cfg["n_hidden_layers"], self.n_out)
            assert self.cfg["output_activation"] == "Sigmoid"
            return torch.sigmoid(out)

    class Encoding(nn.Module):
        def __init__(self, n_input_dims, encoding_config, seed=1337):
            super().__init__()
            self.otype = encoding_config["otype"]
            if self.otype == "SphericalHarmonics":
                assert encoding_config["degree"] == 4
                self.n_output_dims = 16
            elif self.otype == "Frequency":
                self.n_output_dims = n_input_dims * 2 * encoding_config["n_frequencies"]
            else:
                raise NotImplementedError(self.otype)
            self.params = nn.Parameter(torch.zeros(0))

        def forward(self, x):
            if self.otype != "SphericalHarmonics":
                raise NotImplementedError("the Frequency encoding is only used by predicted normals")
            return nerfacto.sh4_tcnn(x * 2 - 1)

    return types.SimpleNamespace(NetworkWithInputEncoding=NetworkWithInputEncoding, Network=Network, Encoding=Encoding)


def seeded_inputs(seed=0):
    """8 rays from cameras at distance 2-2.8 looking through the unit sphere, 48 sorted euclidean bins in [0.2, 8] per ray (most samples
    land outside the unit sphere, where the background field is used)."""
    g = torch.Generator().manual_seed(seed)
    o = torch.randn(R, 3, generator=g)
    o = o / o.norm(dim=-1, keepdim=True) * (2.0 + 0.8 * torch.rand(R, 1, generator=g))
    d = -o + 0.6 * torch.randn(R, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True)
    bins = torch.sort(0.2 + 7.8 * torch.rand(R, S + 1, generator=g), dim=-1).values
    cam = torch.randint(0, CASE["num_images"], (R,), generator=g)
    return o, d, bins, cam


def seeded_params(field, seed=1):
    """Parameters with enough spread that every output varies (the tcnn initialisation leaves the grid at +-1e-4)."""
    g = torch.Generator().manual_seed(seed)
    nb = field.mlp_base
    with torch.no_grad():
        nb.params[: nb.n_net] = torch.randn(nb.n_net, generator=g) * 0.4
        nb.params[nb.n_net:] = torch.rand(nb.params.numel() - nb.n_net, generator=g) * 2 - 1
        field.mlp_head.params.copy_(torch.randn(field.mlp_head.params.numel(), generator=g) * 0.3)
        field.embedding_appearance.embedding.weight.copy_(torch.randn(CASE["num_images"], 32, generator=g) * 0.5)


def main():
    ref_import.install_shims()
    warnings.simplefilter("ignore")
    import nerfstudio.fields.nerfacto_field as nf
    from nerfstudio.cameras.rays import Frustums, RaySamples
    from nerfstudio.field_components.field_heads import FieldHeadNames
    from nerfstudio.field_components.spatial_distortions import SceneContraction

    seen = []
    nf.tcnn = tcnn_standin(seen)
    sig = [[n, None if p.default is inspect.Parameter.empty else p.default] for n, p in inspect.signature(nf.TCNNNerfactoField.__init__).parameters.items()
           if n != "self"]
    default = nf.TCNNNerfactoField(torch.tensor(AABB), num_images=CASE["num_images"])
    sd = default.state_dict()
    tcnn_keys = [k for k in sd if k.endswith(".params")]
    spec = {k: list(v.shape) for k, v in sd.items() if k not in tcnn_keys}
    counts = {k: int(sd[k].numel()) for k in tcnn_keys}
    del default, sd

    o, d, bins, cam = seeded_inputs()
    out = {"origins": o, "directions": d, "bins": bins, "camera_indices": cam, "aabb": torch.tensor(AABB)}
    frustums = Frustums(origins=o[:, None].expand(R, S, 3), directions=d[:, None].expand(R, S, 3), starts=bins[:, :-1, None], ends=bins[:, 1:, None],
                        pixel_area=torch.ones(R, S, 1))
    rs = RaySamples(frustums=frustums, camera_indices=cam[:, None, None].expand(R, S, 1))
    fields = {}
    for norm, mode in RUNS:
        key = (norm, mode == "eval_mean")
        if key not in fields:
            distortion = None if norm == "aabb" else SceneContraction(order=float("inf") if norm == "linf" else None)
            f = nf.TCNNNerfactoField(torch.tensor(AABB), spatial_distortion=distortion, use_average_appearance_embedding=mode == "eval_mean", **CASE)
            seeded_params(f)
            fields[key] = f
        f = fields[key]
        f.train(mode == "train")
        seen.clear()
        with torch.no_grad():
            fo = f(rs)
        tag = f"{norm}_{mode}"
        out[f"rgb_{tag}"] = fo[FieldHeadNames.RGB]
        if mode == "train":
            out[f"density_{norm}"] = fo[FieldHeadNames.DENSITY][..., 0]
            out[f"pre_{norm}"] = f._density_before_activation[..., 0]
            out[f"x01_{norm}"] = seen[0].view(R, S, 3)
        if tag == "linf_train":
            out["base_params"], out["head_params"] = f.mlp_base.params.detach().clone(), f.mlp_head.params.detach().clone()
            out["embedding"] = f.embedding_appearance.embedding.weight.detach().clone()
            with torch.no_grad():
                out["geo_linf"] = f.get_density(rs)[1]
    np.savez_compressed(os.path.join(GOLDEN_DIR, "nerfacto_field.npz"), **{k: v.detach().cpu().numpy() for k, v in out.items()})
    meta = {"signature": sig, "state_dict": spec, "tcnn_params": counts, "case": CASE, "rays": R, "samples": S, "runs": RUNS}
    with open(os.path.join(GOLDEN_DIR, "nerfacto_field.json"), "w") as fh:
        json.dump(meta, fh, indent=1)
    print("wrote", GOLDEN_DIR, {k: tuple(v.shape) for k, v in out.items()}, counts)


if __name__ == "__main__":
    main()
