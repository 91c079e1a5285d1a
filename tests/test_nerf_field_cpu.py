"""CPU: the vanilla NeRF background field (background_model="mlp").  The oracle against the goldens minted from the unmodified reference
(oracle/make_golden_nerf_field.py), the drop-in's constructor signature and state dict, checkpoint loading, the ABI struct mirror and the
entry points' argument checks (they return error codes before any device work)."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import nerf_field as onf
from oracle.make_golden_nerf_field import BACKGROUND, default_repr, seeded_params, signature

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def golden():
    meta = json.load(open(os.path.join(GOLDEN, "nerf_field.json")))
    z = np.load(os.path.join(GOLDEN, "nerf_field.npz"))
    return meta, {k: torch.from_numpy(z[k]) for k in z.files}


def _params(meta):
    return seeded_params({k: tuple(v) for k, v in meta["state_dict"].items()}, meta["param_seed"])


def _close(a, b, tol):
    assert a.shape == b.shape, (a.shape, b.shape)
    err = float((a - b).abs().max()) if a.numel() else 0.0
    assert err <= tol, err


@pytest.mark.parametrize("norm", ["linf", "l2", "none"])
def test_oracle_matches_reference_field(golden, norm):
    meta, g = golden
    params = _params(meta)
    spec = onf.NerfSpec(contraction=None if norm == "none" else norm)
    bins = g["bins"]
    ray_pos = onf.midpoints(g["origins"][:, None], g["directions"][:, None], bins[:, :-1, None], bins[:, 1:, None])
    R, S = bins.shape[0], bins.shape[1] - 1
    for tag, pos, dirs in (("ray", ray_pos, g["directions"][:, None].expand(R, S, 3)), ("pt", g["points"], g["point_directions"])):
        o = onf.field(pos, dirs, params, spec)
        assert torch.equal(o["contracted"], g[f"contracted_{norm}_{tag}"])
        assert torch.equal(o["encoding"], g[f"encoding_{norm}_{tag}"])
        _close(o["density"], g[f"density_{norm}_{tag}"], 2e-6)
        _close(o["embedding"], g[f"embedding_{norm}_{tag}"], 2e-6)
        _close(o["rgb"], g[f"rgb_{norm}_{tag}"], 2e-6)


def test_oracle_matches_reference_background_branch(golden):
    meta, g = golden
    out = onf.background_branch(g["origins"], g["directions"], g["fars"], g["bg_transmittance"], g["rgb_fg"], _params(meta), onf.NerfSpec(),
                                torch.tensor(BACKGROUND), meta["samples"], meta["far_plane_bg"])
    assert torch.equal(out["bins"], g["bins"])
    _close(out["weights"], g["bg_weights"], 2e-6)
    _close(out["rgb_bg"], g["bg_rgb_bg"], 2e-6)
    _close(out["rgb"], g["bg_rgb"], 2e-6)


def test_signatures_and_state_dict_match_reference(golden):
    import sdfstudio_b200 as sb

    meta, _ = golden
    sig = signature(sb.NeRFField.__init__)
    assert sig[-1] == ["precision", "bf16x3"]              # the package's one keyword-only knob
    assert sig[:-1] == meta["signature"]
    assert signature(sb.NeRFEncoding.__init__) == meta["encoding_signature"]
    f = _surface_model_field(sb)
    assert {k: list(v.shape) for k, v in f.state_dict().items()} == meta["state_dict"]
    assert list(f.state_dict()) == list(meta["state_dict"])
    assert default_repr(sb.NeRFField.__init__.__defaults__[0]) == "Identity"


def _surface_model_field(sb, **kw):
    pe = sb.NeRFEncoding(in_dim=3, num_frequencies=10, min_freq_exp=0.0, max_freq_exp=9.0, include_input=True)
    de = sb.NeRFEncoding(in_dim=3, num_frequencies=4, min_freq_exp=0.0, max_freq_exp=3.0, include_input=True)
    return sb.NeRFField(position_encoding=pe, direction_encoding=de, spatial_distortion=sb.SceneContraction(order=float("inf")), **kw)


def test_reference_state_dict_and_checkpoint_load(golden):
    import sdfstudio_b200 as sb
    from sdfstudio_b200.checkpoint import BACKGROUND_PREFIX, load_background_field_checkpoint

    meta, _ = golden
    params = _params(meta)
    f = _surface_model_field(sb)
    f.load_state_dict(params)
    for k, v in f.state_dict().items():
        assert torch.equal(v, params[k])
    # a DDP-wrapped pipeline checkpoint, with the SDF field's entries next to it and fp16-stored tensors
    ckpt = {"step": 7, "pipeline": {**{"module." + BACKGROUND_PREFIX + k: v.half() for k, v in params.items()}, "module._model.field.glin0.bias": torch.zeros(3)}}
    g = _surface_model_field(sb)
    missing, unexpected = load_background_field_checkpoint(g, ckpt)
    assert missing == [] and unexpected == []
    for k, v in g.state_dict().items():
        assert torch.equal(v, params[k].half().float())
    bad = {BACKGROUND_PREFIX + k: v for k, v in params.items() if not k.startswith("field_heads")}
    with pytest.raises(RuntimeError):
        load_background_field_checkpoint(_surface_model_field(sb), bad)


def test_unsupported_options_raise():
    import sdfstudio_b200 as sb

    with pytest.raises(NotImplementedError):
        sb.NeRFField(use_integrated_encoding=True)
    with pytest.raises(NotImplementedError):
        sb.NeRFField(field_heads=())
    f = sb.NeRFField()
    with pytest.raises(NotImplementedError):
        f(None, compute_normals=True)
    with pytest.raises(RuntimeError):                      # no CPU path
        f.density_fn(torch.zeros(4, 3))


def test_struct_size_and_family_predicate():
    import sdfstudio_b200 as sb
    from sdfstudio_b200 import _lib

    lib = _lib.load()
    assert lib.sdfb200_struct_size(8) == C.sizeof(_lib.NerfFieldDesc)
    f = _surface_model_field(sb)
    assert lib.sdfb200_nerf_field_in_family(f._desc()) == 1
    assert lib.sdfb200_nerf_field_packed_bytes(f._desc()) > 0
    assert f.eval()._engine() == "kernel"
    with torch.no_grad():
        assert f.train()._engine() == "kernel"
    assert f.train()._engine() == "compose"
    for kw in ({"head_mlp_layer_width": 64}, {"skip_connections": (3,)}, {"base_mlp_num_layers": 6}):
        g = _surface_model_field(sb, **kw).eval()
        assert lib.sdfb200_nerf_field_in_family(g._desc()) == 0 and g._engine() == "compose", kw
    assert _surface_model_field(sb, precision="fp32").eval()._engine() == "aten"
    d = f._desc()
    d.precision = _lib.PRECISION["fp32"]
    assert lib.sdfb200_nerf_field_in_family(d) == 0
    d = f._desc()
    d.pe_frequencies = 11
    assert lib.sdfb200_nerf_field_in_family(d) == 0
    assert lib.sdfb200_nerf_field_in_family(None) == 0


def test_entry_points_return_error_codes():
    import sdfstudio_b200 as sb
    from sdfstudio_b200 import _lib

    lib = _lib.load()
    f = _surface_model_field(sb)
    d = f._desc(32)
    assert lib.sdfb200_nerf_field_packed_bytes(None) == 0
    assert lib.sdfb200_nerf_field_pack(None, None, None, None, None) == -1
    assert lib.sdfb200_nerf_field_pack(d, None, None, None, None) == -1
    null12 = (C.c_void_p * 12)()
    assert lib.sdfb200_nerf_field_pack(d, null12, null12, 1024, None) == -1
    assert lib.sdfb200_nerf_field_forward(None, None, None, None, None, 4, None, None, None) == -1
    assert lib.sdfb200_nerf_field_forward(d, None, None, None, None, 4, None, None, None) == -1
    assert lib.sdfb200_nerf_field_forward(d, None, None, None, None, -1, None, None, None) == -1
    assert lib.sdfb200_nerf_field_forward(d, None, None, None, None, 0, None, None, None) == 0      # nothing to do
    assert lib.sdfb200_nerf_field_forward(d, 1024, 1024, 1024, None, 4, 1024, 1024, None) == -1   # ray mode without bins
    out = f._desc(32)
    out.head_width = 64
    assert lib.sdfb200_nerf_field_forward(out, 1024, 1024, 1024, 1024, 4, 1024, 1024, None) == -3
    assert lib.sdfb200_nerf_field_pack(out, null12, null12, 1024, None) == -3
    assert lib.sdfb200_nerf_field_packed_bytes(out) == 0
