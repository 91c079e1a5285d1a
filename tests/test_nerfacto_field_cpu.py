"""CPU: the nerfacto background field's oracle against the golden minted from the unmodified reference (oracle/make_golden_nerfacto.py),
the drop-in's constructor / state dict / parameter counts against the reference's, and the background checkpoint loader."""
import inspect
import json
import os

import pytest
import torch

from oracle import nerfacto as onf

from helpers import GOLDEN_DIR, load_golden

G = load_golden("nerfacto_field")
META = json.load(open(os.path.join(GOLDEN_DIR, "nerfacto_field.json")))
R, S = META["rays"], META["samples"]
SPEC = onf.NerfactoSpec(hidden_dim=META["case"]["hidden_dim"], hidden_dim_color=META["case"]["hidden_dim_color"],
                        log2_hashmap_size=META["case"]["log2_hashmap_size"])


def _samples():
    o, d, b = G["origins"], G["directions"], G["bins"]
    pos = onf.midpoints(o[:, None], d[:, None], b[:, :-1, None], b[:, 1:, None]).reshape(-1, 3)
    return pos, d[:, None].expand(R, S, 3).reshape(-1, 3)


def _appearance(mode):
    emb = G["embedding"]
    if mode == "train":
        return emb[G["camera_indices"]][:, None].expand(R, S, -1).reshape(-1, emb.shape[1])
    if mode == "eval_mean":
        return emb.mean(0).expand(R * S, -1)
    return torch.zeros(R * S, emb.shape[1])


@pytest.mark.parametrize("norm,mode", [tuple(r) for r in META["runs"]])
def test_oracle_matches_reference(norm, mode):
    pos, dirs = _samples()
    aabb, contraction = (G["aabb"], None) if norm == "aabb" else (None, norm)
    out = onf.field(pos, dirs, _appearance(mode), G["base_params"], G["head_params"], SPEC, aabb=aabb, contraction=contraction)
    # the normalised positions the reference handed to mlp_base, bit for bit: hence the same grid cells at every level
    x01 = G[f"x01_{norm}"].reshape(-1, 3)
    assert torch.equal(out["x01"], x01)
    assert float((out["rgb"] - G[f"rgb_{norm}_{mode}"].reshape(-1, 3)).abs().max()) <= 2e-6
    if mode == "train":
        assert float(((out["density"] - G[f"density_{norm}"].reshape(-1)).abs() / G[f"density_{norm}"].reshape(-1).abs().clamp_min(1)).max()) <= 2e-6
        assert float((out["pre"] - G[f"pre_{norm}"].reshape(-1)).abs().max()) <= 2e-6
    if norm == "linf" and mode == "train":
        assert float((out["geo"] - G["geo_linf"].reshape(-1, SPEC.geo_feat_dim)).abs().max()) <= 2e-6


def test_golden_outputs_vary():
    """the golden case exercises every part of the composition (nothing saturated or constant)"""
    assert float(G["density_linf"].std()) > 0.01 and float(G["rgb_linf_train"].std()) > 0.01
    assert not torch.allclose(G["rgb_linf_train"], G["rgb_linf_eval_zeros"]) and not torch.allclose(G["rgb_linf_eval_mean"], G["rgb_linf_eval_zeros"])
    assert not torch.allclose(G["density_linf"], G["density_l2"]) and not torch.allclose(G["density_linf"], G["density_aabb"])


def _default_field(**kw):
    import sdfstudio_b200 as sb

    return sb.TCNNNerfactoField(torch.tensor([[-3.0, -3, -3], [3, 3, 3]]), num_images=META["case"]["num_images"], **kw)


def test_signature_state_dict_and_parameter_counts_match_reference():
    import sdfstudio_b200 as sb

    sig = [[n, None if p.default is inspect.Parameter.empty else p.default] for n, p in inspect.signature(sb.TCNNNerfactoField.__init__).parameters.items()
           if n != "self"]
    assert sig == META["signature"]
    sd = _default_field().state_dict()
    assert {k: list(v.shape) for k, v in sd.items() if not k.endswith(".params")} == META["state_dict"]
    assert {k: v.numel() for k, v in sd.items() if k.endswith(".params")} == META["tcnn_params"]
    assert [k for k in sd if not k.endswith(".params")] == list(META["state_dict"])


def test_unsupported_options_raise():
    for kw in ({"use_transient_embedding": True}, {"use_semantics": True}, {"use_pred_normals": True}, {"hidden_dim": 128}, {"hidden_dim_color": 8},
               {"num_layers": 5}, {"num_layers_color": 1}, {"geo_feat_dim": 16}, {"geo_feat_dim": -1}, {"appearance_embedding_dim": 40},
               {"appearance_embedding_dim": -1}):
        with pytest.raises(NotImplementedError):
            _default_field(**kw)


def _small(**kw):
    import sdfstudio_b200 as sb

    return sb.TCNNNerfactoField(torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), num_images=7, hidden_dim=16, hidden_dim_color=32, log2_hashmap_size=10,
                                num_levels=8, **kw)


def _reference_shaped_state(src, prefix="_model.field_background.", dtype=torch.float32, with_encodings=True):
    """what a reference checkpoint holds for this field (pipeline state under `prefix`, tcnn params flat)."""
    sd = {prefix + k: v.clone() for k, v in src.state_dict().items()}
    for k in ("mlp_base.params", "mlp_head.params"):
        sd[prefix + k] = sd[prefix + k].to(dtype)
    if not with_encodings:
        for k in ("direction_encoding.params", "position_encoding.params"):
            del sd[prefix + k]
    sd["_model.field.glin0.bias"] = torch.zeros(3)   # other modules of the model are ignored
    return sd


@pytest.mark.parametrize("variant", ["plain", "module_prefix", "fp16", "no_encoding_params"])
def test_background_checkpoint_loader(variant):
    from sdfstudio_b200 import checkpoint

    src = _small()
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for p in (src.mlp_base.params, src.mlp_head.params, src.embedding_appearance.embedding.weight):
            p.copy_(torch.randn(p.shape, generator=g))
    prefix = "module._model.field_background." if variant == "module_prefix" else "_model.field_background."
    dtype = torch.float16 if variant == "fp16" else torch.float32
    ckpt = {"step": 1, "pipeline": _reference_shaped_state(src, prefix, dtype, variant != "no_encoding_params")}
    dst = _small()
    missing, unexpected = checkpoint.load_background_field_checkpoint(dst, ckpt)
    assert missing == [] and unexpected == []
    for name in ("mlp_base.params", "mlp_head.params", "embedding_appearance.embedding.weight"):
        want = src.get_parameter(name).detach()
        if variant == "fp16" and name != "embedding_appearance.embedding.weight":
            want = want.half().float()
        assert torch.equal(dst.get_parameter(name).detach(), want), name
    assert dst.mlp_base.params.dtype == torch.float32


def test_background_checkpoint_loader_rejects_mismatches():
    from sdfstudio_b200 import checkpoint

    ckpt = {"pipeline": _reference_shaped_state(_small())}
    with pytest.raises(ValueError, match="num_levels"):
        checkpoint.load_background_field_checkpoint(_small(num_layers=3), ckpt)
    with pytest.raises(ValueError, match="hidden_dim_color"):
        checkpoint.load_background_field_checkpoint(_small(num_layers_color=2), ckpt)
    bad = dict(ckpt["pipeline"])
    bad["_model.field_background.direction_encoding.params"] = torch.zeros(4)
    with pytest.raises(ValueError, match="parameter-free"):
        checkpoint.load_background_field_checkpoint(_small(), {"pipeline": bad})
    extra = dict(ckpt["pipeline"])
    extra["_model.field_background.mlp_transient.params"] = torch.zeros(4)
    with pytest.raises(RuntimeError, match="unexpected"):
        checkpoint.load_background_field_checkpoint(_small(), {"pipeline": extra})
    missing, unexpected = checkpoint.load_background_field_checkpoint(_small(), {"pipeline": extra}, strict=False)
    assert unexpected == ["mlp_transient.params"]
    del extra["_model.field_background.mlp_head.params"]
    with pytest.raises(KeyError):
        checkpoint.load_background_field_checkpoint(_small(), {"pipeline": extra})


def test_oracle_mlp_walk_equals_proposal_oracle():
    """oracle.nerfacto's FullyFusedMLP walk (several output rows) and oracle.density's (one output) are the same network: with
    geo_feat_dim = 0 the nerfacto density equals the proposal-network oracle on the same flat parameters"""
    from oracle import density as odensity

    spec = onf.NerfactoSpec(num_levels=8, max_res=128, log2_hashmap_size=10, hidden_dim=32, num_layers=3, geo_feat_dim=0)
    g = torch.Generator().manual_seed(4)
    n_net = spec.n_base_net()
    params = torch.cat([torch.randn(n_net, generator=g, dtype=torch.float64) * 0.3,
                        torch.rand(spec.meta()["total"] * 2, generator=g, dtype=torch.float64) * 2 - 1])
    pos = (torch.rand(300, 3, generator=g, dtype=torch.float64) * 2 - 1) * 3
    dens, pre, geo = onf.density(onf.normalize(pos, contraction="linf"), params, spec)
    d_ref, pre_ref = odensity.density_field(pos, params[:n_net], params[n_net:], 32, 2, 8, 2, 10, 16, spec.growth, contraction="linf")
    assert geo.shape == (300, 0)
    assert torch.allclose(pre, pre_ref[:, 0], rtol=1e-12, atol=1e-12) and torch.allclose(dens, d_ref[:, 0], rtol=1e-12, atol=1e-12)


def test_abi_misuse_is_refused_before_any_launch():
    """argument errors are returned by the library without touching the (here fake) device pointers and without a launch: ray mode needs
    directions for its midpoints even when rgb is not wanted; rgb needs head weights and directions"""
    from sdfstudio_b200 import _lib

    lib = _lib.load()
    f = _small()
    n0 = lib.sdfb200_launch_count()
    fake = 0x1000

    def call(n_samples, directions, rgb, head=fake, bins=fake):
        return lib.sdfb200_nerfacto_field_forward(f.mlp_base.desc, f._desc(n_samples), fake, fake, head, None, fake, directions, bins, 4, None, 0,
                                                  fake, rgb, None, None, None)

    assert call(48, None, None) == -1 and b"directions" in lib.sdfb200_last_error_string()
    assert call(48, fake, None, bins=None) == -1
    assert call(0, None, fake) == -1 and call(0, fake, fake, head=None) == -1
    d = f._desc(0)
    d.hidden_dim = 48
    assert lib.sdfb200_nerfacto_field_forward(f.mlp_base.desc, d, fake, fake, fake, None, fake, fake, None, 4, None, 0, fake, fake, None, None,
                                              None) == -3
    assert lib.sdfb200_launch_count() == n0
