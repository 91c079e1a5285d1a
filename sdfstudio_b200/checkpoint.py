"""Loading existing sdfstudio checkpoints into the drop-in modules (SURVEY.md section 8f row 4): the SDF field, the proposal networks
and the grid and mlp background fields.

A reference ``step-*.ckpt`` (engine/trainer.py:276-297) is ``{"step", "pipeline", "optimizers", "schedulers", "scalers"}`` where
``pipeline`` is ``Pipeline.state_dict()``: the field's tensors sit under ``_model.field.`` (``module.`` in front when the pipeline
was DDP-wrapped, pipelines/base_pipeline.py:426-439).  SDFField keeps the reference's parameter names and shapes
(tests/test_abi_cpu.py::test_state_dict_names_match_reference), so loading is a prefix strip plus the hash-grid entry:

* ``encoding.params`` -- tiny-cuda-nn's single flat parameter vector (fp32 master copy; older builds store fp16): loaded into
  ``Encoding(layout="tcnn").params`` (same level order / per-level sizes, encoding.py ``make_grid_desc``), cast to fp32.
* ``encoding.hash_table`` -- the reference's own torch ``HashEncoding`` ([L*T, F]): loaded into ``layout="torch"``.
"""
from typing import Dict, Tuple

import torch

from .nerf_field import NeRFField

FIELD_PREFIX = "_model.field."


def extract_state(loaded_state: Dict, prefix: str = FIELD_PREFIX) -> Dict[str, torch.Tensor]:
    """checkpoint dict (or its ``pipeline`` entry, or an already flat state_dict) -> tensors under `prefix`, prefix removed."""
    state = loaded_state.get("pipeline", loaded_state) if isinstance(loaded_state, dict) else loaded_state
    state = {(k[len("module."):] if k.startswith("module.") else k): v for k, v in state.items()}
    sub = {k[len(prefix):]: v for k, v in state.items() if k.startswith(prefix)}
    return sub if sub else dict(state)


def load_field_checkpoint(field, loaded_state, prefix: str = FIELD_PREFIX, strict: bool = True) -> Tuple[list, list]:
    """Load a reference checkpoint (path, checkpoint dict or state_dict) into a ``sdfstudio_b200.SDFField``.
    Returns (missing, unexpected) like ``load_state_dict``; with ``strict`` any mismatch other than the read-only ``aabb`` raises."""
    if isinstance(loaded_state, (str, bytes)) or hasattr(loaded_state, "__fspath__"):
        loaded_state = torch.load(loaded_state, map_location="cpu")
    sd = extract_state(loaded_state, prefix)
    enc = field.encoding
    if "encoding.params" in sd:
        if enc.layout != "tcnn":
            raise ValueError("the checkpoint holds a tiny-cuda-nn grid (`encoding.params`); build the field with grid_layout='tcnn'")
        flat = sd["encoding.params"].reshape(-1).to(torch.float32)
        if flat.numel() != enc.params.numel():
            raise ValueError(f"encoding.params has {flat.numel()} entries, this grid configuration needs {enc.params.numel()} "
                             "(check num_levels / log2_hashmap_size / base_res / max_res / hash_features_per_level)")
        sd["encoding.params"] = flat
    if "encoding.hash_table" in sd and enc.layout != "torch":
        raise ValueError("the checkpoint holds a torch HashEncoding table (`encoding.hash_table`); build the field with grid_layout='torch'")
    sd = {k: (v.to(torch.float32) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in sd.items()}
    missing, unexpected = field.load_state_dict(sd, strict=False)
    missing = [m for m in missing if m != "aabb"]
    if strict and (missing or unexpected):
        raise RuntimeError(f"checkpoint does not match the field: missing {missing}, unexpected {list(unexpected)}")
    return missing, list(unexpected)


def load_flat_params(flats: Dict[str, Tuple[torch.nn.Parameter, torch.Tensor]], owner: str, knobs: Dict[str, str]) -> None:
    """Copy tiny-cuda-nn flat ``params`` vectors (fp16-stored ones cast to fp32) into their parameters: `flats` maps a name to
    (parameter, vector).  Every length is checked before anything is copied; a mismatch names the constructor arguments to check."""
    for key, (p, v) in flats.items():
        if v.numel() != p.numel():
            raise ValueError(f"{key} has {v.numel()} entries, {owner} needs {p.numel()} (check {knobs[key]})")
    with torch.no_grad():
        for p, v in flats.values():
            p.copy_(v.reshape(-1).to(device=p.device, dtype=torch.float32))


def load_density_field_checkpoint(density_field, loaded_state, index: int = 0, strict: bool = True):
    """Load ``_model.proposal_networks.{index}.mlp_base.params`` (tiny-cuda-nn ``NetworkWithInputEncoding``: FullyFusedMLP weights then the
    HashGrid table, nerfstudio/fields/density_fields.py:89-96) of a reference neus-facto / bakedsdf checkpoint into a
    ``sdfstudio_b200.HashMLPDensityField``.  The vector length is checked (the output layer is stored 16 rows wide like tcnn pads it); the
    ordering inside the vector follows tcnn's published layout (UNPINNED: tcnn is not vendored in the reference)."""
    if isinstance(loaded_state, (str, bytes)) or hasattr(loaded_state, "__fspath__"):
        loaded_state = torch.load(loaded_state, map_location="cpu")
    sd = extract_state(loaded_state, f"_model.proposal_networks.{index}.")
    key = "mlp_base.params"
    if key not in sd:
        raise KeyError(f"{key} not found under _model.proposal_networks.{index}.")
    load_flat_params({key: (density_field.mlp_base.params, sd[key])}, "this proposal network",
                     {key: "num_levels / log2_hashmap_size / max_res / hidden_dim / num_layers"})
    extra = [k for k in sd if k not in (key, "aabb")]
    if strict and extra:
        raise RuntimeError(f"unexpected entries for the proposal network: {extra}")
    return [], extra


BACKGROUND_PREFIX = "_model.field_background."
_FLAT_KNOBS = {"mlp_base.params": "num_levels / log2_hashmap_size / max_res / hidden_dim / num_layers / geo_feat_dim",
               "mlp_head.params": "hidden_dim_color / num_layers_color / geo_feat_dim / appearance_embedding_dim"}
_EMPTY_PARAMS = ("direction_encoding.params", "position_encoding.params")


def load_background_field_checkpoint(field, loaded_state, prefix: str = BACKGROUND_PREFIX, strict: bool = True) -> Tuple[list, list]:
    """Load the background field of a reference checkpoint.  ``background_model="mlp"`` (``NeRFField``, vanilla_nerf_field.py:52-89):
    the entries keep the reference's names and shapes, so this is ``load_state_dict`` after the prefix strip.
    ``background_model="grid"`` (neus-facto-angelo / bakedangelo, ``TCNNNerfactoField``, nerfstudio/fields/nerfacto_field.py:86-221) into
    a ``sdfstudio_b200.TCNNNerfactoField``: ``mlp_base.params`` / ``mlp_head.params``
    are tiny-cuda-nn's flat vectors (fp16-stored ones are cast to fp32); their lengths are checked, the ordering inside them follows
    tcnn's published layout (UNPINNED).  The zero-length ``params`` of the parameter-free encodings may be present or absent.
    Returns (missing, unexpected); with ``strict`` any other mismatch raises."""
    if isinstance(loaded_state, (str, bytes)) or hasattr(loaded_state, "__fspath__"):
        loaded_state = torch.load(loaded_state, map_location="cpu")
    sd = extract_state(loaded_state, prefix)
    sd = {k: (v.to(torch.float32) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in sd.items()}
    if isinstance(field, NeRFField):
        missing, unexpected = field.load_state_dict(sd, strict=False)
        if strict and (missing or unexpected):
            raise RuntimeError(f"checkpoint does not match the background field: missing {list(missing)}, unexpected {list(unexpected)}")
        return list(missing), list(unexpected)
    for key in _FLAT_KNOBS:
        if key not in sd:
            raise KeyError(f"{key} not found under {prefix}")
    for key in _EMPTY_PARAMS:
        v = sd.pop(key, None)
        if v is not None and v.numel() != 0:
            raise ValueError(f"{key} has {v.numel()} entries, the parameter-free encoding has none")
    load_flat_params({key: (field.get_parameter(key), sd.pop(key)) for key in _FLAT_KNOBS}, "this background field", _FLAT_KNOBS)
    missing, unexpected = field.load_state_dict(sd, strict=False)
    missing = [m for m in missing if m not in _FLAT_KNOBS and m not in _EMPTY_PARAMS and m != "aabb"]
    if strict and (missing or unexpected):
        raise RuntimeError(f"checkpoint does not match the background field: missing {missing}, unexpected {list(unexpected)}")
    return missing, list(unexpected)
