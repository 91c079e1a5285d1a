"""CPU: the torch restatement of the reference's texture export (oracle/texture.py) against the golden minted from the unmodified
reference (oracle/make_golden_texture.py), and the host side of sdfstudio_b200/texturing.py: the OBJ / MTL / PNG writers, the PLY reader
and the argument checks."""
import importlib.util
import json
import os
import struct
import zlib

import numpy as np
import pytest
import torch

from oracle import texture as otex

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def golden():
    z = np.load(os.path.join(GOLDEN, "texture.npz"))
    meta = json.load(open(os.path.join(GOLDEN, "texture.json")))
    return z, meta["cases"]


GOLDEN_CASES = sorted(golden()[1])


def case_inputs(name):
    z, cases = golden()
    g = lambda k: torch.from_numpy(z[f"{name}/{k}"])  # noqa: E731
    return g("vertices"), g("faces"), g("normals"), (g("uvs") if f"{name}/uvs" in z else None), cases[name]["kwargs"]


def oracle_texels(name, device="cpu"):
    """(texture_coordinates, face, bary, (H, W)) of a golden case by the oracle."""
    vertices, faces, normals, uvs, kw = case_inputs(name)
    if kw.get("unwrap_method") == "custom":
        return otex.grid_unwrap(len(faces), kw["px_per_uv_triangle"], device)
    n = kw["num_pixels_per_side"]
    face, bary = otex.rasterize(uvs.to(device), n, 10)
    return uvs.to(device), face, bary, (n, n)


def oracle_bundle(name):
    vertices, faces, normals, _, kw = case_inputs(name)
    tc, face, bary, hw = oracle_texels(name)
    o, d = otex.texel_rays(vertices, faces, normals, face, bary)
    raylen = otex.ray_length(vertices, faces, kw.get("raylen_method", "edge"))
    return tc, otex.texel_bundle(o.view(*hw, 3), d.view(*hw, 3), raylen)


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_oracle_matches_reference(name):
    """Every field of the texel ray bundle the reference hands the model is reproduced bit for bit."""
    z, _ = golden()
    _, bundle = oracle_bundle(name)
    for k, v in bundle.items():
        ref = z[f"{name}/{k}"]
        assert v.shape == ref.shape, (k, v.shape, ref.shape)
        assert np.array_equal(v.numpy(), ref, equal_nan=True), (k, np.abs(v.numpy() - ref).max())


def test_golden_cases_reach_the_search_rules():
    """The golden covers what the search's rules decide: the chunk-tail faces that take no part, texels no chunk claims (face 0, weights
    0), the tie between identical triangles and the NaN of a zero-area triangle."""
    _, face, bary, _ = oracle_texels("xatlas_overlap")
    assert (face == 4).any() and not (face == 5).any()                    # tie inside a chunk: the lower index
    assert (face == 3).any() and not (face == 15).any()                   # tie across chunks: the earlier chunk
    row = face.view(32, 32)[10]
    assert not ((row >= 10) & (row < 20)).any() and ((face.view(32, 32)[9:12:2] == 13).any())   # NaN row: chunk 1 yields nothing
    _, face, _, _ = oracle_texels("xatlas_37")
    assert face.max() < 30                                                 # faces 30..36 (the tail) take no part
    _, face, bary, _ = oracle_texels("xatlas_7")
    assert (face == 0).all() and (bary == 0).all()                        # F < 10: no chunk at all
    _, face, _, _ = oracle_texels("custom_odd")
    assert face.max() == 12 and (face == 12).sum() > (face == 11).sum()    # padding texels clamp to the last face


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_obj_and_mtl_text_match_reference(name):
    from sdfstudio_b200 import texturing

    vertices, faces, normals, _, _ = case_inputs(name)
    tc, _ = oracle_bundle(name)
    _, cases = golden()
    assert texturing.obj_text(vertices.numpy(), faces.numpy(), normals.numpy(), tc.numpy()) == cases[name]["obj"]
    assert "".join(line + "\n" for line in texturing.MTL_LINES) == cases[name]["mtl"]


def parse_obj(text):
    rows = {"v": [], "vt": [], "vn": [], "f": []}
    for line in text.splitlines():
        tok = line.split()
        if tok and tok[0] in rows:
            rows[tok[0]].append([[int(i) for i in t.split("/")] for t in tok[1:]] if tok[0] == "f" else [float(x) for x in tok[1:]])
    return {k: np.array(v) for k, v in rows.items()}


def test_obj_round_trip():
    from sdfstudio_b200 import texturing

    g = torch.Generator().manual_seed(0)
    v, n = torch.randn(50, 3, generator=g), torch.randn(50, 3, generator=g)
    f = torch.randint(0, 50, (70, 3), generator=g)
    tc = torch.rand(70, 3, 2, generator=g)
    obj = parse_obj(texturing.obj_text(v.numpy(), f.numpy(), n.numpy(), tc.numpy()))
    assert np.array_equal(obj["v"].astype(np.float32), v.numpy()) and np.array_equal(obj["vn"].astype(np.float32), n.numpy())
    assert np.array_equal(obj["vt"][:, 0].astype(np.float32), tc.numpy().reshape(-1, 2)[:, 0])
    assert np.array_equal(obj["vt"][:, 1].astype(np.float32), np.float32(1) - tc.numpy().reshape(-1, 2)[:, 1])
    assert np.array_equal(obj["f"][:, :, 0] - 1, f.numpy()) and np.array_equal(obj["f"][:, :, 2], obj["f"][:, :, 0])
    assert np.array_equal(obj["f"][:, :, 1].ravel(), np.arange(1, 3 * 70 + 1))


def decode_png(data):
    """8-bit RGB, filter-0 rows, as png_bytes writes them: decoded with zlib alone, every chunk's CRC checked."""
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, chunks = 8, {}
    while pos < len(data):
        (n,) = struct.unpack(">I", data[pos:pos + 4])
        tag, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        assert struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0] == zlib.crc32(tag + body) & 0xFFFFFFFF
        chunks[tag] = chunks.get(tag, b"") + body
        pos += 12 + n
    w, h, depth, ctype, _, _, _ = struct.unpack(">IIBBBBB", chunks[b"IHDR"])
    assert (depth, ctype) == (8, 2) and b"IEND" in chunks
    raw = np.frombuffer(zlib.decompress(chunks[b"IDAT"]), np.uint8).reshape(h, 1 + 3 * w)
    assert (raw[:, 0] == 0).all()
    return raw[:, 1:].reshape(h, w, 3)


def test_png_decodes_to_the_quantised_image():
    from sdfstudio_b200 import texturing

    img = np.random.default_rng(0).uniform(-0.2, 1.2, (37, 53, 3)).astype(np.float32)
    img[0, 0] = [0.5 / 255, 1.5 / 255, 254.5 / 255]
    want = np.floor(np.clip(img, 0, 1) * 255 + 0.5).astype(np.uint8)
    assert np.array_equal(decode_png(texturing.png_bytes(img)), want)
    assert np.array_equal(decode_png(texturing.png_bytes(np.ones((1, 1, 3)))), np.full((1, 1, 3), 255, np.uint8))


def test_write_textured_mesh_files(tmp_path):
    from sdfstudio_b200 import texturing

    vertices, faces, normals, _, _ = case_inputs("xatlas_30")
    tc, _ = oracle_bundle("xatlas_30")
    z, cases = golden()
    texturing.write_textured_mesh(tmp_path, z["xatlas_30/image"], vertices.numpy(), faces.numpy(), normals.numpy(), tc.numpy())
    assert (tmp_path / "mesh.obj").read_text() == cases["xatlas_30"]["obj"]
    assert (tmp_path / "material_0.mtl").read_text() == cases["xatlas_30"]["mtl"]
    assert decode_png((tmp_path / "material_0.png").read_bytes()).shape == (40, 40, 3)


# ---------------------------------------------------------------------------------------------------------------------------------
# PLY input
# ---------------------------------------------------------------------------------------------------------------------------------
def test_ply_reader_reads_meshing_export(tmp_path):
    from sdfstudio_b200 import meshing, texturing

    g = np.random.default_rng(1)
    m = meshing.Mesh(g.normal(size=(40, 3)), g.integers(0, 40, (60, 3)), g.normal(size=(40, 3)))
    m.export(tmp_path / "m.ply")
    mesh = texturing.get_mesh_from_filename(str(tmp_path / "m.ply"))
    assert mesh.vertices.dtype == torch.float32 and mesh.faces.dtype == torch.int64 and mesh.normals.dtype == torch.float32
    assert np.array_equal(mesh.vertices.numpy(), m.vertices.astype(np.float32))
    assert np.array_equal(mesh.faces.numpy(), m.faces)
    assert np.array_equal(mesh.normals.numpy(), m.vertex_normals.astype(np.float32))
    # no reduction asked (more target faces than the mesh has): pymeshlab is not needed
    assert len(texturing.get_mesh_from_filename(str(tmp_path / "m.ply"), target_num_faces=1000).faces) == 60


def test_ply_without_normals_gets_area_weighted_normals(tmp_path):
    from sdfstudio_b200 import texturing

    # a unit cube's 12 triangles, written with double coordinates and no normals
    v = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float64)
    f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4],
                  [1, 5, 7], [1, 7, 3]], np.int32)
    fr = np.empty(len(f), dtype=[("n", "u1"), ("i", "<i4", (3,))])
    fr["n"], fr["i"] = 3, f
    head = ("ply\nformat binary_little_endian 1.0\ncomment cube\nelement vertex 8\nproperty double x\nproperty double y\nproperty double z\n"
            "element face 12\nproperty list uchar int vertex_indices\nend_header\n")
    (tmp_path / "c.ply").write_bytes(head.encode() + v.astype("<f8").tobytes() + fr.tobytes())
    mesh = texturing.get_mesh_from_filename(str(tmp_path / "c.ply"))
    assert mesh.faces.tolist() == f.tolist() and np.array_equal(mesh.vertices.numpy(), v.astype(np.float32))
    fv = v[f]
    acc = np.zeros_like(v)
    for k in range(3):
        np.add.at(acc, f[:, k], np.cross(fv[:, 1] - fv[:, 0], fv[:, 2] - fv[:, 0]))   # twice each face's area along its normal
    acc /= np.linalg.norm(acc, axis=1, keepdims=True)
    assert np.allclose(mesh.normals.numpy(), acc, atol=1e-6)


@pytest.mark.skipif(importlib.util.find_spec("pymeshlab") is not None, reason="pymeshlab is installed")
def test_decimation_without_pymeshlab_is_an_import_error(tmp_path):
    from sdfstudio_b200 import meshing, texturing

    g = np.random.default_rng(2)
    meshing.Mesh(g.normal(size=(10, 3)), g.integers(0, 10, (20, 3))).export(tmp_path / "m.ply")
    with pytest.raises(ImportError, match="pymeshlab"):
        texturing.get_mesh_from_filename(str(tmp_path / "m.ply"), target_num_faces=10)


# ---------------------------------------------------------------------------------------------------------------------------------
# argument errors
# ---------------------------------------------------------------------------------------------------------------------------------
def _cpu_pipeline():
    import types

    return types.SimpleNamespace(device=torch.device("cpu"), model=None)


def test_export_argument_errors(tmp_path):
    from sdfstudio_b200 import texturing

    vertices, faces, normals, _, _ = case_inputs("custom_odd")
    mesh = texturing.Mesh(vertices, faces, normals)
    with pytest.raises(ValueError, match="Unwrap method"):
        texturing.export_textured_mesh(mesh, _cpu_pipeline(), tmp_path, unwrap_method="smart")
    with pytest.raises(ValueError, match="Ray length method"):
        texturing.export_textured_mesh(mesh, _cpu_pipeline(), tmp_path, unwrap_method="custom", px_per_uv_triangle=4, raylen_method="far")
    with pytest.raises(ValueError, match="px_per_uv_triangle"):
        texturing.export_textured_mesh(mesh, _cpu_pipeline(), tmp_path, unwrap_method="custom")


@pytest.mark.skipif(importlib.util.find_spec("xatlas") is not None, reason="xatlas is installed")
def test_missing_xatlas_names_the_custom_method(tmp_path):
    from sdfstudio_b200 import texturing

    vertices, faces, normals, _, _ = case_inputs("xatlas_30")
    with pytest.raises(ImportError, match='unwrap_method="custom"'):
        texturing.unwrap_mesh_with_xatlas(vertices, faces, normals)
    with pytest.raises(ImportError, match='unwrap_method="custom"'):
        texturing.export_textured_mesh(texturing.Mesh(vertices, faces, normals), _cpu_pipeline(), tmp_path)


def test_signatures_match_reference_defaults():
    """The drop-ins keep the reference's parameter names and defaults (texture_utils.py, scripts/texture.py:36-42)."""
    import inspect

    from sdfstudio_b200 import texturing

    def params(fn):
        return [(p.name, None if p.default is inspect.Parameter.empty else p.default) for p in inspect.signature(fn).parameters.values()]

    assert params(texturing.unwrap_mesh_per_uv_triangle) == [("vertices", None), ("faces", None), ("vertex_normals", None),
                                                             ("px_per_uv_triangle", None)]
    assert params(texturing.unwrap_mesh_with_xatlas) == [("vertices", None), ("faces", None), ("vertex_normals", None),
                                                         ("num_pixels_per_side", 1024), ("num_faces_per_barycentric_chunk", 10)]
    assert params(texturing.export_textured_mesh) == [("mesh", None), ("pipeline", None), ("output_dir", None), ("px_per_uv_triangle", None),
                                                      ("unwrap_method", "xatlas"), ("raylen_method", "edge"), ("num_pixels_per_side", 1024)]
    assert params(texturing.get_mesh_from_filename) == [("filename", None), ("target_num_faces", None)]
    assert params(texturing.texture_mesh)[3:] == [("px_per_uv_triangle", 4), ("unwrap_method", "xatlas"), ("num_pixels_per_side", 2048),
                                                  ("target_num_faces", 50000)]
