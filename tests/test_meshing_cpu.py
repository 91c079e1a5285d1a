"""CPU: the generated marching-cubes table, the numpy restatement of the kernel (oracle/marching_cubes.py) on analytic volumes, the
restatement of the reference's mesh-extraction functions against the golden minted from the unmodified reference, the drop-ins'
signatures, the Mesh container, and the PLY writer and reader every exporter shares."""
import inspect
import json
import os
import struct
from collections import Counter
from pathlib import Path

import numpy as np
import pytest

from oracle import marching_cubes as omc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _grid(n, lo=-1.0, hi=1.0):
    x = np.linspace(lo, hi, n)
    return np.meshgrid(x, x, x, indexing="ij")


def sphere_volume(n, r=0.6):
    X, Y, Z = _grid(n)
    return (np.sqrt(X**2 + Y**2 + Z**2) - r).astype(np.float32)


def torus_volume(n):
    X, Y, Z = _grid(n)
    return (np.sqrt((np.sqrt(X**2 + Y**2) - 0.5) ** 2 + Z**2) - 0.2).astype(np.float32)


def two_spheres_volume(n):
    X, Y, Z = _grid(n)
    return np.minimum(np.sqrt((X - 0.45) ** 2 + Y**2 + Z**2) - 0.3, np.sqrt((X + 0.45) ** 2 + Y**2 + Z**2) - 0.3).astype(np.float32)


def noise_volume(n, seed=0):
    """uniform noise in (0, 1) inside a border of 1.0: the level-0.5 surface is closed in the box."""
    v = np.ones((n + 2,) * 3, np.float32)
    v[1:-1, 1:-1, 1:-1] = np.random.default_rng(seed).random((n,) * 3, dtype=np.float32)
    return v


def undirected_edge_counts(faces):
    e = np.sort(np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]), axis=1)
    _, c = np.unique(e, axis=0, return_counts=True)
    return c


def directed_edges_balance(faces):
    c = Counter(map(tuple, np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]).tolist()))
    return all(c[(a, b)] == c[(b, a)] for (a, b) in c)


def cube_keys(vol, level):
    """(case, 6-bit face decisions) of every cube with a cut edge, computed independently of the oracle's vectorised path."""
    nx, ny, nz = vol.shape
    lvl = np.float32(level)
    case = np.zeros((nx - 1, ny - 1, nz - 1), np.int64)
    for n in range(8):
        case |= (vol[n & 1:nx - 1 + (n & 1), (n >> 1) & 1:ny - 1 + ((n >> 1) & 1), (n >> 2) & 1:nz - 1 + ((n >> 2) & 1)] < lvl).astype(np.int64) << n
    return case


# ---------------------------------------------------------------------------------------------------------------------------------
# the table
# ---------------------------------------------------------------------------------------------------------------------------------
def test_committed_table_is_the_generated_one():
    with open(omc.TABLES_H) as fh:
        assert fh.read() == omc.tables_header()


def test_table_entries_trace_the_face_rule():
    """each entry uses exactly the case's cut edges; the fan boundaries are closed loops whose segments are the face rule's segments on
    all six faces, oriented with the inside corners on their left (seen from outside); the fans' interior diagonals cancel."""
    _, entries = omc.table()
    assert len(entries) == sum(1 << len(omc.ambiguous_faces(c)) for c in range(256))
    for case, bits, tris in entries:
        used = sorted({e for t in tris for e in t})
        assert used == omc.cut_edges(case), (case, bits)
        directed = Counter((t[m], t[(m + 1) % 3]) for t in tris for m in range(3))
        boundary = {d for d in directed if directed[(d[1], d[0])] == 0}
        for d, c in directed.items():
            assert c == 1, (case, bits, d)
        amb = omc.ambiguous_faces(case)
        expect = set()
        for f in range(6):
            joined = f in amb and bool((bits >> amb.index(f)) & 1)
            for e1, e2 in omc._face_segments(case, f, joined):
                t, h = omc._orient(case, f, e1, e2)
                # the fans wind opposite to the traced loops (descent normals)
                expect.add((h, t) if omc._flip() else (t, h))
        assert boundary == expect, (case, bits)


def test_single_corner_triangle_points_down_the_values():
    (a, b, c), = omc.triangulate(1, 0)
    mid = [sum(omc.corner_xyz(x) for x in omc.edge_corners(e)) / 2 for e in (a, b, c)]
    assert np.dot(np.cross(mid[1] - mid[0], mid[2] - mid[0]), omc.corner_xyz(0) - mid[0]) > 0


# ---------------------------------------------------------------------------------------------------------------------------------
# the kernel's restatement on analytic volumes
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name, make, euler", [("sphere", sphere_volume, 2), ("torus", torus_volume, 0), ("two_spheres", two_spheres_volume, 4)])
def test_analytic_meshes_are_closed_manifolds(name, make, euler):
    V, F, N = omc.marching_cubes(make(64))
    assert len(F) > 0
    counts = undirected_edge_counts(F)
    assert (counts == 2).all(), name
    assert len(V) - len(counts) + len(F) == euler
    assert len(np.unique(F)) == len(V)                    # no unreferenced vertex
    assert np.isfinite(N).all() and np.allclose(np.linalg.norm(N, axis=1), 1.0, atol=1e-5)


def test_vertices_lie_on_their_edges_at_t():
    vol = sphere_volume(40)
    V, F, _ = omc.marching_cubes(vol, spacing=(1.0, 1.0, 1.0))
    frac = V - np.floor(V)
    on_axis = frac != 0
    assert (on_axis.sum(1) <= 1).all()
    for v in V[on_axis.sum(1) == 1]:
        a = int(np.nonzero(v != np.floor(v))[0][0])
        i0 = np.floor(v).astype(int)
        i1 = i0.copy()
        i1[a] += 1
        v0, v1 = vol[tuple(i0)], vol[tuple(i1)]
        t = (np.float32(0) - v0) / (v1 - v0)
        assert np.float32(i0[a]) + t == np.float32(v[a])


def test_sphere_orientation_and_area():
    r, n = 0.6, 128
    vol = sphere_volume(n, r)
    h = 2.0 / (n - 1)
    V, F, N = omc.marching_cubes(vol, spacing=(h, h, h))
    V = V.astype(np.float64)
    signed = np.einsum("ij,ij->i", V[F[:, 0]], np.cross(V[F[:, 1]], V[F[:, 2]])).sum() / 6
    assert signed < 0                                       # descent: normals point into the sphere
    area = 0.5 * np.linalg.norm(np.cross(V[F[:, 1]] - V[F[:, 0]], V[F[:, 2]] - V[F[:, 0]]), axis=1).sum()
    assert abs(area / (4 * np.pi * r * r) - 1) < 0.01
    # vertex normals agree with the face normals and point inward
    c = V - 1.0                                             # the lattice starts at -1
    assert (np.einsum("ij,ij->i", N, c) < 0).all()


# Entries a trilinear cube does not realise.  Only the two checkerboard cases (105, 150: all six faces ambiguous) have any: 4e6 random
# cubes of those cases, corner magnitudes spread over 12 e-folds, realised 46 of their 64 decider patterns and never these 18.  Each of
# them joins the inside corners across both faces of an opposite pair (bits 0-1, 2-3 or 4-5); the table still holds their traced loops.
_CHECKERBOARD_UNREALISED = (3, 7, 11, 12, 13, 14, 15, 19, 28, 35, 44, 48, 49, 50, 51, 52, 56, 60)
UNREACHED = {(c, b) for c in (105, 150) for b in _CHECKERBOARD_UNREALISED}


def test_noise_volume_hits_every_case_and_stays_watertight():
    vol = noise_volume(100)
    V, F, _ = omc.marching_cubes(vol, 0.5)
    assert directed_edges_balance(F)
    case = cube_keys(vol, 0.5)
    assert len(np.unique(case)) == 256
    # which (case, decider bits) entries occurred: recompute the decisions from the face rule on the corner values
    cs = case.reshape(-1)
    nx, ny, nz = vol.shape
    ii, jj, kk = np.unravel_index(np.arange(cs.size), (nx - 1, ny - 1, nz - 1))
    p0 = (ii * ny + jj) * nz + kk
    rel = vol.reshape(-1)[p0[:, None] + omc._corner_offsets(ny, nz)[None, :]] - np.float32(0.5)
    bits = np.zeros(cs.size, np.int64)
    rank = np.zeros(cs.size, np.int64)
    for f in range(6):
        q = omc.face_corners(f)
        amb = np.array([omc.face_ambiguous(c, f) for c in range(256)])[cs]
        out = ((cs >> q[0]) & 1) == 0
        a, c = np.where(out, rel[:, q[0]], rel[:, q[1]]), np.where(out, rel[:, q[2]], rel[:, q[3]])
        b, d = np.where(out, rel[:, q[1]], rel[:, q[0]]), np.where(out, rel[:, q[3]], rel[:, q[2]])
        with np.errstate(all="ignore"):
            s = (a * c - b * d) / (((a + c) - b) - d)
        bits |= np.where(amb, (s < 0).astype(np.int64) << rank, 0)
        rank += amb
    hit = set(zip(cs.tolist(), bits.tolist()))
    _, entries = omc.table()
    missing = {(c, b) for c, b, _ in entries} - hit
    assert missing == set(UNREACHED), sorted(missing)


def test_masks_extents_and_degenerate_corners():
    vol = sphere_volume(24)
    assert omc.marching_cubes(vol[:1])[1].shape == (0, 3)
    assert omc.marching_cubes(np.ones((5, 5, 5), np.float32))[1].shape == (0, 3)
    # a mask keeps only the cubes it sets, and no vertex without a face
    m = np.zeros(vol.shape, np.uint8)
    m[:12] = 1
    V, F, _ = omc.marching_cubes(vol, mask=m)
    assert len(F) and len(np.unique(F)) == len(V) and (V[:, 0] <= 12).all()
    # corners exactly at the level: degenerate but finite
    q = np.round(sphere_volume(20) * 4).astype(np.float32)
    V, F, N = omc.marching_cubes(q, 0.0)
    assert len(F) and np.isfinite(V).all() and np.isfinite(N).all()


# ---------------------------------------------------------------------------------------------------------------------------------
# the reference's mesh-extraction functions: restatement == golden, signatures
# ---------------------------------------------------------------------------------------------------------------------------------
def _golden():
    with open(os.path.join(ROOT, "tests", "golden", "marching_cubes.json")) as fh:
        meta = json.load(fh)
    return meta, np.load(os.path.join(ROOT, "tests", "golden", "marching_cubes.npz"))


def restated_calls(name):
    from oracle import make_golden_marching_cubes as mk

    fn, kw, f = mk.cases()[name]
    calls = []

    def mc(volume, level, spacing, mask, offset):
        calls.append(dict(volume=volume, level=level, spacing=list(spacing), mask=mask, offset=offset.tolist()))

    kw = dict(kw)
    kw.pop("inv_contraction", None)
    if fn == "get_surface_sliding":
        omc.surface_sliding(f, mc, **kw)
    elif fn == "get_surface_occupancy":
        omc.surface_occupancy(f, mc, **kw)
    else:
        omc.surface_sliding_with_contraction(f, mc, **kw)
    return calls


GOLDEN_CASES = ["sliding_512", "sliding_512_mask", "sliding_1024_partial", "contraction_512", "occupancy_100"]


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_restatement_matches_reference_golden(name):
    meta, arr = _golden()
    want = meta["cases"][name]
    got = restated_calls(name)
    assert len(got) == len(want) > 0
    for n, (g, w) in enumerate(zip(got, want)):
        assert g["level"] == w["level"] and g["spacing"] == w["spacing"] and g["offset"] == w["offset"]
        assert list(g["volume"].shape) == w["shape"]
        assert (None if g["mask"] is None else int(g["mask"].sum())) == w["mask_count"]
        flat = g["volume"].reshape(-1)
        assert np.array_equal(flat[arr[f"{name}/{n}/cross_idx"]], arr[f"{name}/{n}/cross_val"])
        assert np.array_equal(g["volume"][g["volume"].shape[0] // 2, ::4, ::4], arr[f"{name}/{n}/slice"])


def test_dropin_signatures_match_reference():
    from sdfstudio_b200 import meshing

    meta, _ = _golden()
    for name, sig in meta["signatures"].items():
        params = inspect.signature(getattr(meshing, name)).parameters
        mine = [[n, None if p.default is inspect.Parameter.empty else p.default] for n, p in params.items()]
        ref = [[n, None if d is None else eval(d, {"Path": Path})] for n, d in sig]
        assert mine == ref, name


# ---------------------------------------------------------------------------------------------------------------------------------
# Mesh and PLY files
# ---------------------------------------------------------------------------------------------------------------------------------
def read_ply(path):
    with open(path, "rb") as fh:
        data = fh.read()
    head, body = data.split(b"end_header\n", 1)
    lines = head.decode().splitlines()
    assert lines[0] == "ply" and lines[1] == "format binary_little_endian 1.0"
    nv = int(next(l for l in lines if l.startswith("element vertex")).split()[-1])
    nf = int(next(l for l in lines if l.startswith("element face")).split()[-1])
    props = [l.split()[-1] for l in lines if l.startswith("property float")]
    v = np.frombuffer(body, dtype=[(p, "<f4") for p in props], count=nv)
    f = np.frombuffer(body, dtype=[("n", "u1"), ("i", "<i4", (3,))], count=nf, offset=nv * 4 * len(props))
    assert (f["n"] == 3).all() and len(body) == nv * 4 * len(props) + nf * 13
    return np.stack([v["x"], v["y"], v["z"]], 1), np.array(f["i"]), np.stack([v["nx"], v["ny"], v["nz"]], 1)


def test_mesh_export_roundtrip_concatenate_and_merge(tmp_path):
    from sdfstudio_b200.meshing import Mesh

    V, F, N = omc.marching_cubes(sphere_volume(16), spacing=(0.1, 0.1, 0.1))
    a = Mesh(V, F, N)
    b = Mesh(V + 10.0, F, N)
    m = Mesh.concatenate([a, b])
    assert m.vertices.shape == (2 * len(V), 3) and m.faces[len(F):].min() == len(V)
    p = tmp_path / "m.ply"
    m.export(p)
    v2, f2, n2 = read_ply(p)
    assert np.array_equal(v2, m.vertices.astype(np.float32)) and np.array_equal(f2, m.faces) and np.array_equal(n2, m.vertex_normals.astype(np.float32))
    # welding: two copies of the same mesh collapse onto one, faces follow, first-occurrence order kept
    w = Mesh.concatenate([a, Mesh(V, F, N)])
    w.merge_vertices(digits_vertex=6)
    assert np.array_equal(w.vertices, a.vertices) and np.array_equal(w.faces, np.concatenate([F, F]))
    assert Mesh.concatenate([]).faces.shape == (0, 3)


def test_ply_reader_rejects_ascii_and_polygons(tmp_path):
    from sdfstudio_b200 import meshing

    (tmp_path / "a.ply").write_bytes(b"ply\nformat ascii 1.0\nelement vertex 0\nend_header\n")
    with pytest.raises(ValueError, match="binary_little_endian"):
        meshing.read_ply(tmp_path / "a.ply")
    fr = np.zeros(1, dtype=[("n", "u1"), ("i", "<i4", (3,))])
    fr["n"] = 4
    (tmp_path / "q.ply").write_bytes(b"ply\nformat binary_little_endian 1.0\nelement vertex 0\nproperty float x\nproperty float y\n"
                                     b"property float z\nelement face 1\nproperty list uchar int vertex_indices\nend_header\n" + fr.tobytes())
    with pytest.raises(ValueError, match="triangle"):
        meshing.read_ply(tmp_path / "q.ply")


def test_coloured_ply_round_trip_and_uncoloured_bytes(tmp_path):
    """Mesh.export with vertex colours reads back through meshing.read_ply with its colours quantised as the texture PNG's; without
    colours the file is byte for byte the float-only PLY."""
    from sdfstudio_b200 import meshing

    g = np.random.default_rng(0)
    v, n, f = g.normal(size=(7, 3)), g.normal(size=(7, 3)), g.integers(0, 7, size=(5, 3))
    c = np.array([[0.0, 1.0, 0.5], [-0.2, 1.3, 0.499], [0.5 / 255, 1.5 / 255, 2.5 / 255], [np.nan, 0.25, 0.75], [0.1, 0.2, 0.3],
                  [0.998, 0.002, 0.0], [1.0, 1.0, 1.0]], np.float32)
    meshing.Mesh(v, f, n).export(tmp_path / "c.ply", vertex_colors=c)
    rv, rf, rn = meshing.read_ply(tmp_path / "c.ply")
    assert np.array_equal(rv, v.astype(np.float32)) and np.array_equal(rf, f) and np.array_equal(rn, n.astype(np.float32))
    data = (tmp_path / "c.ply").read_bytes()
    head, body = data.split(b"end_header\n")
    assert head.endswith(b"property uchar red\nproperty uchar green\nproperty uchar blue\nproperty uchar alpha\nelement face 5\n"
                         b"property list uchar int vertex_indices\n")
    rec = np.frombuffer(body, dtype=[("p", "<f4", (6,)), ("c", "u1", (4,))], count=7)
    with np.errstate(invalid="ignore"):
        want = np.floor(np.clip(c, 0, 1) * np.float32(255) + np.float32(0.5)).astype(np.uint8)
    assert np.array_equal(rec["c"][:, :3][~np.isnan(c).any(1)], want[~np.isnan(c).any(1)]) and (rec["c"][:, 3] == 255).all()
    assert rec["c"][2, :3].tolist() == [1, 2, 3] and rec["c"][0].tolist() == [0, 255, 128, 255]

    meshing.Mesh(v, f, n).export(tmp_path / "u.ply")
    vert = b"".join(struct.pack("<6f", *v[i], *n[i]) for i in range(7))
    face = b"".join(struct.pack("<B3i", 3, *f[i]) for i in range(5))
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex 7\n" + "".join(f"property float {p}\n" for p in ("x", "y", "z", "nx", "ny", "nz"))
              + "element face 5\nproperty list uchar int vertex_indices\nend_header\n").encode()
    assert (tmp_path / "u.ply").read_bytes() == header + vert + face
