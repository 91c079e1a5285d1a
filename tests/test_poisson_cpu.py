"""CPU checks of the Poisson reconstruction: the fp64 oracle's operator (zero row sums, the interior stencil, SPD), its meshes on a
sphere and a torus, the vertex removal and density trim of ExportPoissonMesh on hand-built meshes, the signature of
``poisson_mesh`` against ExportPoissonMesh's fields, and the refusals.

Bounds the GPU tests use, set here on the oracle: on a uniformly sampled sphere (about two points per surface cell) at depths 5 and 6
the mesh is closed (every edge in exactly two faces, Euler characteristic 2), every face normal points outward, and every vertex lies
within SPHERE_BOUND_H = 0.5 h of the sphere (measured: 0.27 h at depth 5, 0.39 h at depth 6)."""
import inspect
import json
import os

import numpy as np
import pytest
import torch

from oracle import poisson as op

SPHERE_BOUND_H = 0.5


def topology(v, f):
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    _, cnt = np.unique(e, axis=0, return_counts=True)
    return bool((cnt == 2).all()), len(v) - len(cnt) + len(f)


def outward_fraction(v, f, centre_fn):
    fn = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    c = v[f].mean(1)
    return float(((fn * (c - centre_fn(c))).sum(1) > 0).mean())


def test_stiffness_rows_and_stencil():
    h = 0.25
    L = op.stiffness(4, h).toarray()
    np.testing.assert_allclose(L.sum(1), 0.0, atol=1e-15)
    m = 5
    centre = (2 * m + 2) * m + 2
    row = L[centre].reshape(m, m, m)[1:4, 1:4, 1:4]
    for d in np.ndindex(3, 3, 3):
        nz = sum(x != 1 for x in d)
        want = {0: 8 * h / 3, 1: 0.0, 2: -h / 6, 3: -h / 12}[nz]
        assert row[d] == pytest.approx(want, abs=1e-15)


def test_system_spd():
    p, n, _ = op.sphere_cloud(500)
    s = op.assemble(p, n, 2)
    A = (s["L"] + s["alpha_a"] * s["S"]).toarray()
    np.testing.assert_allclose(A, A.T, atol=1e-15)
    assert np.linalg.eigvalsh(A).min() > 0


@pytest.mark.parametrize("depth", [5, 6])
def test_oracle_sphere(depth):
    p, n, c = op.sphere_cloud(20000)
    s, v, f, _, dens, rgb = op.reconstruct(p, n, c, depth)
    closed, euler = topology(v, f)
    assert closed and euler == 2
    assert outward_fraction(v, f, lambda x: 0 * x) == 1.0
    assert np.abs(np.linalg.norm(v, axis=1) - 0.6).max() <= SPHERE_BOUND_H * s["h"]
    assert (dens > 0).all() and (rgb >= 0).all() and (rgb <= 1 + 1e-12).all()


def test_oracle_torus():
    p, n, c = op.torus_cloud(30000)
    _, v, f, _, _, _ = op.reconstruct(p, n, c, 5)
    closed, euler = topology(v, f)
    assert closed and euler == 0


def _mesh():
    from sdfstudio_b200 import meshing

    v = np.arange(15, dtype=np.float64).reshape(5, 3)
    f = np.array([[0, 1, 2], [1, 2, 3], [2, 3, 4], [0, 2, 4]])
    m = meshing.Mesh(v, f, v * 0 + 1)
    m.vertex_colors = v / 15
    return m


def test_remove_vertices_by_mask():
    from sdfstudio_b200 import poisson

    m = poisson.remove_vertices_by_mask(_mesh(), np.array([False, True, False, False, False]))
    np.testing.assert_array_equal(m.vertices, np.arange(15).reshape(5, 3)[[0, 2, 3, 4]])
    np.testing.assert_array_equal(m.faces, [[1, 2, 3], [0, 1, 3]])
    np.testing.assert_array_equal(m.vertex_colors, (np.arange(15).reshape(5, 3) / 15)[[0, 2, 3, 4]])
    ov, of = op.remove_vertices_by_mask(_mesh().vertices, _mesh().faces, [False, True, False, False, False])
    np.testing.assert_array_equal(ov, m.vertices)
    np.testing.assert_array_equal(of, m.faces)
    # a mask that drops a vertex of every face leaves vertices without faces
    m = poisson.remove_vertices_by_mask(_mesh(), np.array([False, False, True, False, False]))
    assert m.faces.shape == (0, 3) and len(m.vertices) == 4
    m = poisson.remove_vertices_by_mask(_mesh(), np.zeros(5, bool))
    np.testing.assert_array_equal(m.faces, _mesh().faces)
    with pytest.raises(ValueError):
        poisson.remove_vertices_by_mask(_mesh(), np.zeros(4, bool))


def test_density_trim():
    from sdfstudio_b200 import poisson

    assert not poisson.low_density_mask(np.full(7, 3.0)).any()            # strict <: all equal keeps all
    d = np.array([1.0, 1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0, 8.0, 9.0, 10.0])
    np.testing.assert_array_equal(poisson.low_density_mask(d), d < np.quantile(d, 0.1))
    assert poisson.low_density_mask(d).sum() == 0                         # quantile 1.0: the tied minimum is not below it
    d = np.array([0.0, 1.0, 1.0, 2.0, 5.0])
    np.testing.assert_array_equal(poisson.low_density_mask(d), [True, False, False, False, False])
    np.testing.assert_array_equal(poisson.low_density_mask(torch.tensor(d)), op.low_density_mask(d))
    assert poisson.low_density_mask(np.zeros(0)).shape == (0,)


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(os.path.dirname(__file__), "golden", "poisson.json")) as fh:
        return json.load(fh)


def test_poisson_mesh_signature(golden):
    """poisson_mesh takes ExportPoissonMesh's fields (all but load_config and output_dir, which become renderer / output_dir) with the
    reference's defaults, as minted from scripts/exporter.py."""
    from sdfstudio_b200 import poisson

    params = inspect.signature(poisson.poisson_mesh).parameters
    fields = [(name, d) for name, d in golden["fields"] if name not in ("load_config", "output_dir")]
    assert len(fields) == 17
    for name, d in fields:
        default = params[name].default
        assert (list(default) if isinstance(default, tuple) else default) == d["default"], name
    assert inspect.signature(poisson.create_from_point_cloud_poisson).parameters["depth"].default == 8
    assert inspect.signature(poisson.create_from_point_cloud_poisson).parameters["scale"].default == 1.1


def test_normal_check_message(golden):
    """validate_pipeline's lines after its opening "Checking ..." line, in order, are the ValueError's message."""
    from sdfstudio_b200 import poisson

    case = golden["validate_pipeline"]["missing_normals"]
    assert case["exit_code"] == 1 and case["rays"] == [dict(origins=[[0.0, 0.0, 0.0]], directions=[[1.0, 1.0, 1.0]])]
    outputs = {k: None for k in case["outputs"]}
    assert poisson._normal_check_message(case["kwargs"].get("normal_output_name", "normals"), outputs) == "\n".join(case["printed"][1:])
    assert golden["validate_pipeline"]["present"]["exit_code"] is None
    assert golden["validate_pipeline"]["open3d"]["rays"] == []      # no check, no render with normal_method="open3d"


@pytest.mark.parametrize("case", ["depth0", "depth11", "depth_float", "empty", "zero_extent", "zero_normals", "nan_point", "scale"])
def test_refusals(case):
    from sdfstudio_b200 import poisson

    p, n, c = (torch.from_numpy(a) for a in op.sphere_cloud(100))
    depth, scale = 5, 1.1
    if case == "depth0":
        depth = 0
    elif case == "depth11":
        depth = 11
    elif case == "depth_float":
        depth = 5.0
    elif case == "empty":
        p, n, c = p[:0], n[:0], c[:0]
    elif case == "zero_extent":
        p = torch.full_like(p, 0.25)
    elif case == "zero_normals":
        n = torch.zeros_like(n)
    elif case == "nan_point":
        p[3, 1] = float("nan")
    else:
        scale = 0.5
    with pytest.raises(ValueError):
        poisson.build_system(p, n, c, depth, scale)
