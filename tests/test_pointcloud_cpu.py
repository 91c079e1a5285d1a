"""CPU checks of the point-cloud exporter: restatement (a) of the reference's generate_point_cloud against the golden bundle minted
from the unmodified reference, the open3d outlier rules of restatement (c) on hand-built clouds, the vertex-only PLY, and the
signatures and defaults of the drop-ins."""
import inspect
import json
import os
import struct

import numpy as np
import pytest
import torch

from oracle import pointcloud as opc
from oracle.make_golden_pointcloud import CASES, ERRORS, stub_kept
from sdfstudio_b200 import meshing, pointcloud

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(GOLDEN, "pointcloud.json")) as fh:
        meta = json.load(fh)
    return meta, np.load(os.path.join(GOLDEN, "pointcloud.npz"))


def _run_a(pk, gk, record):
    def remove(pts, nb, sr):
        record["outlier_input"] = pts.copy()
        return stub_kept(len(pts))

    def estimate(pts):
        record["estimated"] = True
        return None

    pipeline = opc.FakePipeline(**pk)
    return pipeline, opc.reference_flow(pipeline, remove, estimate, **gk)


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_a_equals_golden(golden, name):
    meta, arrays = golden
    case = meta["cases"][name]
    record = {}
    pipeline, out = _run_a(case["pipeline"], case["kwargs"], record)
    assert pipeline.datamanager.calls == case["batches"] and out["batches"] == case["batches"]
    np.testing.assert_array_equal(out["points"], arrays[f"{name}/points"])
    np.testing.assert_array_equal(out["colors"], arrays[f"{name}/colors"])
    if f"{name}/normals" in arrays:
        np.testing.assert_array_equal(out["normals"], arrays[f"{name}/normals"])
    else:
        assert out["normals"] is None or case["estimated"]
    assert (list(out["outlier_args"]) if out["outlier_args"] else None) == case["outlier_args"]
    assert out["estimated"] == case["estimated"]
    if f"{name}/outlier_points" in arrays:
        np.testing.assert_array_equal(record["outlier_input"], arrays[f"{name}/outlier_points"])
    assert len(out["points"]) == case["n_points"]


def test_golden_covers_the_flow(golden):
    meta, _ = golden
    c = meta["cases"]
    assert c["normals_masked"]["batches"] > 3                    # every third batch keeps no point
    assert c["normals_masked"]["kwargs"]["num_points"] % c["normals_masked"]["pipeline"]["n"]
    assert c["zero_points"]["batches"] == 1
    assert c["no_outliers"]["outlier_args"] is None and c["estimate"]["estimated"]
    assert c["estimate"]["outlier_args"] == [20, 2.5]


@pytest.mark.parametrize("name", sorted(ERRORS))
def test_restatement_a_errors(golden, name):
    meta, _ = golden
    err = meta["errors"][name]
    assert err["exit_code"] == 1
    pipeline = opc.FakePipeline(**err["pipeline"])
    with pytest.raises(ValueError):
        opc.reference_flow(pipeline, lambda p, n, s: stub_kept(len(p)), lambda p: None, **err["kwargs"])
    assert pipeline.datamanager.calls == err["batches"]


def test_box_assert(golden):
    meta, _ = golden
    with pytest.raises(AssertionError) as e:
        opc.reference_flow(opc.FakePipeline(n=50, seed=10), None, None, bounding_box_min=(0, 0, 0), bounding_box_max=(1, 0, 1))
    assert str(e.value) == meta["errors"]["box_min_not_below_max"]["message"]


def _describe(v):
    if v is inspect.Parameter.empty:
        return {"required": True}
    return {"default": list(v) if isinstance(v, tuple) else v}


def test_signatures(golden):
    meta, _ = golden
    sig = meta["signatures"]
    ours = [[p.name, _describe(p.default)] for p in inspect.signature(pointcloud.generate_point_cloud).parameters.values()]
    assert ours == sig["generate_point_cloud"]
    params = inspect.signature(pointcloud.point_cloud).parameters
    for name, d in sig["ExportPointCloud"]:
        if name in ("load_config", "output_dir"):
            continue
        assert name in params, name
        assert _describe(params[name].default) == d, name


# ---------------------------------------------------------------------------------------------------------------------------------
# (c): open3d's outlier rules
# ---------------------------------------------------------------------------------------------------------------------------------
def test_duplicates_beyond_k_are_dropped():
    rng = np.random.default_rng(0)
    pts = np.concatenate([np.full((25, 3), 0.25, np.float32), rng.uniform(-1, 1, (200, 3)).astype(np.float32)])
    mean, _ = opc.knn(pts, 20)
    assert (mean[:25] == 0).all() and (mean[25:] > 0).all()
    kept, _ = opc.statistical_outliers(mean, 10.0)
    assert not np.isin(np.arange(25), kept).any() and len(kept) == 200


def test_small_clouds():
    pts = np.array([[0, 0, 0], [1, 0, 0], [0, 2, 0], [0, 0, 3], [1, 1, 1]], np.float32)
    mean, idx = opc.knn(pts, 20)
    assert (idx[:, 5:] == -1).all() and (idx[:, 0] == np.arange(5)).all()
    assert mean[0] == (0.0 + 1.0 + np.sqrt(3.0) + 2.0 + 3.0) / 5
    assert len(opc.statistical_outliers(opc.knn(pts[:1], 20)[0], 1.0)[0]) == 0       # N = 1: its only neighbour is itself
    mean0, idx0 = opc.knn(np.zeros((0, 3), np.float32), 20)
    assert mean0.shape == (0,) and idx0.shape == (0, 20)
    assert len(opc.statistical_outliers(mean0, 1.0)[0]) == 0


def test_threshold_is_strict_and_bessel_corrected():
    kept, thr = opc.statistical_outliers(np.array([1.0, 1.0, 1.0, 1.0]), 2.0)   # std 0: every point sits on the threshold
    assert thr == 1.0 and len(kept) == 0
    kept, thr = opc.statistical_outliers(np.array([1.0, 3.0, 5.0, 0.0]), 1.0)    # valid: 1, 3, 5; std = sqrt(8 / 2) = 2
    assert thr == 5.0 and kept.tolist() == [0, 1]
    m = np.random.default_rng(1).uniform(0.1, 1.0, 101)
    _, thr = opc.statistical_outliers(m, 0.7)
    assert thr == pytest.approx(m.mean() + 0.7 * m.std(ddof=1), rel=1e-14)


@pytest.mark.parametrize("nb,ratio", [(0, 1.0), (-3, 1.0), (20, 0.0), (20, -1.0)])
def test_outlier_refusals(nb, ratio):
    with pytest.raises(ValueError):
        pointcloud.remove_statistical_outlier(torch.zeros(4, 3), nb, ratio)


# ---------------------------------------------------------------------------------------------------------------------------------
# PLY
# ---------------------------------------------------------------------------------------------------------------------------------
def test_vertex_only_ply_layout(tmp_path):
    pts = torch.tensor([[0.5, -1.0, 2.0], [3.0, 4.0, -5.5]])
    cols = torch.tensor([[0.0, 0.5, 1.2], [1.0, 0.2, -0.1]])
    pointcloud.PointCloud(pts, cols).export(tmp_path / "a.ply")
    data = (tmp_path / "a.ply").read_bytes()
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex 2\nproperty float x\nproperty float y\nproperty float z\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\nproperty uchar alpha\nend_header\n").encode()
    body = struct.pack("<3f4B", 0.5, -1.0, 2.0, 0, 128, 255, 255) + struct.pack("<3f4B", 3.0, 4.0, -5.5, 255, 51, 0, 255)
    assert data == header + body
    v, f, n = meshing.read_ply(str(tmp_path / "a.ply"))
    np.testing.assert_array_equal(v, pts.numpy())
    assert f.shape == (0, 3) and n is None


def test_ply_with_normals_round_trip(tmp_path):
    g = torch.Generator().manual_seed(3)
    pts, nrm, cols = torch.randn(50, 3, generator=g), torch.randn(50, 3, generator=g), torch.rand(50, 3, generator=g)
    pointcloud.PointCloud(pts, cols, nrm).export(tmp_path / "b.ply")
    v, f, n = meshing.read_ply(str(tmp_path / "b.ply"))
    np.testing.assert_array_equal(v, pts.numpy())
    np.testing.assert_array_equal(n, nrm.numpy())
    assert len(f) == 0


def test_mesh_ply_bytes_unchanged(tmp_path):
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    nrm = np.array([[0, 0, 1]] * 3, np.float32)
    faces = np.array([[0, 1, 2]])
    meshing.write_ply(str(tmp_path / "m.ply"), v, faces, nrm)
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex 3\n" +
              "".join(f"property float {c}\n" for c in ("x", "y", "z", "nx", "ny", "nz")) +
              "element face 1\nproperty list uchar int vertex_indices\nend_header\n").encode()
    body = b"".join(struct.pack("<6f", *v[i], *nrm[i]) for i in range(3)) + struct.pack("<B3i", 3, 0, 1, 2)
    assert (tmp_path / "m.ply").read_bytes() == header + body
