"""GPU checks of the point-cloud exporter: sdfb200_knn against restatement (b) bit for bit on clouds that stress an exact grid search
(surfaces, clusters with far outliers, lattice ties, duplicates, flat and collinear clouds, tiny clouds), N k past 2^31, the refusals,
determinism and shuffles, the outlier removal against (c), the normals against numpy's eigh, and the export flows against (a)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import pointcloud as opc

pytestmark = pytest.mark.gpu

KS = [1, 20, 30, 32]


@pytest.fixture(autouse=True)
def _keep_global_rng():
    """Every test here restores the global CPU and CUDA generators, so that the tests after this file draw what they would draw
    without it (some seed the global generator, e.g. through ``test_gpu_meshing._field``)."""
    with torch.random.fork_rng(devices=range(torch.cuda.device_count())):
        yield


def _cloud(name: str) -> np.ndarray:
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "cube":
        p = rng.uniform(-1, 1, (3000, 3))
    elif name == "sphere":
        p = rng.normal(size=(3000, 3))
        p = 0.7 * p / np.linalg.norm(p, axis=1, keepdims=True)
    elif name == "clusters_outliers":
        centres = rng.uniform(-0.5, 0.5, (4, 3))
        p = np.concatenate([c + 0.01 * rng.normal(size=(700, 3)) for c in centres] + [rng.uniform(-80, 80, (6, 3))])
    elif name == "lattice":
        g = np.arange(13) * 0.125
        p = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    elif name == "copies":
        p = np.concatenate([np.full((400, 3), 0.3), rng.uniform(-1, 1, (30, 3)), np.full((50, 3), -0.2)])
    elif name == "planar":
        p = np.concatenate([rng.uniform(-1, 1, (2500, 2)), np.full((2500, 1), 0.25)], axis=1)
    elif name == "collinear":
        p = np.stack([rng.uniform(-2, 3, 1500), np.full(1500, -0.5), np.full(1500, 0.75)], axis=1)
    elif name == "n5":
        p = rng.uniform(-1, 1, (5, 3))
    elif name == "n1":
        p = np.array([[0.1, 0.2, 0.3]])
    else:
        p = np.zeros((0, 3))
    return p.astype(np.float32)


CLOUDS = ["cube", "sphere", "clusters_outliers", "lattice", "copies", "planar", "collinear", "n5", "n1", "n0"]


def _knn(p, k, **kw):
    from sdfstudio_b200 import pointcloud

    return pointcloud.nearest_neighbours(torch.from_numpy(p).cuda(), k, **kw)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("name", CLOUDS)
def test_knn_matches_restatement(name, k):
    p = _cloud(name)
    mean, idx = _knn(p, k)
    ref_mean, ref_idx = opc.knn(p, k)
    np.testing.assert_array_equal(idx.cpu().numpy(), ref_idx)
    assert np.array_equal(mean.cpu().numpy().view(np.int64), ref_mean.view(np.int64))


def test_knn_only_one_output():
    p = _cloud("sphere")
    mean, idx = _knn(p, 20, neighbours=False)
    assert idx is None and torch.equal(mean, _knn(p, 20)[0])
    mean, idx = _knn(p, 20, mean_distances=False)
    assert mean is None and torch.equal(idx, _knn(p, 20)[1])


def test_knn_offsets_past_2_31():
    """N k just past 2^31 int32 entries: the rows at the end of the index output are right (checked by brute force on the GPU)."""
    k = 32
    n = 2**31 // k + 1
    g = torch.Generator(device="cuda").manual_seed(5)
    pts = torch.rand(n, 3, generator=g, device="cuda") * 2 - 1
    _, idx = _knn_t(pts, k)
    assert idx.shape == (n, k)
    p64 = pts.double()
    for r in (0, n // 2, n - 2, n - 1):
        d = p64 - p64[r]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        order = torch.sort(d2, stable=True).indices[:k]
        assert torch.equal(idx[r].long(), order), r


def _knn_t(pts, k):
    from sdfstudio_b200 import pointcloud

    return pointcloud.nearest_neighbours(pts, k, mean_distances=False)


def test_refusals_launch_nothing():
    from sdfstudio_b200 import _lib

    lib = _lib.load()
    p = torch.rand(100, 3, generator=torch.Generator(device="cuda").manual_seed(0), device="cuda")
    order = torch.arange(100, dtype=torch.int32, device="cuda")
    cs = torch.tensor([0, 100], dtype=torch.int32, device="cuda")
    mean = torch.full((100,), -7.0, dtype=torch.float64, device="cuda")
    idx = torch.full((100, 33), -7, dtype=torch.int32, device="cuda")
    box = (C.c_float * 6)(0, 0, 0, 1, 1, 1)
    nan_box = (C.c_float * 6)(0, float("nan"), 0, 1, 1, 1)
    s = _lib.stream_ptr()
    torch.cuda.synchronize()
    before = _lib.launch_count()
    calls = [
        (_lib.ptr(p), _lib.ptr(order), 100, _lib.ptr(cs), box, 1, 0, _lib.ptr(mean), _lib.ptr(idx), s),
        (_lib.ptr(p), _lib.ptr(order), 100, _lib.ptr(cs), box, 1, 33, _lib.ptr(mean), _lib.ptr(idx), s),
        (_lib.ptr(p), _lib.ptr(order), 100, _lib.ptr(cs), nan_box, 1, 20, _lib.ptr(mean), _lib.ptr(idx), s),
        (None, _lib.ptr(order), 100, _lib.ptr(cs), box, 1, 20, _lib.ptr(mean), _lib.ptr(idx), s),
        (_lib.ptr(p), _lib.ptr(order), 100, None, box, 1, 20, _lib.ptr(mean), _lib.ptr(idx), s),
        (_lib.ptr(p), _lib.ptr(order), 100, _lib.ptr(cs), box, 1, 20, None, None, s),
    ]
    for args in calls:
        assert lib.sdfb200_knn(*args) == -1
    assert lib.sdfb200_point_normals(_lib.ptr(p), 100, _lib.ptr(idx), 0, _lib.ptr(p), s) == -1
    assert lib.sdfb200_point_normals(_lib.ptr(p), 100, None, 20, _lib.ptr(p), s) == -1
    torch.cuda.synchronize()
    assert _lib.launch_count() == before
    assert (mean == -7).all() and (idx == -7).all()
    bad = torch.from_numpy(_cloud("cube")).cuda()
    bad[17, 1] = float("nan")
    with pytest.raises(ValueError):
        _knn_t(bad, 20)
    for k in (0, 33):
        with pytest.raises(ValueError):
            _knn_t(bad, k)


@pytest.mark.parametrize("name", ["sphere", "lattice", "copies"])
def test_reruns_and_shuffles(name):
    p = _cloud(name)
    mean, idx = _knn(p, 20)
    mean2, idx2 = _knn(p, 20)
    assert torch.equal(mean, mean2) and torch.equal(idx, idx2)
    perm = np.random.default_rng(3).permutation(len(p))
    inv = np.argsort(perm)
    smean, sidx = _knn(p[perm], 20)
    smean, sidx = smean.cpu().numpy(), sidx.cpu().numpy()
    assert np.array_equal(smean[inv].view(np.int64), mean.cpu().numpy().view(np.int64))
    # the list of a point, mapped back to original indices, may differ only among candidates tied at one distance
    p64 = p.astype(np.float64)
    idx = idx.cpu().numpy()
    for i in range(len(p)):
        a, b = idx[i], perm[sidx[inv[i]]]
        if np.array_equal(a, b):
            continue
        d = p64[a] - p64[i]
        e = p64[b] - p64[i]
        da = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        db = (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2]
        assert np.array_equal(da, db), i                            # same distance at every rank, so only tied entries differ


# relative distance to the threshold within which the package's torch sums and (c)'s numpy sums may decide a point differently
THRESHOLD_MARGIN = 1e-12


@pytest.mark.parametrize("name,ratio", [("sphere", 1.0), ("clusters_outliers", 2.0), ("cube", 0.5), ("copies", 1.0), ("lattice", 1.0),
                                        ("n5", 1.0), ("n1", 1.0), ("n0", 1.0)])
def test_outlier_removal_matches_restatement(name, ratio):
    from sdfstudio_b200 import pointcloud

    p = _cloud(name)
    kept, mean = pointcloud.remove_statistical_outlier(torch.from_numpy(p).cuda(), 20, ratio)
    ref_mean, _ = opc.knn(p, 20)
    ref_kept, thr = opc.statistical_outliers(ref_mean, ratio)
    assert np.array_equal(mean.cpu().numpy().view(np.int64), ref_mean.view(np.int64))
    near = np.isfinite(thr) & (np.abs(ref_mean - thr) <= THRESHOLD_MARGIN * abs(thr))
    assert near.sum() == 0
    np.testing.assert_array_equal(kept.cpu().numpy(), ref_kept)
    if name == "clusters_outliers":
        assert not np.isin(np.arange(len(p) - 6, len(p)), ref_kept).any()   # the far outliers go


@pytest.mark.parametrize("name", ["sphere", "cube", "planar", "clusters_outliers", "lattice"])
def test_normals_against_eigh(name):
    from sdfstudio_b200 import pointcloud

    p = _cloud(name)
    nrm = pointcloud.estimate_normals(torch.from_numpy(p).cuda()).cpu().numpy().astype(np.float64)
    _, idx = opc.knn(p, 30)
    cov = opc.covariances(p, idx)
    w, v = np.linalg.eigh(cov)
    ref = v[:, :, 0]
    # bound of the estimate_normals docstring: c u ||C|| / gap with c = 64, plus the fp32 rounding of the output
    scale = np.linalg.norm(cov, axis=(1, 2))
    gap = w[:, 1] - w[:, 0]
    bound = 64 * 2.0**-53 * scale / np.maximum(gap, 1e-300) + 4 * 2.0**-24
    zero = (cov == 0).all(axis=(1, 2))
    # the sine of the angle, from the component of the unit normal perpendicular to eigh's vector (not sqrt(1 - cos^2), which would
    # turn the fp32 rounding of the output into an error of its square root)
    u = nrm / np.maximum(np.linalg.norm(nrm, axis=1, keepdims=True), 1e-300)
    sin = np.linalg.norm(u - (u * ref).sum(1, keepdims=True) * ref, axis=1)
    ok = zero | (sin <= bound) | (bound >= 1)
    assert ok.all(), (name, np.flatnonzero(~ok)[:5], sin[~ok][:5], bound[~ok][:5])
    assert np.allclose(np.linalg.norm(nrm[~zero], axis=1), 1, atol=1e-6)
    big = np.abs(nrm).argmax(1)
    assert (nrm[np.arange(len(nrm)), big] > 0).all()                        # the sign rule
    assert (nrm[zero] == [0, 0, 1]).all()


def test_normals_zero_covariance():
    from sdfstudio_b200 import pointcloud

    p = torch.full((40, 3), 0.5, device="cuda")
    assert (pointcloud.estimate_normals(p) == torch.tensor([0.0, 0.0, 1.0], device="cuda")).all()


def _remove_c(record):
    def remove(pts, nb, ratio):
        record["args"] = (nb, ratio)
        return opc.statistical_outliers(opc.knn(pts, nb)[0], ratio)[0]

    return remove


@pytest.mark.parametrize("kw", [dict(num_points=1500, normal_output_name="normal"), dict(num_points=700, std_ratio=2.5),
                                dict(num_points=1200, use_bounding_box=False, remove_outliers=False)])
def test_generate_point_cloud_matches_restatement(kw):
    from sdfstudio_b200 import pointcloud

    pipe = opc.FakePipeline(n=1000, seed=1, miss_every=3, device="cuda")
    cloud = pointcloud.generate_point_cloud(pipe, **kw)
    ref = opc.reference_flow(opc.FakePipeline(n=1000, seed=1, miss_every=3), _remove_c({}), None, **kw)
    assert pipe.datamanager.calls == ref["batches"]
    np.testing.assert_array_equal(cloud.points.cpu().numpy(), ref["points"])
    np.testing.assert_array_equal(cloud.colors.cpu().numpy(), ref["colors"])
    if ref["normals"] is None:
        assert cloud.normals is None
    else:
        np.testing.assert_array_equal(cloud.normals.cpu().numpy(), ref["normals"])


def test_generate_point_cloud_errors():
    from sdfstudio_b200 import pointcloud

    with pytest.raises(ValueError, match="rgb_output_name"):
        pointcloud.generate_point_cloud(opc.FakePipeline(n=100, device="cuda"), rgb_output_name="colour")
    pipe = opc.FakePipeline(n=400, seed=9, device="cuda")
    with pytest.raises(ValueError, match="Cannot estimate normals"):
        pointcloud.generate_point_cloud(pipe, num_points=300, estimate_normals=True, normal_output_name="normal")
    assert pipe.datamanager.calls == 2


def test_point_cloud_on_surface_renderer(tmp_path):
    import sdfstudio_b200 as sb
    from sdfstudio_b200 import meshing, pointcloud
    from sdfstudio_b200.cameras import Cameras
    from oracle.make_golden_tsdf import look_at, on_sphere
    from test_gpu_meshing import _field

    renderer = sb.SurfaceRenderer(_field("fp32"), sb.NeuSSampler(num_samples=32, num_samples_importance=32).eval(),
                                  collider=sb.NearFarCollider(0.05, 4.0), kind="neus").eval()
    c2w = look_at(on_sphere(6, 2.2, 3))[:, :3, :]
    cams = Cameras(c2w, 40.0, 40.0, 24.0, 20.0, 48, 40, device=torch.device("cuda"))
    kw = dict(num_points=3000, num_rays_per_batch=2048, estimate_normals=True)
    cloud = pointcloud.point_cloud(renderer, cams, tmp_path, seed=4, **kw)
    rays = pointcloud._PixelRays(cams, 2048, 4)
    ref = opc.reference_flow(pointcloud._RendererPipeline(renderer, rays), _remove_c({}), lambda pts: None, num_points=3000,
                             estimate_normals=True)
    assert len(cloud) > 1000
    np.testing.assert_array_equal(cloud.points.cpu().numpy(), ref["points"])
    np.testing.assert_array_equal(cloud.colors.cpu().numpy(), ref["colors"])
    v, f, n = meshing.read_ply(str(tmp_path / "point_cloud.ply"))
    np.testing.assert_array_equal(v, ref["points"])
    np.testing.assert_array_equal(n, cloud.normals.cpu().numpy())
    assert len(f) == 0
