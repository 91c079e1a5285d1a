"""neus-acc on the CPU: the oracle (oracle/occupancy.py) and the host side of sdfstudio_b200.NeuSAccSampler against the golden minted
from the unmodified reference NeuSAccSampler (oracle/make_golden_neus_acc.py), and the oracle march against a scalar loop."""
import inspect
import json
import os

import numpy as np
import pytest
import torch

from oracle import occupancy

from helpers import GOLDEN_DIR, load_golden


def _meta():
    with open(os.path.join(GOLDEN_DIR, "neus_acc.json")) as fh:
        return json.load(fh)


def _sampler():
    import sdfstudio_b200 as sb

    m = _meta()
    return sb.NeuSAccSampler(aabb=torch.tensor(m["aabb"]), neus_sampler=None, resolution=m["resolution"])


def test_oracle_lattice_and_prune_match_reference_bitwise():
    g, m = load_golden("neus_acc"), _meta()
    assert torch.equal(occupancy.lattice(torch.tensor(m["aabb"]), m["resolution"]), g["cube_coordinate"])
    vs = g["voxel_size"][0]
    b1 = occupancy.prune(g["binary0"], g["sdf1"], vs, float(g["step_size1"][0]), g["inv_s"][:1])
    assert torch.equal(b1, g["binary1"])
    b2 = occupancy.prune(b1, g["sdf2"], vs, float(g["step_size2"][0]), g["inv_s"][1:])
    assert torch.equal(b2, g["binary2"])
    assert 0 < int(b2.sum()) < int(b1.sum()) < b1.numel()
    assert float(g["step_size1"][0]) == 14.0 / float(g["inv_s"][0]) / 16


def test_mirror_signature_state_dict_and_ray_samples_match_reference():
    import sdfstudio_b200 as sb

    g, m = load_golden("neus_acc"), _meta()
    sig = [[n, None if p.default is inspect.Parameter.empty else p.default] for n, p in inspect.signature(sb.NeuSAccSampler.__init__).parameters.items()
           if n != "self"]
    assert sig == m["signature"]
    s = _sampler()
    spec = {k: [list(v.shape), str(v.dtype)] for k, v in s.state_dict().items()}
    assert spec == m["state_dict"]
    assert torch.equal(s.cube_coordinate, g["cube_coordinate"])
    assert torch.equal(s._binary, torch.ones_like(g["binary0"]))
    rb = sb.RayBundle(origins=g["cr_origins"], directions=g["cr_directions"], pixel_area=g["cr_pixel_area"], camera_indices=g["cr_camera_indices"])
    rs = s.create_ray_samples_from_ray_indices(rb, g["cr_ray_indices"], g["cr_t_starts"], g["cr_t_ends"])
    for name, got in (("origins", rs.frustums.origins), ("directions", rs.frustums.directions), ("starts", rs.frustums.starts),
                      ("ends", rs.frustums.ends), ("pixel_area", rs.frustums.pixel_area), ("camera_indices", rs.camera_indices),
                      ("deltas", rs.deltas)):
        assert torch.equal(got, g["cr_out_" + name]), name
    s.update_step_size(0, inv_s=lambda: g["inv_s"][:1])
    assert s.step_size == float(g["step_size1"][0])
    s.update_binary_grid(1000, sdf_fn=lambda x: x[:, 0], inv_s=lambda: g["inv_s"][:1])   # warm-up: no work, no device needed
    assert int(s._update_counter) == 0


def test_unsupported_inputs_are_rejected():
    import sdfstudio_b200 as sb

    with pytest.raises(NotImplementedError, match="ray_resampling"):
        sb.NeuSAccSampler(aabb=torch.tensor([[-1.0] * 3, [1.0] * 3]), importance_sampling=True)
    with pytest.raises(AssertionError):
        sb.NeuSAccSampler(aabb=torch.tensor([[-1.0, -1.0, -2.0], [1.0, 1.0, 1.0]]))
    ri = torch.tensor([0, 0, 2, 1])
    with pytest.raises(ValueError, match="non-decreasing"):
        sb.packed.accumulate_along_rays(torch.ones(4, 1), ri, n_rays=3)
    with pytest.raises(ValueError, match="non-decreasing"):
        sb.packed.render_weight_from_alpha(torch.ones(4, 1), ray_indices=ri, n_rays=3)
    with pytest.raises(ValueError, match="non-decreasing"):
        sb.packed.accumulate_along_rays(torch.ones(4, 1), torch.tensor([0, 1, 2, 3]), n_rays=3)   # index out of range


def test_segment_offsets():
    from sdfstudio_b200 import packed

    ri = torch.tensor([0, 0, 2, 2, 2, 4])
    assert packed.segment_offsets(ri, 6).tolist() == [0, 2, 2, 5, 5, 6, 6]
    assert packed.segment_offsets(torch.zeros(0, dtype=torch.int64), 2).tolist() == [0, 0, 0]


def _sphere_grid(res, radius=0.5, shell=0.15):
    c = (np.arange(res) + 0.5) / res * 2 - 1
    x, y, z = np.meshgrid(c, c, c, indexing="ij")
    r = np.sqrt(x * x + y * y + z * z)
    return np.abs(r - radius) < shell


def test_oracle_march_matches_scalar_loop():
    res = 16
    grid = _sphere_grid(res)
    roi = [-1.0, -1.0, -1.0, 1.0, 1.0, 1.0]
    g = torch.Generator().manual_seed(3)
    o = (torch.randn(6, 3, generator=g) * 0.3 + torch.tensor([0.0, 0.0, -2.0])).numpy()
    d = torch.nn.functional.normalize(torch.tensor([0.0, 0.0, 1.0]) + 0.3 * torch.randn(6, 3, generator=g), dim=-1).numpy()
    d[0] = [0.0, 0.0, 1.0]   # axis-aligned: 0 * inf in the voxel skip
    near, far = np.full(6, 0.5, np.float32), np.full(6, 3.5, np.float32)
    near[5], far[5] = 3.0, 1.0   # near > far
    step = 0.01
    counts, ri, ts, te = occupancy.march(o, d, near, far, roi, grid, step)
    off = occupancy.offsets_of(counts)
    assert counts[5] == 0 and counts[0] > 0 and counts.sum() > 0
    for r in range(6):
        ref = occupancy.march_scalar(o[r], d[r], near[r], far[r], roi, grid, step)
        assert counts[r] == len(ref)
        assert np.all(ri[off[r]: off[r + 1]] == r)
        got = list(zip(ts[off[r]: off[r + 1]].tolist(), te[off[r]: off[r + 1]].tolist()))
        assert got == [(float(a), float(b)) for a, b in ref]


def test_oracle_march_terminates_on_absorbing_ray():
    # just below 2^15 a 1e-3 step still rounds t up by one ulp; from 2^15 on it is absorbed (t + dt == t), where nerfacc's loop would
    # never end
    grid = np.ones((4, 4, 4), bool)
    roi = [-1e9, -1e9, -1e9, 1e9, 1e9, 1e9]
    o, d = np.zeros((1, 3)), np.array([[1.0, 0.0, 0.0]])
    counts, ri, ts, te = occupancy.march(o, d, [32767.5], [1e8], roi, grid, 1e-3)
    assert 100 < counts[0] < 1000
    assert np.all(te > ts) and float(te[-1]) <= 32768.0
    ref = occupancy.march_scalar(o[0], d[0], 32767.5, 1e8, roi, grid, 1e-3)
    assert list(zip(ts.tolist(), te.tolist())) == [(float(a), float(b)) for a, b in ref]
