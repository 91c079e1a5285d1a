"""TEST INFRASTRUCTURE -- mints tests/golden/neus_acc.npz + neus_acc.json from the UNMODIFIED reference NeuSAccSampler
(model_components/ray_samplers.py:1315-1503) on CPU (run in the build container only):

* the constructor signature, the state-dict names / shapes / dtypes and ``cube_coordinate``;
* ``_binary`` / ``_update_counter`` / ``step_size`` along a seeded sequence of update_step_size / update_binary_grid calls (warm-up no-op,
  update, off-period no-op, second update) on a seeded analytic sdf, with the sdf values each update evaluated;
* ``create_ray_samples_from_ray_indices`` on given indices.

nerfacc is absent here; the sampler only reads ``roi_aabb`` from nerfacc.OccupancyGrid, so a minimal module holding it stands in.

    python -m oracle.make_golden_neus_acc
"""
import inspect
import json
import os
import sys
import warnings

import numpy as np
import torch

from . import ref_import

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
AABB = [[-1.2, -1.2, -1.2], [1.2, 1.2, 1.2]]
RESOLUTION = 16
INV_S = (50.0, 200.0)


def analytic_sdf(seed: int = 0):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(3, 3, generator=g) * 3.0
    b = torch.rand(3, generator=g) * 6.0

    def sdf(x):
        return x.norm(dim=-1) - 0.6 + 0.05 * torch.sin(x @ a.t() + b).sum(-1)

    return sdf


def main():
    ref_import.install_shims()
    warnings.simplefilter("ignore")

    class _OccupancyGrid(torch.nn.Module):
        def __init__(self, roi_aabb, resolution=128, contraction_type=None):
            super().__init__()
            self.roi_aabb = roi_aabb

    sys.modules["nerfacc"].OccupancyGrid = _OccupancyGrid
    from nerfstudio.cameras.rays import RayBundle
    from nerfstudio.model_components.ray_samplers import NeuSAccSampler

    sig = [[n, None if p.default is inspect.Parameter.empty else p.default] for n, p in inspect.signature(NeuSAccSampler.__init__).parameters.items()
           if n != "self"]
    s = NeuSAccSampler(aabb=torch.tensor(AABB), neus_sampler=None, resolution=RESOLUTION)
    spec = {k: [list(v.shape), str(v.dtype)] for k, v in s.state_dict().items()}
    out = {"cube_coordinate": s.cube_coordinate.clone(), "voxel_size": s.voxel_size.reshape(1).clone()}

    base = analytic_sdf(0)
    seen = []

    def sdf_fn(x):
        v = base(x)
        seen.append(v.clone())
        return v

    inv1 = lambda: torch.tensor([INV_S[0]])  # noqa: E731
    inv2 = lambda: torch.tensor([INV_S[1]])  # noqa: E731
    log = []
    s.update_step_size(0, inv_s=inv1)
    log.append(("step_size", 0, s.step_size))
    s.update_binary_grid(1000, sdf_fn=sdf_fn, inv_s=inv1)          # warm-up: no-op
    assert not seen and int(s._update_counter) == 0
    out["binary0"] = s._binary.clone()
    out["step_size1"] = torch.tensor([s.step_size], dtype=torch.float64)
    s.update_binary_grid(2000, sdf_fn=sdf_fn, inv_s=inv1)          # update 1
    out["sdf1"], out["binary1"], out["counter1"] = torch.cat(seen), s._binary.clone(), s._update_counter.clone()
    seen.clear()
    s.update_binary_grid(2500, sdf_fn=sdf_fn, inv_s=inv1)          # off period: no-op
    assert not seen and torch.equal(s._binary, out["binary1"])
    s.update_step_size(2500, inv_s=inv2)
    out["step_size2"] = torch.tensor([s.step_size], dtype=torch.float64)
    s.update_binary_grid(3000, sdf_fn=sdf_fn, inv_s=inv2)          # update 2
    out["sdf2"], out["binary2"], out["counter2"] = torch.cat(seen), s._binary.clone(), s._update_counter.clone()
    out["inv_s"] = torch.tensor(INV_S, dtype=torch.float32)

    # create_ray_samples_from_ray_indices on given (sorted) indices
    g = torch.Generator().manual_seed(1)
    R = 12
    rb = RayBundle(origins=torch.randn(R, 3, generator=g), directions=torch.randn(R, 3, generator=g), pixel_area=torch.rand(R, 1, generator=g),
                   camera_indices=torch.randint(0, 49, (R, 1), generator=g))
    ri = torch.sort(torch.randint(0, R, (40,), generator=g)).values
    ts = torch.rand(40, 1, generator=g) * 3
    te = ts + torch.rand(40, 1, generator=g) * 0.01
    rs = s.create_ray_samples_from_ray_indices(rb, ri, ts, te)
    out.update({"cr_origins": rb.origins, "cr_directions": rb.directions, "cr_pixel_area": rb.pixel_area, "cr_camera_indices": rb.camera_indices,
                "cr_ray_indices": ri, "cr_t_starts": ts, "cr_t_ends": te, "cr_out_origins": rs.frustums.origins,
                "cr_out_directions": rs.frustums.directions, "cr_out_starts": rs.frustums.starts, "cr_out_ends": rs.frustums.ends,
                "cr_out_pixel_area": rs.frustums.pixel_area, "cr_out_camera_indices": rs.camera_indices, "cr_out_deltas": rs.deltas})
    np.savez_compressed(os.path.join(GOLDEN_DIR, "neus_acc.npz"), **{k: v.detach().cpu().numpy() for k, v in out.items()})
    meta = {"signature": sig, "state_dict": spec, "aabb": AABB, "resolution": RESOLUTION, "log": log}
    with open(os.path.join(GOLDEN_DIR, "neus_acc.json"), "w") as fh:
        json.dump(meta, fh, indent=1)
    print("wrote", GOLDEN_DIR, {k: tuple(v.shape) for k, v in out.items()}, int(out["binary1"].sum()), int(out["binary2"].sum()))


if __name__ == "__main__":
    main()
