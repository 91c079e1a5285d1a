"""CPU restatement of the neus-acc occupancy path (NeuSAccSampler, model_components/ray_samplers.py:1315-1503, and the nerfacc 0.3.5
functions neus_acc.py calls), the oracle of csrc/occupancy.cu and the packed kernels of csrc/render.cu:

* ``lattice``  -- the voxel centres, with the reference's own torch.linspace / meshgrid (:1361-1376).
* ``prune``    -- update_binary_grid's alpha test (:1405-1426) in the reference's torch fp32 expressions.
* ``march``    -- nerfacc.cuda.ray_marching for the AABB contraction with cone_angle = 0, in numpy float32, vectorised over rays.  numpy
                  float32 arithmetic is IEEE round-to-nearest without contraction, so it reproduces the kernel bit for bit; np.fmin /
                  np.fmax give fminf / fmaxf's NaN rules.  nerfacc itself is compiled with FMA contraction, so its t values may differ
                  from this restatement in the last bit: the march is checked against this file only (parity-unpinned, DESIGN §4).
                  Like the kernel it stops a ray once a step no longer advances t, where nerfacc would loop forever, and after
                  MAX_ITERS loop iterations.
* ``packed_weights64`` / ``accumulate64`` -- render_weight_from_alpha and accumulate_along_rays in float64.
"""
import numpy as np
import torch

MAX_ITERS = 1 << 26   # csrc/occupancy.cu kMarchMaxIters


def lattice(aabb: torch.Tensor, resolution: int) -> torch.Tensor:
    voxel_size = (aabb[1, 0] - aabb[0, 0]) / resolution
    offs = [torch.linspace(aabb[0, i] + voxel_size / 2.0, aabb[1, i] - voxel_size / 2.0, resolution) for i in range(3)]
    x, y, z = torch.meshgrid(*offs, indexing="ij")
    return torch.stack([x, y, z], dim=-1).reshape(-1, 3)


def prune_alpha(sdf: torch.Tensor, voxel_size: torch.Tensor, step_size: float, inv_s: torch.Tensor) -> torch.Tensor:
    """alpha of the occupied voxels' centres (fp32 like the reference; pass float64 tensors for the exact value)."""
    bound = voxel_size * (3**0.5) / 2.0
    sdf = sdf.abs()
    sdf = torch.maximum(sdf - bound, torch.zeros_like(sdf))
    prev_cdf = torch.sigmoid((sdf + step_size * 0.5) * inv_s)
    next_cdf = torch.sigmoid((sdf - step_size * 0.5) * inv_s)
    p = prev_cdf - next_cdf
    return ((p + 1e-5) / (prev_cdf + 1e-5)).clip(0.0, 1.0)


def prune(binary: torch.Tensor, sdf: torch.Tensor, voxel_size: torch.Tensor, step_size: float, inv_s: torch.Tensor,
          alpha_thres: float = 0.001) -> torch.Tensor:
    """New binary grid: the occupied voxels (in flat order, `sdf` evaluated at their centres) whose alpha <= alpha_thres are cleared."""
    mask = binary.reshape(-1).clone()
    mask[mask.clone()] = prune_alpha(sdf, voxel_size, step_size, inv_s) > alpha_thres
    return mask.reshape(binary.shape)


def _f32(x):
    return np.asarray(x, dtype=np.float32)


def march(origins, directions, nears, fars, roi_aabb, binary, step_size):
    """-> (counts [R] int64, ray_indices [N] int64, t_starts [N] f32, t_ends [N] f32), samples grouped by ray in ray order."""
    o, d = _f32(origins).reshape(-1, 3), _f32(directions).reshape(-1, 3)
    near, far = _f32(nears).reshape(-1), _f32(fars).reshape(-1)
    roi = _f32(roi_aabb).reshape(6)
    lo, hi = roi[:3], roi[3:]
    ext = hi - lo
    grid = np.asarray(binary, dtype=bool).reshape(-1)
    res = int(round(grid.size ** (1 / 3)))
    assert res**3 == grid.size
    res_f = np.float32(res)
    dt = np.float32(step_size)
    half = dt * np.float32(0.5)
    R = o.shape[0]
    with np.errstate(all="ignore"):
        inv_d = np.float32(1.0) / d
        sgn = np.copysign(np.float32(1.0), d)
        t0 = near.copy()
        t1 = t0 + dt
        t_mid = (t0 + t1) * np.float32(0.5)
        alive = t1 > t0
        iters = np.zeros(R, np.int64)
        count = np.zeros(R, np.int64)
        rec_r, rec_t0, rec_t1 = [], [], []
        while True:
            a = np.nonzero(alive & (t_mid < far))[0]
            if a.size == 0:
                break
            x = o[a] + t_mid[a, None] * d[a]
            inside = ~((x < lo) | (x > hi)).any(axis=1)
            u = ((x - lo) / ext) * res_f
            vi = np.clip(np.trunc(np.where(inside[:, None], u, 0)), 0, res - 1).astype(np.int64)
            occ = inside & grid[(vi[:, 0] * res + vi[:, 1]) * res + vi[:, 2]]
            oc = a[occ]
            rec_r.append(oc), rec_t0.append(t0[oc].copy()), rec_t1.append(t1[oc].copy())
            count[oc] += 1
            t0[oc] = t1[oc]
            t1[oc] = t0[oc] + dt
            t_mid[oc] = (t0[oc] + t1[oc]) * np.float32(0.5)
            alive[oc] = t1[oc] > t0[oc]
            # empty voxel: advance_to_next_voxel
            em = ~occ
            e = a[em]
            ue = u[em]
            edge = np.floor((ue + np.float32(0.5)) + np.float32(0.5) * sgn[e])
            tc = (((edge - ue) * inv_d[e]) / res_f) * ext
            dist = np.fmax(np.fmin(np.fmin(tc[:, 0], tc[:, 1]), tc[:, 2]), np.float32(0.0))
            target = t_mid[e] + dist
            t = t_mid[e].copy()
            stepping = np.ones(e.size, bool)
            while stepping.any():
                k = np.nonzero(stepping)[0]
                nt = t[k] + dt
                stuck = ~(nt > t[k])
                alive[e[k[stuck]]] = False
                go = k[~stuck]
                t[go] = nt[~stuck]
                iters[e[go]] += 1
                stepping[k[stuck]] = False
                stepping[go] = (t[go] < target[go]) & (iters[e[go]] < MAX_ITERS)
            t_mid[e] = t
            t0[e] = t - half
            t1[e] = t + half
            alive[e] &= t1[e] > t0[e]
            iters[a] += 1
            alive[a] &= iters[a] < MAX_ITERS
    rr = np.concatenate(rec_r) if rec_r else np.zeros(0, np.int64)
    order = np.argsort(rr, kind="stable")
    ts = np.concatenate(rec_t0)[order] if rec_r else np.zeros(0, np.float32)
    te = np.concatenate(rec_t1)[order] if rec_r else np.zeros(0, np.float32)
    return count, rr[order].astype(np.int64), ts.astype(np.float32), te.astype(np.float32)


def march_scalar(o, d, near, far, roi_aabb, binary, step_size, max_iters=MAX_ITERS):
    """The same loop for one ray, written as nerfacc's scalar C++ with numpy float32 scalars: the cross-check of ``march``."""
    f = np.float32
    grid = np.asarray(binary, dtype=bool).reshape(-1)
    res = int(round(grid.size ** (1 / 3)))
    roi = _f32(roi_aabb).reshape(6)
    lo, hi = roi[:3], roi[3:]
    ext = [hi[c] - lo[c] for c in range(3)]
    o, d = [f(v) for v in o], [f(v) for v in d]
    dt, res_f = f(step_size), f(res)
    out = []
    with np.errstate(all="ignore"):
        inv_d = [f(1.0) / d[c] for c in range(3)]
        t0 = f(near)
        t1 = t0 + dt
        t_mid = (t0 + t1) * f(0.5)
        alive, iters = bool(t1 > t0), 0
        while alive and t_mid < f(far):
            x = [o[c] + t_mid * d[c] for c in range(3)]
            u = [((x[c] - lo[c]) / ext[c]) * res_f for c in range(3)]
            inside = all(not (x[c] < lo[c] or x[c] > hi[c]) for c in range(3))
            occupied = False
            if inside:
                iv = [min(max(int(u[c]), 0), res - 1) for c in range(3)]
                occupied = bool(grid[(iv[0] * res + iv[1]) * res + iv[2]])
            if occupied:
                out.append((t0, t1))
                t0 = t1
                t1 = t0 + dt
                t_mid = (t0 + t1) * f(0.5)
                alive = bool(t1 > t0)
            else:
                tc = [(((np.floor((u[c] + f(0.5)) + f(0.5) * np.copysign(f(1.0), d[c])) - u[c]) * inv_d[c]) / res_f) * ext[c] for c in range(3)]
                dist = np.fmax(np.fmin(np.fmin(tc[0], tc[1]), tc[2]), f(0.0))
                target = t_mid + dist
                t = t_mid
                while True:
                    nt = t + dt
                    if not nt > t:
                        alive = False
                        break
                    t = nt
                    iters += 1
                    if not (t < target and iters < max_iters):
                        break
                t_mid = t
                t0 = t_mid - dt * f(0.5)
                t1 = t_mid + dt * f(0.5)
                alive = alive and bool(t1 > t0)
            iters += 1
            if iters >= max_iters:
                alive = False
    return out


def offsets_of(counts) -> np.ndarray:
    return np.concatenate([[0], np.cumsum(np.asarray(counts, dtype=np.int64))])


def packed_weights64(alphas: torch.Tensor, offsets) -> torch.Tensor:
    """w = alpha * exclusive prod (1 - alpha) per segment, float64 (differentiable)."""
    a = alphas.reshape(-1).double()
    parts = []
    for r in range(len(offsets) - 1):
        seg = a[int(offsets[r]): int(offsets[r + 1])]
        if seg.numel() == 0:
            continue
        T = torch.cat([seg.new_ones(1), torch.cumprod(1.0 - seg, 0)[:-1]])
        parts.append(seg * T)
    return torch.cat(parts) if parts else a.new_zeros(0)


def accumulate64(weights: torch.Tensor, ray_indices: torch.Tensor, values=None, n_rays: int = None) -> torch.Tensor:
    w = weights.reshape(-1, 1).double()
    src = w * values.double() if values is not None else w
    out = torch.zeros(n_rays, src.shape[1], dtype=torch.float64)
    return out.index_add(0, ray_indices.reshape(-1).long(), src)
