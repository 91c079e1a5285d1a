"""TEST INFRASTRUCTURE -- CPU restatement of the multi-resolution hash-grid encodings (SURVEY.md section 8a rows a8, a8').

Two table layouts:

* ``torch`` layout  -- the reference's own ``HashEncoding`` (nerfstudio/field_components/encodings.py:283-403):
  every level hashed, ``scale_l = floor(min_res * g**l)``, corners = ceil/floor of ``x*scale``, table ``[L*T, F]`` with
  level offset ``l*T``.  Pinned against the reference (tests/test_oracle_pinned.py).
* ``tcnn`` layout   -- tiny-cuda-nn's HashGrid as configured at sdf_field.py:230-241 (coarse levels dense, level sizes
  rounded up to 8, ``pos = x*scale + 0.5``).  tiny-cuda-nn is not vendored in the reference: PARITY UNPINNED.
"""
import math

import numpy as np
import torch

PRIME_Y = 2654435761
PRIME_Z = 805459861


# ----------------------------------------------------------------------------------------------------------------
# torch layout (reference HashEncoding)
# ----------------------------------------------------------------------------------------------------------------
def torch_layout_scalings(num_levels: int, min_res: int, max_res: float) -> torch.Tensor:
    """Per-level scale, float32.  encodings.py:301-303 (floor of min_res * growth**level, computed in torch)."""
    levels = torch.arange(num_levels)
    growth = np.exp((np.log(max_res) - np.log(min_res)) / (num_levels - 1))
    return torch.floor(min_res * growth**levels)


def growth_factor(num_levels: int, base_res: int, max_res: float) -> float:
    """sdf_field.py:226."""
    return float(np.exp((np.log(max_res) - np.log(base_res)) / (num_levels - 1)))


def hash_index(ix, iy, iz, table_size: int):
    """Instant-NGP spatial hash.  encodings.py:338-355: int32 coords are promoted to int64 by the multiply, xor-ed,
    then ``% T``.  For non-negative coords and T a power of two this equals the low bits of the uint32 product."""
    ix = ix.to(torch.int64)
    iy = iy.to(torch.int64)
    iz = iz.to(torch.int64)
    h = torch.bitwise_xor(torch.bitwise_xor(ix * 1, iy * PRIME_Y), iz * PRIME_Z)
    return h % table_size


def encode_torch_layout(x, table, scalings, table_size: int, smoothstep: bool, return_indices: bool = False, fp32_positions: bool = False):
    """x [N,3] in [0,1] -> [N, L*F].  encodings.py:357-398 (+ smoothstep remap encodings.py:700-701).

    ``table`` is ``[L*T, F]``; ``scalings`` is the float32 per-level scale tensor.
    Blend order follows the reference: x-lerp (weight ``offset_x`` on the *ceil* corner), then y, then z.
    ``fp32_positions``: ``x*scale`` takes its fp32 value (the reference's and the kernels' rounding) with the derivative of
    ``x*scale``, so that an fp64 evaluation blends the same cell with the same offsets as the fp32 kernels.
    """
    dt = x.dtype
    L = scalings.shape[0]
    F = table.shape[1]
    scaled = x[:, None, :] * scalings.view(-1, 1).to(x.device, dt)  # [N, L, 3]
    if fp32_positions:
        scaled = scaled + ((x.detach().float()[:, None, :] * scalings.view(-1, 1).to(x.device, torch.float32)).to(dt) - scaled.detach())
    c = torch.ceil(scaled).to(torch.int32)
    f = torch.floor(scaled).to(torch.int32)
    off = scaled - f
    if smoothstep:
        off = off * off * (3.0 - 2.0 * off)
    lvl_off = (torch.arange(L, dtype=torch.int64, device=x.device) * table_size).view(1, L)

    def H(a, b, cc):
        return hash_index(a, b, cc, table_size) + lvl_off

    cx, cy, cz = c[..., 0], c[..., 1], c[..., 2]
    fx, fy, fz = f[..., 0], f[..., 1], f[..., 2]
    idx = [H(cx, cy, cz), H(cx, fy, cz), H(fx, fy, cz), H(fx, cy, cz), H(cx, cy, fz), H(cx, fy, fz), H(fx, fy, fz), H(fx, cy, fz)]
    f0, f1, f2, f3, f4, f5, f6, f7 = (table[i] for i in idx)  # each [N, L, F]
    ox, oy, oz = off[..., 0:1], off[..., 1:2], off[..., 2:3]
    f03 = f0 * ox + f3 * (1 - ox)
    f12 = f1 * ox + f2 * (1 - ox)
    f56 = f5 * ox + f6 * (1 - ox)
    f47 = f4 * ox + f7 * (1 - ox)
    f0312 = f03 * oy + f12 * (1 - oy)
    f4756 = f47 * oy + f56 * (1 - oy)
    out = f0312 * oz + f4756 * (1 - oz)
    out = out.reshape(x.shape[0], L * F)
    if return_indices:
        return out, torch.stack(idx, dim=-1)  # [N, L, 8] int64 rows of `table`
    return out


# ----------------------------------------------------------------------------------------------------------------
# tcnn layout (tiny-cuda-nn GridEncoding, "Hash" grid type) -- PARITY UNPINNED (source not in /root/reference)
# ----------------------------------------------------------------------------------------------------------------
def tcnn_grid_meta(n_levels: int, n_features: int, log2_hashmap_size: int, base_resolution: int, per_level_scale: float):
    """Level scale / resolution / parameter offsets following tiny-cuda-nn's grid.h conventions:
    scale = base * g**l - 1 (computed via exp2(l*log2(g))), resolution = ceil(scale)+1,
    params_in_level = min(res**3 rounded up to 8, 2**log2_hashmap_size); a level is dense iff res**3 <= its size."""
    T = 1 << log2_hashmap_size
    log2g = math.log2(per_level_scale)
    scales, ress, offsets, sizes, hashed = [], [], [0], [], []
    for l in range(n_levels):
        scale = float(np.float32(np.exp2(np.float32(l * log2g)) * np.float32(base_resolution) - np.float32(1.0)))
        res = int(math.ceil(scale)) + 1
        dense = res**3
        n = min(((dense + 7) // 8) * 8, T) if dense <= (1 << 62) else T
        scales.append(scale)
        ress.append(res)
        sizes.append(n)
        hashed.append(dense > n)
        offsets.append(offsets[-1] + n)
    return {"scale": scales, "res": ress, "size": sizes, "offset": offsets[:-1], "total": offsets[-1], "hashed": hashed}


def encode_tcnn_layout(x, params, meta, n_features: int, smoothstep: bool, return_indices: bool = False, fp32_positions: bool = False):
    """x [N,3] in [0,1] -> [N, L*F] (fp32 math; tcnn itself stores/returns fp16).  ``params`` is the flat table
    ``[total, F]``.  pos = x*scale + 0.5; cell = floor(pos); w = pos - cell (smoothstep: w^2(3-2w)); corner bit set ->
    cell+1 with weight w, else weight 1-w; dense index x + y*res + z*res^2, hashed index = spatial hash (uint32),
    both ``% level_size``.  Runs on ``x.device``.  ``return_indices``: also the [N, L, 8] rows of ``params`` of corner k
    (bit 0 = x, 1 = y, 2 = z set -> cell + 1).  ``fp32_positions``: ``pos`` takes its fp32 value with the derivative of
    ``x*scale``, as in ``encode_torch_layout``."""
    dt = x.dtype
    N = x.shape[0]
    L = len(meta["scale"])
    out = torch.zeros(N, L, n_features, dtype=dt, device=x.device)
    rows = torch.empty(N, L, 8, dtype=torch.int64, device=x.device) if return_indices else None
    for l in range(L):
        scale, res, size, off, hashed = (meta[k][l] for k in ("scale", "res", "size", "offset", "hashed"))
        # tiny-cuda-nn computes pos with a fused multiply-add (one rounding); emulate it through float64
        pos = (x.double() * float(scale) + 0.5).to(dt)
        if fp32_positions:
            pos = pos + ((x.detach().double() * float(scale) + 0.5).float().to(dt) - pos.detach())
        cell = torch.floor(pos)
        w = pos - cell
        cell = cell.to(torch.int64)
        if smoothstep:
            w = w * w * (3.0 - 2.0 * w)
        acc = torch.zeros(N, n_features, dtype=dt, device=x.device)
        for corner in range(8):
            wt = torch.ones(N, dtype=dt, device=x.device)
            cc = []
            for d in range(3):
                if corner & (1 << d):
                    wt = wt * w[:, d]
                    cc.append(cell[:, d] + 1)
                else:
                    wt = wt * (1 - w[:, d])
                    cc.append(cell[:, d])
            if hashed:
                idx = torch.bitwise_xor(torch.bitwise_xor(cc[0] & 0xFFFFFFFF, (cc[1] * PRIME_Y) & 0xFFFFFFFF), (cc[2] * PRIME_Z) & 0xFFFFFFFF)
            else:
                idx = (cc[0] + cc[1] * res + cc[2] * res * res) & 0xFFFFFFFF
            idx = idx % size + off
            if rows is not None:
                rows[:, l, corner] = idx
            acc = acc + wt[:, None] * params[idx]
        out[:, l] = acc
    if return_indices:
        return out.reshape(N, L * n_features), rows
    return out.reshape(N, L * n_features)
