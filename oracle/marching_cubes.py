"""CPU restatement of the marching-cubes kernel (sdfstudio_b200/csrc/marching_cubes.cu) and of the three mesh-extraction functions of
the reference (nerfstudio/utils/marching_cubes.py:14-341) up to their ``measure.marching_cubes`` calls.

Cube conventions (shared with the kernel and the generated table, csrc/mc_tables.h):

* corner n = dx | dy << 1 | dz << 2; a corner is inside when ``v < level``; the cube's case has bit n set when corner n is inside;
* edge e = axis * 4 + b along ``axis`` from its owner corner, b = (offset on the lower other axis) | (offset on the higher other axis) << 1;
* face f = A * 2 + s is the face at offset s on axis A; its corners (u, v) run over the two other axes U < V.

The face rule: a face whose diagonal corners agree and whose neighbouring corners differ is ambiguous.  With a, c the values (minus the
level) of its outside diagonal pair and b, d those of its inside pair, each pair taken in face order ((0,0), (1,1)) / ((1,0), (0,1)), the
saddle value is (a c - b d) / (a + c - b - d), denominator > 0.  A saddle below 0 joins the inside corners across the face (the two
segments cut off the outside corners), otherwise the outside corners are joined.  Both cubes that share a face evaluate the same fp32
expression on the same four values, so they pair the face's cut edges the same way.  Each cube's cut edges are traced into closed loops
over its six faces and every loop is fan-triangulated from its lowest edge index.  The table entry of a cube is selected by its case and
the decider bits of its ambiguous faces (bit r = r-th ambiguous face in face order).

    python -m oracle.marching_cubes      # rewrites sdfstudio_b200/csrc/mc_tables.h
"""
import functools
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLES_H = os.path.join(ROOT, "sdfstudio_b200", "csrc", "mc_tables.h")

_OTHER = {0: (1, 2), 1: (0, 2), 2: (0, 1)}


def corner_xyz(n):
    return np.array([n & 1, (n >> 1) & 1, (n >> 2) & 1], dtype=np.float64)


def edge_index(owner: int, axis: int) -> int:
    o1, o2 = _OTHER[axis]
    return axis * 4 + ((owner >> o1) & 1) + (((owner >> o2) & 1) << 1)


def edge_corners(e: int):
    axis, b = divmod(e, 4)
    o1, o2 = _OTHER[axis]
    owner = ((b & 1) << o1) | (((b >> 1) & 1) << o2)
    return owner, owner | (1 << axis)


def face_corners(f: int):
    """corners (0,0), (1,0), (1,1), (0,1) of face f, in face coordinates (u, v) over the axes U < V other than A."""
    A, s = divmod(f, 2)
    U, V = _OTHER[A]
    return [(s << A) | (u << U) | (v << V) for u, v in ((0, 0), (1, 0), (1, 1), (0, 1))]


def face_ambiguous(case: int, f: int) -> bool:
    q00, q10, q11, q01 = (((case >> c) & 1) for c in face_corners(f))
    return q00 == q11 and q10 == q01 and q00 != q10


def ambiguous_faces(case: int):
    return [f for f in range(6) if face_ambiguous(case, f)]


def _face_segments(case: int, f: int, inside_joined: bool):
    """unoriented segments (pairs of cut edges) of face f."""
    A, _ = divmod(f, 2)
    q = face_corners(f)
    ins = [(case >> c) & 1 for c in q]
    # the face edge between cyclic neighbours q[m] and q[m+1]
    fedges = [edge_index(min(q[m], q[(m + 1) % 4]), int(np.log2(q[m] ^ q[(m + 1) % 4]))) for m in range(4)]
    cut = [fedges[m] for m in range(4) if ins[m] != ins[(m + 1) % 4]]
    if not cut:
        return []
    if len(cut) == 2:
        return [tuple(cut)]
    # ambiguous: isolate the outside corners (inside joined) or the inside corners; corner m touches face edges m-1 and m
    isolate = 0 if inside_joined else 1
    return [(fedges[(m - 1) % 4], fedges[m]) for m in range(4) if ins[m] == isolate]


def _orient(case: int, f: int, e1: int, e2: int):
    """(tail, head) such that the inside corners lie on the left of the segment seen from outside the cube."""
    A, s = divmod(f, 2)
    n = np.zeros(3)
    n[A] = 2 * s - 1
    p = sum(corner_xyz(c) for c in edge_corners(e1)) / 2
    q = sum(corner_xyz(c) for c in edge_corners(e2)) / 2
    c0, c1 = edge_corners(e1)
    inner = c0 if (case >> c0) & 1 else c1
    side = np.dot(corner_xyz(inner) - p, np.cross(n, q - p))
    assert side != 0
    return (e1, e2) if side > 0 else (e2, e1)


# Orientation of the fans relative to the traced loops, fixed once so that the right-hand normal points down the values (toward the
# inside corners): skimage's gradient_direction="descent".
_FLIP = None


@functools.lru_cache(maxsize=None)
def triangulate(case: int, bits: int):
    """triangles (tuples of 3 edge indices) of (case, decider bits), in table order."""
    amb = ambiguous_faces(case)
    assert 0 <= bits < (1 << len(amb))
    succ = {}
    for f in range(6):
        joined = f in amb and bool((bits >> amb.index(f)) & 1)
        for e1, e2 in _face_segments(case, f, joined):
            t, h = _orient(case, f, e1, e2)
            assert t not in succ, (case, bits, f)
            succ[t] = h
    assert sorted(succ) == sorted(succ.values()), (case, bits)
    loops, seen = [], set()
    for e in sorted(succ):
        if e in seen:
            continue
        loop = [e]
        seen.add(e)
        while succ[loop[-1]] != e:
            loop.append(succ[loop[-1]])
            seen.add(loop[-1])
        loops.append(loop)
    tris = []
    for loop in loops:
        for m in range(1, len(loop) - 1):
            tris.append((loop[0], loop[m + 1], loop[m]) if _flip() else (loop[0], loop[m], loop[m + 1]))
    return tuple(tris)


def _flip() -> bool:
    global _FLIP
    if _FLIP is None:
        _FLIP = False
        (a, b, c), = triangulate.__wrapped__(1, 0)
        mid = [sum(corner_xyz(x) for x in edge_corners(e)) / 2 for e in (a, b, c)]
        normal = np.cross(mid[1] - mid[0], mid[2] - mid[0])
        _FLIP = bool(np.dot(normal, corner_xyz(0) - mid[0]) < 0)       # must point toward the inside corner 0
    return _FLIP


def cut_edges(case: int):
    return sorted(e for e in range(12) if ((case >> edge_corners(e)[0]) & 1) != ((case >> edge_corners(e)[1]) & 1))


def table():
    """(entry offset per case, [(case, bits, triangles)] in entry order)."""
    offsets, entries = [], []
    for case in range(256):
        offsets.append(len(entries))
        for bits in range(1 << len(ambiguous_faces(case))):
            entries.append((case, bits, triangulate(case, bits)))
    return offsets, entries


def tables_header() -> str:
    offsets, entries = table()
    tri_start, edges = [0], []
    for _, _, tris in entries:
        for t in tris:
            edges.extend(t)
        tri_start.append(len(edges) // 3)
    amb_mask = [sum(1 << f for f in ambiguous_faces(c)) for c in range(256)]
    max_tris = max(len(t) for _, _, t in entries)

    def arr(ctype, name, vals, per_line=24):
        rows = [", ".join(str(v) for v in vals[i:i + per_line]) for i in range(0, len(vals), per_line)]
        return f"__device__ const {ctype} {name}[{len(vals)}] = {{\n  " + ",\n  ".join(rows) + "\n};\n"

    out = ["// Generated from the face rule by tables_header() of the oracle's marching_cubes module, which states the rule; running that\n"
           "// module rewrites this file.  Do not edit.\n",
           "#pragma once\n#include <stdint.h>\n\nnamespace sdfb200 {\nnamespace mc {\n\n",
           f"constexpr int kEntries = {len(entries)};\nconstexpr int kMaxTris = {max_tris};\n\n",
           "// bit f set: face f of the case is ambiguous\n", arr("uint8_t", "kAmbiguousFaces", amb_mask), "\n",
           "// first entry of each case; entry = kCaseEntry[case] + decider bits of the ambiguous faces\n", arr("uint16_t", "kCaseEntry", offsets), "\n",
           "// triangles of entry i: [kTriStart[i], kTriStart[i + 1])\n", arr("uint16_t", "kTriStart", tri_start), "\n",
           "// three edge indices per triangle\n", arr("uint8_t", "kTriEdges", edges), "\n",
           "}  // namespace mc\n}  // namespace sdfb200\n"]
    return "".join(out)


# ---------------------------------------------------------------------------------------------------------------------------------
# the kernel, restated on numpy fp32
# ---------------------------------------------------------------------------------------------------------------------------------
_F = np.float32


def _corner_offsets(ny, nz):
    return np.array([((n & 1) * ny + ((n >> 1) & 1)) * nz + ((n >> 2) & 1) for n in range(8)], dtype=np.int64)


def _gradient(flat, shape, p, axis, spacing):
    """central difference at lattice points p (one-sided at the border), divided by the spacing, fp32."""
    nx, ny, nz = shape
    stride = (ny * nz, nz, 1)[axis]
    idx = (p // stride) % shape[axis]
    n = shape[axis]
    hi = np.where(idx + 1 < n, p + stride, p)
    lo = np.where(idx > 0, p - stride, p)
    d = flat[hi] - flat[lo]
    d = np.where((idx > 0) & (idx + 1 < n), d * _F(0.5), d)
    return (d / _F(spacing[axis])).astype(_F)


def marching_cubes(volume, level=0.0, spacing=(1.0, 1.0, 1.0), mask=None, origin=(0.0, 0.0, 0.0)):
    """(verts [V,3] fp32, faces [F,3] int64, normals [V,3] fp32) in the kernel's order and arithmetic."""
    vol = np.ascontiguousarray(volume, dtype=_F)
    nx, ny, nz = vol.shape
    empty = (np.zeros((0, 3), _F), np.zeros((0, 3), np.int64), np.zeros((0, 3), _F))
    if min(nx, ny, nz) < 2:
        return empty
    lvl = _F(level)
    inside = vol < lvl
    case = np.zeros((nx - 1, ny - 1, nz - 1), np.uint8)
    for n in range(8):
        dx, dy, dz = n & 1, (n >> 1) & 1, (n >> 2) & 1
        case |= inside[dx:nx - 1 + dx, dy:ny - 1 + dy, dz:nz - 1 + dz].astype(np.uint8) << n
    active = (case != 0) & (case != 255)
    if mask is not None:
        active &= np.asarray(mask)[: nx - 1, : ny - 1, : nz - 1] != 0
    ci, cj, ck = np.nonzero(active)
    if ci.size == 0:
        return empty
    cases = case[ci, cj, ck].astype(np.int64)
    p0 = (ci.astype(np.int64) * ny + cj) * nz + ck
    flat = vol.reshape(-1)
    rel = flat[p0[:, None] + _corner_offsets(ny, nz)[None, :]] - lvl            # [C, 8] fp32
    # decider bits: bit f of `joined` set when face f is ambiguous and its saddle lies inside
    joined = np.zeros(cases.shape, np.int64)
    for f in range(6):
        q = face_corners(f)
        ins = [(cases >> c) & 1 for c in q]
        amb = (ins[0] == ins[2]) & (ins[1] == ins[3]) & (ins[0] != ins[1])
        first_out = ins[0] == 0
        a = np.where(first_out, rel[:, q[0]], rel[:, q[1]])
        c = np.where(first_out, rel[:, q[2]], rel[:, q[3]])
        b = np.where(first_out, rel[:, q[1]], rel[:, q[0]])
        d = np.where(first_out, rel[:, q[3]], rel[:, q[2]])
        with np.errstate(all="ignore"):
            s = (a * c - b * d) / (((a + c) - b) - d)
        joined |= (amb & (s < _F(0))).astype(np.int64) << f
    # compact the decider bits to the case's ambiguous faces
    bits = np.zeros_like(joined)
    rank = np.zeros_like(joined)
    for f in range(6):
        amb_f = np.array([face_ambiguous(c, f) for c in range(256)])[cases]
        bits |= np.where(amb_f, ((joined >> f) & 1) << rank, 0)
        rank += amb_f
    key = cases * 64 + bits
    ntri = np.zeros(key.shape, np.int64)
    uniq = np.unique(key)
    tri_of = {int(k): np.array(triangulate(int(k) // 64, int(k) % 64), np.int64).reshape(-1, 3) for k in uniq}
    for k, t in tri_of.items():
        ntri[key == k] = len(t)
    # vertex keys (owner point * 3 + axis) of every cut edge of every processed cube, in ascending order
    e_owner = np.array([edge_corners(e)[0] for e in range(12)])
    e_axis = np.array([e // 4 for e in range(12)])
    off = _corner_offsets(ny, nz)
    edge_key = (p0[:, None] + off[e_owner][None, :]) * 3 + e_axis[None, :]       # [C, 12]
    cutm = np.array([[e in cut_edges(c) for e in range(12)] for c in range(256)])[cases]
    vkeys = np.unique(edge_key[cutm])
    # faces, cube by cube in linear order, triangles in table order
    base = np.concatenate([[0], np.cumsum(ntri)])
    faces = np.empty((int(base[-1]), 3), np.int64)
    for k, t in tri_of.items():
        sel = np.nonzero(key == k)[0]
        if len(t) == 0:
            continue
        rows = base[sel][:, None] + np.arange(len(t))[None, :]
        faces[rows.reshape(-1)] = np.searchsorted(vkeys, edge_key[sel][:, t].reshape(-1, 3)).reshape(-1, 3)
    # vertices: t = (level - v0) / (v1 - v0) on the owner's axis, origin + spacing * (idx + t)
    vp, vax = vkeys // 3, vkeys % 3
    step = np.array([ny * nz, nz, 1], np.int64)[vax]
    v0, v1 = flat[vp], flat[vp + step]
    with np.errstate(all="ignore"):
        t = ((lvl - v0) / (v1 - v0)).astype(_F)
    idx = np.stack([vp // (ny * nz), (vp // nz) % ny, vp % nz], axis=1)
    verts = np.empty((len(vkeys), 3), _F)
    for a in range(3):
        ta = np.where(vax == a, t, _F(0))
        verts[:, a] = _F(origin[a]) + _F(spacing[a]) * (idx[:, a].astype(_F) + ta)
    # normals: corner gradients interpolated with t, negated and normalised
    g = np.empty((len(vkeys), 3), _F)
    for a in range(3):
        g0 = _gradient(flat, (nx, ny, nz), vp, a, spacing)
        g1 = _gradient(flat, (nx, ny, nz), vp + step, a, spacing)
        g[:, a] = g0 + t * (g1 - g0)
    ln = np.sqrt((g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1]) + g[:, 2] * g[:, 2]).astype(_F)
    with np.errstate(all="ignore"):
        inv = np.where(ln > 0, _F(1) / ln, _F(0)).astype(_F)
    normals = (-(g * inv[:, None])).astype(_F)
    return verts, faces, normals


if __name__ == "__main__":
    with open(TABLES_H, "w") as fh:
        fh.write(tables_header())
    print(TABLES_H)


# ---------------------------------------------------------------------------------------------------------------------------------
# the reference's three functions (utils/marching_cubes.py:14-341) on torch-CPU tensors, up to their measure.marching_cubes calls.
# `mc(volume, level, spacing, mask, offset)` receives what the reference hands to skimage (numpy), plus the offset it adds.
# ---------------------------------------------------------------------------------------------------------------------------------
def _lattice(lo, hi, n):
    """np.meshgrid(np.linspace(lo, hi, n) x3, indexing="ij") flattened, as float32 (utils/marching_cubes.py:54-59)."""
    xx, yy, zz = torch.meshgrid(*[torch.from_numpy(np.linspace(lo[a], hi[a], n)) for a in range(3)], indexing="ij")
    return torch.stack([xx, yy, zz], dim=-1).reshape(-1, 3).float()


def _evaluate(fn, points):
    return torch.cat([fn(p) for p in torch.split(points, 100000, dim=0)], dim=0)


def surface_sliding(sdf, mc, resolution=512, bounding_box_min=(-1.0, -1.0, -1.0), bounding_box_max=(1.0, 1.0, 1.0), coarse_mask=None):
    assert resolution % 512 == 0
    avg_pool_3d = torch.nn.AvgPool3d(2, stride=2)
    upsample = torch.nn.Upsample(scale_factor=2, mode="nearest")
    if coarse_mask is not None:
        coarse_mask = coarse_mask.permute(2, 1, 0)[None, None].float()
    cropN, level, N = 512, 0, resolution // 512
    xs, ys, zs = (np.linspace(bounding_box_min[a], bounding_box_max[a], N + 1) for a in range(3))
    for i in range(N):
        for j in range(N):
            for k in range(N):
                lo = (xs[i], ys[j], zs[k])
                hi = (xs[i + 1], ys[j + 1], zs[k + 1])
                points = _lattice(lo, hi, cropN).reshape(cropN, cropN, cropN, 3).permute(3, 0, 1, 2)
                current_mask = None
                if coarse_mask is not None:
                    current_mask = (torch.nn.functional.grid_sample(coarse_mask, points.permute(1, 2, 3, 0)[None]) > 0.0).numpy()[0, 0]
                pyramid = [points]
                for _ in range(3):
                    points = avg_pool_3d(points[None])[0]
                    pyramid.append(points)
                mask = None
                threshold = 2 * (hi[0] - lo[0]) / cropN * 8
                for pid, pts in enumerate(pyramid[::-1]):
                    cn = pts.shape[-1]
                    pts = pts.reshape(3, -1).permute(1, 0).contiguous()
                    if mask is None:
                        if coarse_mask is not None:
                            pts_sdf = torch.ones_like(pts[:, 1])
                            valid = torch.nn.functional.grid_sample(coarse_mask, pts[None, None, None])[0, 0, 0, 0] > 0
                            if valid.any():
                                pts_sdf[valid] = _evaluate(sdf, pts[valid].contiguous())
                        else:
                            pts_sdf = _evaluate(sdf, pts)
                    else:
                        mask = mask.reshape(-1)
                        if mask.any():
                            pts_sdf[mask] = _evaluate(sdf, pts[mask].contiguous())
                    if pid < 3:
                        mask = upsample((torch.abs(pts_sdf) < threshold).reshape(cn, cn, cn)[None, None].float()).bool()
                        pts_sdf = upsample(pts_sdf.reshape(cn, cn, cn)[None, None]).reshape(-1)
                    threshold /= 2.0
                z = pts_sdf.numpy()
                if current_mask is not None:
                    vz = z.reshape(cropN, cropN, cropN)[current_mask]
                    if vz.shape[0] <= 0 or (np.min(vz) > level or np.max(vz) < level):
                        continue
                if not (np.min(z) > level or np.max(z) < level):
                    spacing = tuple((hi[a] - lo[a]) / (cropN - 1) for a in range(3))
                    mc(z.astype(np.float32).reshape(cropN, cropN, cropN), level, spacing, current_mask, np.array(lo))


def surface_occupancy(occupancy_fn, mc, resolution=512, bounding_box_min=(-1.0, -1.0, -1.0), bounding_box_max=(1.0, 1.0, 1.0), level=0.5):
    N = resolution
    z = _evaluate(lambda p: occupancy_fn(p.contiguous()).contiguous(), _lattice(bounding_box_min, bounding_box_max, N)).numpy()
    if not (np.min(z) > level or np.max(z) < level):
        spacing = tuple((bounding_box_max[a] - bounding_box_min[a]) / (N - 1) for a in range(3))
        mc(z.reshape(N, N, N), level, spacing, None, np.array(bounding_box_min))


def surface_sliding_with_contraction(sdf, mc, resolution=512, bounding_box_min=(-1.0, -1.0, -1.0), bounding_box_max=(1.0, 1.0, 1.0),
                                     coarse_mask=None):
    max_pool_3d = torch.nn.MaxPool3d(3, stride=1, padding=1)
    cropN, level, N = 512, 0, resolution // 512
    xs, ys, zs = (np.linspace(bounding_box_min[a], bounding_box_max[a], N + 1) for a in range(3))
    for i in range(N):
        for j in range(N):
            for k in range(N):
                lo = (xs[i], ys[j], zs[k])
                hi = (xs[i + 1], ys[j + 1], zs[k + 1])
                points = _lattice(lo, hi, cropN).reshape(cropN, cropN, cropN, 3)
                current_mask = torch.nn.functional.grid_sample(coarse_mask, points[None] * 0.5)
                points = points.reshape(-1, 3)
                valid = current_mask.reshape(-1) > 0
                pts_sdf = torch.ones_like(points[..., 0]) * 100.0
                if valid.any():
                    pts_sdf[valid] = _evaluate(sdf, points[valid].contiguous())
                min_sdf = max_pool_3d(pts_sdf.reshape(1, 1, cropN, cropN, cropN) * -1.0) * -1.0
                min_mask = (current_mask > 0.0).float()
                z = (pts_sdf.reshape(1, 1, cropN, cropN, cropN) * min_mask + min_sdf * (1.0 - min_mask)).numpy()
                cm = (current_mask > 0.0).numpy()[0, 0]
                vz = z.reshape(cropN, cropN, cropN)[cm]
                if vz.shape[0] <= 0 or (np.min(vz) > level or np.max(vz) < level):
                    continue
                if not (np.min(z) > level or np.max(z) < level):
                    spacing = tuple((hi[a] - lo[a]) / (cropN - 1) for a in range(3))
                    mc(z.astype(np.float32).reshape(cropN, cropN, cropN), level, spacing, cm, np.array(lo))
