"""fp64 restatement (numpy, scipy.sparse) of the Poisson reconstruction of sdfstudio_b200/poisson.py, at depths up to 6: the
discretisation of include/sdfb200.h ("Poisson") assembled as sparse matrices, a tight conjugate-gradient solve, the iso value, the
densities and colours at the vertices, and the trim of ExportPoissonMesh (``densities < quantile(densities, 0.1)``).

The mesh comes from the CPU restatement of the marching-cubes kernel (oracle/marching_cubes.py) on -chi at -iso."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle import marching_cubes as omc

SCALE = 1.1
POINT_WEIGHT = 4.0
KERNEL_DEPTH_OFFSET = 2


def element_stiffness(h: float) -> np.ndarray:
    """The Q1 element stiffness of a cube of side h, corners l = 4 lx + 2 ly + lz: h/3 on the diagonal, 0 between corners differing in
    one axis, -h/12 in two or three."""
    bits = np.array([[(l >> 2) & 1, (l >> 1) & 1, l & 1] for l in range(8)])
    diff = (bits[:, None, :] != bits[None, :, :]).sum(-1)
    return np.choose(diff, [h / 3, 0.0, -h / 12, -h / 12])


def cube(points: np.ndarray, depth: int, scale: float = SCALE):
    lo, hi = points.min(0).astype(np.float64), points.max(0).astype(np.float64)
    extent = float(max(hi - lo))
    if not extent > 0:
        raise ValueError("the point cloud's box has zero extent")
    w = scale * extent
    centre = [(float(lo[a]) + float(hi[a])) / 2 for a in range(3)]
    return tuple(c - w / 2 for c in centre), w / 2 ** depth


def locate(points, origin, h, n):
    t = (points.astype(np.float64) - np.asarray(origin)) / h
    c = np.clip(np.floor(t), 0, n - 1)
    return c.astype(np.int64), t - c


def hats(u):
    """[P,8] hats and [P,8,3] gradients (times h) of the corners l = 4 lx + 2 ly + lz at local coordinates u [P,3]."""
    phi = np.empty((len(u), 8))
    grad = np.empty((len(u), 8, 3))
    for l in range(8):
        b = [(l >> 2) & 1, (l >> 1) & 1, l & 1]
        w = [u[:, a] if b[a] else 1 - u[:, a] for a in range(3)]
        s = [1.0 if b[a] else -1.0 for a in range(3)]
        phi[:, l] = w[0] * w[1] * w[2]
        grad[:, l] = np.stack([s[0] * w[1] * w[2], s[1] * w[0] * w[2], s[2] * w[0] * w[1]], 1)
    return phi, grad


def corner_nodes(c, n):
    m = n + 1
    return np.stack([((c[:, 0] + ((l >> 2) & 1)) * m + c[:, 1] + ((l >> 1) & 1)) * m + c[:, 2] + (l & 1) for l in range(8)], 1)


def stiffness(n: int, h: float) -> sp.csr_matrix:
    """L over the n^3 cells, natural boundaries."""
    g = np.arange(n)
    cells = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    ids = corner_nodes(cells, n)
    ke = element_stiffness(h)
    rows = np.repeat(ids, 8, axis=1).ravel()
    cols = np.tile(ids, (1, 8)).ravel()
    vals = np.tile(ke.ravel(), len(cells))
    m = (n + 1) ** 3
    return sp.coo_matrix((vals, (rows, cols)), shape=(m, m)).tocsr()


def usable(points, normals, colors=None):
    """The points that take part (finite, non-zero normal) with their normalised normals (and colours)."""
    ok = np.isfinite(normals).all(1) & (normals != 0).any(1)
    nrm = normals[ok].astype(np.float64)
    nrm = nrm / np.linalg.norm(nrm, axis=1, keepdims=True)
    return points[ok], nrm, (None if colors is None else colors[ok].astype(np.float64))


def assemble(points, normals, depth: int, scale: float = SCALE):
    """dict(L, S, b, a, alpha_a, origin, h, n, points) of the system (L + alpha a S) x = a b."""
    if not 1 <= depth <= 6:
        raise ValueError("the oracle runs depths 1 .. 6")
    pts, nrm, _ = usable(points, normals)
    if len(pts) == 0:
        raise ValueError("no point has a finite, non-zero normal")
    origin, h = cube(pts, depth, scale)
    n = 2 ** depth
    c, u = locate(pts, origin, h, n)
    phi, grad = hats(u)
    ids = corner_nodes(c, n)
    m = (n + 1) ** 3
    b = np.bincount(ids.ravel(), weights=(np.einsum("pla,pa->pl", grad, nrm) / h).ravel(), minlength=m)
    S = sp.coo_matrix(((phi[:, :, None] * phi[:, None, :]).ravel(), (np.repeat(ids, 8, 1).ravel(), np.tile(ids, (1, 8)).ravel())),
                      shape=(m, m)).tocsr()
    occupied = len(np.unique((c[:, 0] * n + c[:, 1]) * n + c[:, 2]))
    a = h * h * occupied / len(pts)
    return dict(L=stiffness(n, h), S=S, b=b, a=a, alpha_a=POINT_WEIGHT * a, origin=origin, h=h, n=n, depth=depth, points=pts)


def solve(system, rtol: float = 1e-12):
    """chi (fp64 node values) by conjugate gradients with a Jacobi preconditioner to ``rtol``, and the iso value."""
    A = (system["L"] + system["alpha_a"] * system["S"]).tocsr()
    rhs = system["a"] * system["b"]
    d = A.diagonal()
    M = sp.diags(1.0 / d)
    x, info = spla.cg(A, rhs, rtol=rtol, atol=0.0, maxiter=20000, M=M)
    assert info == 0, info
    system["A"], system["chi"] = A, x
    n = system["n"]
    c, u = locate(system["points"], system["origin"], system["h"], n)
    phi, _ = hats(u)
    system["iso"] = float(np.mean((phi * x[corner_nodes(c, n)]).sum(1)))
    return system


def splat(points, colors, depth, origin, h):
    """(level, h_level, node sums [(n+1)^3, 4]: sum phi, sum phi rgb) at depth - 2."""
    lvl = max(depth - KERNEL_DEPTH_OFFSET, 0)
    n, hl = 2 ** lvl, h * 2 ** (depth - lvl)
    c, u = locate(points, origin, hl, n)
    phi, _ = hats(u)
    ids = corner_nodes(c, n).ravel()
    m = (n + 1) ** 3
    out = np.stack([np.bincount(ids, weights=phi.ravel(), minlength=m)]
                   + [np.bincount(ids, weights=(phi * colors[:, ch:ch + 1]).ravel(), minlength=m) for ch in range(3)], 1)
    return lvl, hl, out


def interpolate(points, origin, h, n, node_vals):
    c, u = locate(points, origin, h, n)
    phi, _ = hats(u)
    return np.einsum("pl,plc->pc", phi, node_vals[corner_nodes(c, n)])


def reconstruct(points, normals, colors, depth: int, scale: float = SCALE):
    """(system, vertices, faces, normals, densities, colours) in fp64 (the mesh from the marching-cubes restatement)."""
    system = solve(assemble(points, normals, depth, scale))
    n = system["n"]
    vol = (-system["chi"]).reshape(n + 1, n + 1, n + 1).astype(np.float32)
    verts, faces, vnormals = omc.marching_cubes(vol, level=np.float32(-system["iso"]), spacing=(system["h"],) * 3)
    verts = np.asarray(verts, dtype=np.float64) + np.asarray(system["origin"])
    pts, _, col = usable(points, normals, colors if colors is not None else np.zeros_like(points))
    lvl, hl, nodes = splat(pts, col, depth, system["origin"], system["h"])
    at = interpolate(verts, system["origin"], hl, 2 ** lvl, nodes)
    dens = at[:, 0]
    rgb = np.where(dens[:, None] > 0, at[:, 1:] / np.where(dens > 0, dens, 1.0)[:, None], 0.0)
    return system, verts, np.asarray(faces, dtype=np.int64), np.asarray(vnormals), dens, rgb


def low_density_mask(densities, q: float = 0.1):
    d = np.asarray(densities, dtype=np.float64)
    return d < np.quantile(d, q)


def remove_vertices_by_mask(vertices, faces, mask):
    """open3d's rules: drop the masked vertices and every face touching one, keep the rest in order, reindex."""
    keep = ~np.asarray(mask, dtype=bool)
    new = np.cumsum(keep) - 1
    f = faces[keep[faces].all(1)]
    return vertices[keep], new[f]


# -- test clouds ----------------------------------------------------------------------------------------------------------------------
def sphere_cloud(n: int, radius: float = 0.6, seed: int = 0):
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    colors = 0.5 + 0.5 * d
    return (radius * d).astype(np.float32), d.astype(np.float32), colors.astype(np.float32)


def torus_cloud(n: int, R: float = 0.6, r: float = 0.25, seed: int = 1):
    rng = np.random.default_rng(seed)
    # area-uniform: accept theta with probability (R + r cos theta) / (R + r)
    th = np.empty(0)
    while len(th) < n:
        t = rng.uniform(0, 2 * np.pi, 4 * n)
        th = np.concatenate([th, t[rng.uniform(0, 1, 4 * n) < (R + r * np.cos(t)) / (R + r)]])
    th = th[:n]
    ph = rng.uniform(0, 2 * np.pi, n)
    nrm = np.stack([np.cos(th) * np.cos(ph), np.cos(th) * np.sin(ph), np.sin(th)], 1)
    p = np.stack([(R + r * np.cos(th)) * np.cos(ph), (R + r * np.cos(th)) * np.sin(ph), r * np.sin(th)], 1)
    return p.astype(np.float32), nrm.astype(np.float32), (0.5 + 0.5 * nrm).astype(np.float32)


def plane_cloud(n: int, seed: int = 2):
    rng = np.random.default_rng(seed)
    p = np.concatenate([rng.uniform(-0.5, 0.5, (n, 2)), np.full((n, 1), 0.1)], 1)
    nrm = np.tile([0.0, 0.0, 1.0], (n, 1))
    return p.astype(np.float32), nrm.astype(np.float32), rng.uniform(0, 1, (n, 3)).astype(np.float32)


def clustered_cloud(n: int, seed: int = 3):
    rng = np.random.default_rng(seed)
    centres = rng.uniform(-0.5, 0.5, (5, 3))
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    p = centres[np.arange(n) % 5] + 0.12 * d
    return p.astype(np.float32), d.astype(np.float32), rng.uniform(0, 1, (n, 3)).astype(np.float32)


CLOUDS = {"sphere": sphere_cloud, "torus": torus_cloud, "plane": plane_cloud, "clusters": clustered_cloud}
