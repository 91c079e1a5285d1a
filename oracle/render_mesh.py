"""fp64 restatement of the mesh renderer (include/sdfb200.h, sdfb200_mesh_rasterize / sdfb200_mesh_shade) in numpy.

``rasterize`` tests every (pixel, face) pair by brute force, in the kernel's op order: numpy's elementwise float64 operations each round on
their own, so the keys are bit-identical to the kernel's.  ``shade`` is the shading in float64 (pow and sqrt may differ from the device's in
the last bit, so bytes are compared within 1).  ``merge`` is the merged video frame.

The four camera paths (spiral, ellipse, interpolate, viewer JSON) are not restated here: they are host arithmetic, and
tests/test_render_mesh_cpu.py compares the package's paths bit for bit with goldens minted from the unmodified reference
(oracle/make_golden_render_mesh.py), a stronger check than a restatement.
"""
import numpy as np

BACKGROUND = np.uint64(0xFFFFFFFFFFFFFFFF)


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def to_camera(cam, p):
    """Rows 0-2 of inverse(c2w) (cam[:12], fp32) applied to fp32 points [..., 3], in double."""
    m = np.asarray(cam[:12], np.float32).astype(np.float64).reshape(3, 4)
    p = np.asarray(p, np.float32).astype(np.float64)
    return np.stack([((m[r, 0] * p[..., 0] + m[r, 1] * p[..., 1]) + m[r, 2] * p[..., 2]) + m[r, 3] for r in range(3)], -1)


def setup(cam, vertices, faces):
    """(v [F,3,3] camera space, e [F,3,3] oriented edge normals, num [F], front [F] bool) of every face."""
    v = to_camera(cam, np.asarray(vertices, np.float32)[np.asarray(faces, np.int64)])
    E = np.stack([_cross(v[:, 1], v[:, 2]), _cross(v[:, 2], v[:, 0]), _cross(v[:, 0], v[:, 1])], 1)
    det = _dot(v[:, 0], E[:, 0])
    return v, -E, -det, det < 0


def pixel_dirs(cam, H, W):
    """(dx [W], dy [H]) of the rays through the pixel centres."""
    k = np.asarray(cam[12:], np.float32).astype(np.float64)
    fx, cx, fy, cy = k[0], k[2], k[4], k[5]
    return (np.arange(W, dtype=np.float64) + 0.5 - cx) / fx, -((np.arange(H, dtype=np.float64) + 0.5 - cy) / fy)


def edge_products(e, dx, dy):
    """w [..., 3] = (dx e.x + dy e.y) - e.z for edge normals e [..., 3, 3] and directions dx, dy broadcast against e's leading dims."""
    return (dx[..., None] * e[..., 0] + dy[..., None] * e[..., 1]) - e[..., 2]


def rasterize(vertices, faces, cams, H, W, z_near, chunk=4096):
    """keys [B,H,W] uint64 over every (pixel, face) pair."""
    cams = np.asarray(cams, np.float32).reshape(-1, 18)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    keys = np.full((len(cams), H, W), BACKGROUND, np.uint64)
    zn = np.float64(np.float32(z_near))
    for b, cam in enumerate(cams):
        if len(faces) == 0:
            continue
        _, e, num, front = setup(cam, vertices, faces)
        dx, dy = pixel_dirs(cam, H, W)
        DX, DY = np.broadcast_to(dx[None, :], (H, W)).reshape(-1), np.broadcast_to(dy[:, None], (H, W)).reshape(-1)
        best = keys[b].reshape(-1)
        with np.errstate(all="ignore"):
            for f0 in range(0, len(faces), chunk):
                ee, nn, ff = e[f0:f0 + chunk], num[f0:f0 + chunk], front[f0:f0 + chunk]
                w = edge_products(ee[None], DX[:, None], DY[:, None])          # [P, f, 3]
                S = (w[..., 0] + w[..., 1]) + w[..., 2]
                depth = nn[None] / S
                ok = ff[None] & (w[..., 0] >= 0) & (w[..., 1] >= 0) & (w[..., 2] >= 0) & (S > 0) & (depth >= zn)
                k = (depth.astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.arange(f0, f0 + len(ee), dtype=np.uint64)[None]
                k = np.where(ok, k, BACKGROUND).min(1)
                best[:] = np.minimum(best, k)
    return keys


def split(keys):
    """(face int32, -1 background; depth fp32, +inf background)."""
    keys = np.asarray(keys, np.uint64)
    bg = keys == BACKGROUND
    face = np.where(bg, -1, (keys & np.uint64(0xFFFFFFFF)).astype(np.int64)).astype(np.int32)
    depth = (keys >> np.uint64(32)).astype(np.uint32).view(np.float32)
    return face, np.where(bg, np.float32(np.inf), depth)


def _unit(a):
    n = np.sqrt(_dot(a, a))
    with np.errstate(all="ignore"):
        return np.where(n[..., None] > 0, a / n[..., None], a)


def shade(keys, vertices, vertex_normals, faces, cams, light_positions, light_params):
    """(rgb, normal) [B,H,W,3] float64 colours before quantisation, background 1."""
    keys = np.asarray(keys, np.uint64)
    B, H, W = keys.shape
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    lp = np.asarray(light_params, np.float32).astype(np.float64)
    rgb, nrm = np.ones((B, H, W, 3)), np.ones((B, H, W, 3))
    for b in range(B):
        cam = np.asarray(cams, np.float32).reshape(-1, 18)[b]
        face, _ = split(keys[b])
        jj, ii = np.nonzero(face >= 0)
        if len(jj) == 0:
            continue
        f = face[jj, ii].astype(np.int64)
        v, e, num, _ = setup(cam, vertices, faces[f])
        dx, dy = pixel_dirs(cam, H, W)
        w = edge_products(e, dx[ii], dy[jj])
        S = (w[:, 0] + w[:, 1]) + w[:, 2]
        depth = num / S
        bc = w / S[:, None]
        m = np.asarray(cam[:12], np.float32).astype(np.float64).reshape(3, 4)
        n = np.asarray(vertex_normals, np.float32).astype(np.float64)[faces[f]]
        n = np.stack([(m[r, 0] * n[..., 0] + m[r, 1] * n[..., 1]) + m[r, 2] * n[..., 2] for r in range(3)], -1)

        def blend(nk):
            return (bc[:, 0:1] * nk[:, 0] + bc[:, 1:2] * nk[:, 1]) + bc[:, 2:3] * nk[:, 2]

        nrm[b, jj, ii] = _unit(blend(n)) * 0.5 + 0.5
        flip = _dot(n, -v) < 0
        nn = _unit(blend(np.where(flip[..., None], -n, n)))
        d = np.stack([dx[ii], dy[jj], -np.ones(len(ii))], -1)
        hit = depth[:, None] * d
        eye = _unit(-hit)
        c = np.broadcast_to(lp[24:27], (len(ii), 3)).copy()
        L = np.asarray(light_positions, np.float32).astype(np.float64).reshape(-1, 4, 3)[b]
        for k in range(4):
            col, dif, spe, shi = lp[6 * k:6 * k + 3], lp[6 * k + 3], lp[6 * k + 4], lp[6 * k + 5]
            l = _unit(L[k] - hit)
            ndl = _dot(nn, l)
            r = (2.0 * ndl)[:, None] * nn - l
            edr = _dot(eye, r)
            with np.errstate(all="ignore"):
                spec = np.where(edr > 0, np.power(np.maximum(edr, 0), shi), 0.0)
            c = c + col[None] * (dif * np.maximum(ndl, 0) + spe * spec)[:, None]
        rgb[b, jj, ii] = c
    return rgb, nrm


def quantise(c):
    return np.floor(np.clip(c, 0.0, 1.0) * 255.0 + 0.5).astype(np.uint8)


def merge(images, merge_type):
    """The merged video frame: "concat" side by side; "half" the left W // 2 columns of the first output, the rest of the second."""
    if merge_type == "concat":
        return np.concatenate(images, axis=1)
    mask = np.zeros_like(images[0])
    mask[:, : mask.shape[1] // 2, :] = 1
    return images[0] * mask + images[1] * (1 - mask)
