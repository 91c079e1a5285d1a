"""Torch restatement of the texture export of the reference (nerfstudio/exporter/texture_utils.py:43-323, :379-405): which face each
texel of the texture lies on, its barycentric weights and the ray that colours it.  Runs on CPU or CUDA.

Unlike the reference, the search keeps the per-texel face index and weights as outputs (``face`` [P] int64, ``bary`` [P,3]) so that
the kernels can be compared with them directly; the texel rays are then computed from them exactly as the reference computes its
origins and directions.  Every floating-point operation is the reference's, in its order, as separate ATen ops.
"""
import math

import torch


def parallelogram_area(p, v0, v1):
    """texture_utils.py:43-56: twice the signed area of (p, v0, v1)."""
    return (p[..., 0] - v0[..., 0]) * (v1[..., 1] - v0[..., 1]) - (p[..., 1] - v0[..., 1]) * (v1[..., 0] - v0[..., 0])


def texel_linspaces(width, height, device):
    """The two torch.linspace vectors of get_texture_image (:59-75): texel centres along u (width) and v (height)."""
    px_w, px_h = 1.0 / width, 1.0 / height
    return torch.linspace(px_w / 2, 1 - px_w / 2, width, device=device), torch.linspace(px_h / 2, 1 - px_h / 2, height, device=device)


def texel_centres(lin_w, lin_h):
    """[H*W, 2] texel centres in row-major order: torch.meshgrid(lin_w, lin_h, indexing="xy") stacked (:71-73)."""
    return torch.stack(torch.meshgrid(lin_w, lin_h, indexing="xy"), dim=-1).reshape(-1, 2)


def barycentric(p, tri):
    """(w0, w1, w2) of points p [..., 2] in triangles tri [..., 3, 2] (:185-192, :285-288)."""
    v0, v1, v2 = tri[..., 0, :], tri[..., 1, :], tri[..., 2, :]
    area = parallelogram_area(v2, v0, v1)
    return parallelogram_area(p, v1, v2) / area, parallelogram_area(p, v2, v0) / area, parallelogram_area(p, v0, v1) / area


def rasterize(texture_coordinates, num_pixels_per_side, chunk=10):
    """The xatlas path's per-texel search (:263-301).  Returns face [P] int64 and bary [P,3], P = num_pixels_per_side**2."""
    n = num_pixels_per_side
    dev = texture_coordinates.device
    p = texel_centres(*texel_linspaces(n, n, dev))[None]                          # (1, P, 2)
    P = p.shape[1]
    best = torch.full((1, P), torch.finfo(torch.float32).max, device=dev)
    face = torch.zeros(1, P, dtype=torch.long, device=dev)
    w = [torch.zeros(1, P, device=dev) for _ in range(3)]
    cols = torch.arange(P, device=dev)
    for i in range(texture_coordinates.shape[0] // chunk):
        s = i * chunk
        tri = texture_coordinates[s:s + chunk, None]                               # (c, 1, 3, 2)
        ws = barycentric(p, tri)                                                   # 3 x (c, P)
        dist = torch.abs(ws[0]) + torch.abs(ws[1]) + torch.abs(ws[2])
        d, idx = torch.min(dist, dim=0, keepdim=True)
        take = d < best
        best = torch.where(take, d, best)
        face = torch.where(take, idx + s, face)
        w = [torch.where(take, wk[idx[0], cols][None], wo) for wk, wo in zip(ws, w)]
    return face[0], torch.stack([wk[0] for wk in w], dim=-1)


def grid_layout(num_faces, px_per_uv_triangle):
    """Sizes of the custom unwrap (:100-108): (squares_per_side_w, squares_per_side_h, width, height)."""
    num_squares = math.ceil(num_faces / 2)
    sw = math.ceil(math.sqrt(num_squares))
    sh = math.ceil(num_squares / sw)
    return sw, sh, sw * (px_per_uv_triangle + 3), sh * px_per_uv_triangle


def grid_square(num_faces, px_per_uv_triangle, device):
    """The two triangles of the first rectangle [6, 2] and the rectangle's extent lr [2] (:119-149)."""
    ppt = px_per_uv_triangle
    _, _, W, H = grid_layout(num_faces, ppt)
    lr_w, lr_h = (ppt + 3) / W, ppt / H
    lr = torch.tensor([lr_w, lr_h], device=device)
    px_w, px_h = 1.0 / W, 1.0 / H
    px = torch.tensor([px_w, px_h], device=device)
    scalar = (ppt - 1) / ppt
    upper_left = torch.tensor([[0, 0], [ppt / W, 0], [0, ppt / H]], device=device) * scalar + px / 2
    lower_right = [lr_w, lr_h]
    lower = torch.tensor([lower_right, [3 * px_w, lr_h], [lr_w, 0]], device=device)
    lower = (lower - torch.tensor(lower_right, device=device)) * scalar + torch.tensor(lower_right, device=device) - px / 2
    return torch.stack([upper_left, lower], dim=0).reshape(6, 2), lr


def grid_unwrap(num_faces, px_per_uv_triangle, device):
    """The custom unwrap (:100-192) without the gathers: texture_coordinates [F,3,2], face [P] int64 (clamped to F - 1), bary [P,3] and
    the texture's (height, width)."""
    ppt = px_per_uv_triangle
    sw, sh, W, H = grid_layout(num_faces, ppt)
    square, lr = grid_square(num_faces, ppt, device)
    offsets = torch.stack(torch.meshgrid(torch.arange(sw, device=device), torch.arange(sh, device=device), indexing="xy"), dim=-1) * lr
    tc = (square.reshape(1, 1, 6, 2) + offsets.view(sh, sw, 1, 2)).view(-1, 3, 2)[:num_faces]
    jj, ii = torch.meshgrid(torch.arange(W, device=device), torch.arange(H, device=device), indexing="xy")
    sqw = ppt + 3
    square_index = torch.div(ii, ppt, rounding_mode="floor") * sw + torch.div(jj, sqw, rounding_mode="floor")
    lower = (jj % sqw + ii % ppt) >= (sqw - 2)
    face = torch.clamp(square_index * 2 + lower, min=0, max=num_faces - 1).reshape(-1)
    p = texel_centres(*texel_linspaces(W, H, device))
    w = barycentric(p, tc[face])
    return tc, face, torch.stack(w, dim=-1), (H, W)


def texel_rays(vertices, faces, vertex_normals, face, bary):
    """Origins and directions of the texels before the ray-length shift (:194-205, :303-321)."""
    fv = vertices[faces[face]]
    fn = vertex_normals[faces[face]]
    w0, w1, w2 = bary[:, 0:1], bary[:, 1:2], bary[:, 2:3]
    origins = (fv[:, 0] * w0 + fv[:, 1] * w1 + fv[:, 2] * w2).float()
    directions = -(fn[:, 0] * w0 + fn[:, 1] * w1 + fn[:, 2] * w2).float()
    return origins, torch.nn.functional.normalize(directions, dim=-1)


def ray_length(vertices, faces, raylen_method="edge"):
    """:379-387: twice the mean length of each face's first edge, or 0.0."""
    if raylen_method == "edge":
        fv = vertices[faces]
        return 2.0 * torch.mean(torch.norm(fv[:, 1, :] - fv[:, 0, :], dim=-1)).float()
    if raylen_method == "none":
        return 0.0
    raise ValueError(f"Ray length method {raylen_method} not supported.")


def texel_bundle(origins, directions, raylen):
    """:391-396: the fields of the texture's camera ray bundle (shapes [..., 3] / [..., 1])."""
    origins = origins - 0.5 * raylen * directions
    one = torch.ones_like(origins[..., 0:1])
    return dict(origins=origins, directions=directions, pixel_area=one, camera_indices=torch.zeros_like(one), directions_norm=one,
                nears=torch.zeros_like(one), fars=one * raylen)
