"""Two restatements of the reference's TSDF fusion (nerfstudio/exporter/tsdf_utils.py:92-270).

(a) ``from_aabb``, ``integrate`` and ``mesh_from_marching_cubes``: the reference's ATen ops in its order, on whole batches, on the CPU
    or the GPU.  ``integrate`` keeps the reference's batched ``torch.bmm`` and ``grid_sample`` calls and its image-by-image update, so on
    the CPU it reproduces the reference bit for bit.
(b) ``integrate_ops``: numpy float32, one voxel's chain of separately rounded operations in the order include/sdfb200.h documents for
    sdfb200_tsdf_integrate, sequential over the images.  The kernel must equal it bit for bit.  It differs from (a) only where (a)'s
    backend rounds otherwise: the summation order inside ``bmm``, and the CPU ``grid_sample``'s unnormalisation.
"""
import numpy as np
import torch
import torch.nn.functional as F


def from_aabb(aabb, volume_dims):
    """TSDF.from_aabb (:92-114): (voxel_coords [3,X,Y,Z], values, weights, colors [X,Y,Z,3], voxel_size [3], origin [3])."""
    origin = aabb[0]
    voxel_size = (aabb[1] - aabb[0]) / volume_dims
    axes = [torch.arange(int(d)) for d in volume_dims]
    grid = torch.stack(torch.meshgrid(axes, indexing="ij"), dim=0)
    voxel_coords = origin.view(3, 1, 1, 1) + grid * voxel_size.view(3, 1, 1, 1)
    dims = volume_dims.tolist()
    return voxel_coords, -torch.ones(dims), torch.zeros(dims), torch.zeros(dims + [3]), voxel_size, origin


def truncation(voxel_size, truncation_margin=5.0):
    return voxel_size[0] * truncation_margin


def integrate(voxel_coords, values, weights, colors, trunc, c2w, K, depth_images, color_images=None):
    """TSDF.integrate_tsdf (:168-270) on one batch, updating values / weights / colors in place.  depth_images [B,1,H,W],
    color_images [B,3,H,W] or None."""
    dev = voxel_coords.device
    B = c2w.shape[0]
    shape = voxel_coords.shape[1:]
    image_size = torch.tensor([depth_images.shape[-1], depth_images.shape[-2]], device=dev)
    pts = voxel_coords.view(3, -1)
    pts = torch.cat([pts, torch.ones(1, pts.shape[1], device=dev)], dim=0)[None].expand(B, 4, -1)
    cam = torch.bmm(torch.inverse(c2w), pts)
    cam[:, 2, :] = -cam[:, 2, :]
    cam[:, 1, :] = -cam[:, 1, :]
    voxel_depth = torch.sqrt(torch.sum(cam[:, :3, :] ** 2, dim=-2, keepdim=True))
    pix = torch.bmm(K, cam[:, 0:3, :] / cam[:, 2:3, :])[:, :2, :]
    grid = (2.0 * pix.permute(0, 2, 1) / image_size.view(1, 1, 2) - 1.0)[:, None]
    sampled_depth = F.grid_sample(depth_images, grid, mode="nearest", padding_mode="zeros", align_corners=False).squeeze(2)
    if color_images is not None:
        sampled_colors = F.grid_sample(color_images, grid, mode="nearest", padding_mode="zeros", align_corners=False).squeeze(2)
    dist = sampled_depth - voxel_depth
    tsdf = torch.clamp(dist / trunc, min=-1.0, max=1.0)
    valid = (voxel_depth > 0) & (sampled_depth > 0) & (dist > -trunc)
    for i in range(B):
        m = valid[i].view(*shape)
        old_v, old_w = values[m], weights[m]
        total = old_w + 1.0
        values[m] = (old_v * old_w + tsdf[i][valid[i]] * 1.0) / total
        weights[m] = torch.clamp(total, max=1.0)
        if color_images is not None:
            new_c = sampled_colors[i][:, valid[i].squeeze(0)].permute(1, 0)
            colors[m] = (colors[m] * old_w[:, None] + new_c * 1.0) / total[:, None]


def integrate_batched(state, trunc, c2w, K, depth_images, color_images, batch_size):
    """export_tsdf_mesh's loop (:343-349): ``integrate`` over consecutive batches of ``batch_size`` images."""
    for i in range(0, len(c2w), batch_size):
        integrate(*state, trunc, c2w[i:i + batch_size], K[i:i + batch_size], depth_images[i:i + batch_size],
                  None if color_images is None else color_images[i:i + batch_size])


def mesh_from_marching_cubes(values, colors, origin, voxel_size, vertices, faces, normals):
    """TSDF.get_mesh (:116-136) after skimage: colours gathered at the rounded (half to even) vertex indices, vertices moved to world
    space.  ``vertices`` [V,3] in voxel units."""
    idx = torch.round(vertices).long()
    c = colors[idx[:, 0], idx[:, 1], idx[:, 2]]
    return origin.view(1, 3) + vertices * voxel_size.view(1, 3), faces, normals, c


def pack_cams(c2w, K):
    """[B,18] fp32: rows 0-2 of torch.inverse(c2w), rows 0-1 of K."""
    inv = torch.inverse(c2w)
    return torch.cat([inv[:, :3, :].reshape(-1, 12), K[:, :2, :].reshape(-1, 6)], dim=1).float().contiguous()


def pixel_index(p, size):
    """g = (2 p) / size - 1, ATen's CUDA unnormalisation ((g + 1) size - 1) / 2, rint (half to even); -1 outside or non-finite."""
    s = np.float32(size)
    g = (np.float32(2) * p) / s - np.float32(1)
    f = np.rint(((g + np.float32(1)) * s - np.float32(1)) / np.float32(2))
    with np.errstate(invalid="ignore"):
        inside = (f >= 0) & (f < s)
    return np.where(inside, np.where(inside, f, 0).astype(np.int64), -1)


def project(voxel_coords, cams, b, H, W):
    """Image b's (voxel_depth [N], ix [N], iy [N]) in (b)'s op order; voxel_coords [3,N] float32 numpy, cams [B,18] float32 numpy."""
    x, y, z = voxel_coords
    m = cams[b]

    def dot(r):
        return ((m[r] * x + m[r + 1] * y) + m[r + 2] * z) + m[r + 3]

    cx, cy, cz = dot(0), -dot(4), -dot(8)
    vd = np.sqrt((cx * cx + cy * cy) + cz * cz)
    u, v, w = cx / cz, cy / cz, cz / cz
    k = m[12:]
    px = (k[0] * u + k[1] * v) + k[2] * w
    py = (k[3] * u + k[4] * v) + k[5] * w
    return vd, pixel_index(px, W), pixel_index(py, H)


def integrate_ops(voxel_coords, values, weights, colors, trunc, cams, depth, color=None):
    """(b): sdfb200_tsdf_integrate's documented op order in numpy float32.  voxel_coords [3,N], values / weights [N], colors [N,3],
    cams [B,18], depth [B,H,W], color [B,3,H,W] or None, trunc a float32.  Returns new (values, weights, colors) and, per image, the
    pixel indices and validity (for counting where (a) and (b) disagree)."""
    with np.errstate(all="ignore"):
        f32 = np.float32
        xyz = np.asarray(voxel_coords, f32)
        v, w, c = np.array(values, f32), np.array(weights, f32), np.array(colors, f32)
        trunc = f32(trunc)
        B, H, W = depth.shape
        trace = []
        for b in range(B):
            vd, ix, iy = project(xyz, cams, b, H, W)
            inside = (ix >= 0) & (iy >= 0)
            sd = np.where(inside, depth[b][np.maximum(iy, 0), np.maximum(ix, 0)], f32(0))
            dist = sd - vd
            valid = (vd > 0) & (sd > 0) & (dist > -trunc)
            t = np.clip(dist / trunc, f32(-1), f32(1))
            total = w + f32(1)
            v = np.where(valid, (v * w + t) / total, v)
            if color is not None:
                nc = color[b][:, np.maximum(iy, 0), np.maximum(ix, 0)].T
                c = np.where(valid[:, None], (c * w[:, None] + nc) / total[:, None], c)
            w = np.where(valid, np.minimum(total, f32(1)), w)
            trace.append((ix, iy, valid))
        return v, w, c, trace
