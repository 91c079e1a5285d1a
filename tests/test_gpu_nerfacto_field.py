"""The nerfacto background field on the GPU (csrc/hash_mlp.cuh, sdfstudio_b200/nerfacto_field.py) against the fp64 oracle
(oracle/nerfacto.py): the eval kernel across normalisations, table types, widths, appearance modes and sizes, the C-ABI's error paths, the
differentiable training composition, and an angelo-shaped step with the reference's background merge."""
import math

import numpy as np
import pytest
import torch

from oracle import nerfacto as onf
from oracle.field import OracleField, scene_contraction

from helpers import build_case, make_bundle

pytestmark = pytest.mark.gpu

AABB = [[-3.0, -3, -3], [3, 3, 3]]
NUM_IMAGES = 5


def _maxrel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _field(norm="linf", hidden=64, hidden_color=64, num_layers=2, num_layers_color=3, mean_app=False, seed=0, log2=12, num_levels=16,
           num_images=NUM_IMAGES):
    import sdfstudio_b200 as sb

    sd = None if norm == "aabb" else sb.SceneContraction(order=float("inf") if norm == "linf" else None)
    f = sb.TCNNNerfactoField(torch.tensor(AABB), num_images=num_images, num_layers=num_layers, hidden_dim=hidden, num_layers_color=num_layers_color,
                             hidden_dim_color=hidden_color, log2_hashmap_size=log2, num_levels=num_levels, max_res=512,
                             use_average_appearance_embedding=mean_app, spatial_distortion=sd)
    g = torch.Generator().manual_seed(seed)
    nb, nh = f.mlp_base, f.mlp_head
    with torch.no_grad():   # spread enough that every output varies; padding stays zero like the tcnn layout
        w = nb.params[: nb.n_net].view(-1)
        w.copy_((w != 0).float() * torch.randn(w.shape, generator=g) * (2.0 / math.sqrt(hidden)))
        nb.params[nb.n_net:] = torch.rand(nb.n_grid, generator=g) * 2 - 1
        h = nh.params
        h.copy_((h != 0).float() * torch.randn(h.shape, generator=g) * (1.5 / math.sqrt(hidden_color)))
        f.embedding_appearance.embedding.weight.mul_(0.5)
    return f.cuda()


def _rays(R, S, seed=1):
    """rays from cameras at distance 2-2.8 through the unit sphere, sorted euclidean bins in [0.2, 8]"""
    g = torch.Generator().manual_seed(seed)
    o = torch.randn(R, 3, generator=g)
    o = o / o.norm(dim=-1, keepdim=True) * (2.0 + 0.8 * torch.rand(R, 1, generator=g))
    d = -o + 0.6 * torch.randn(R, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True)
    bins = torch.sort(0.2 + 7.8 * torch.rand(R, S + 1, generator=g), dim=-1).values
    cam = torch.randint(0, NUM_IMAGES, (R,), generator=g)
    return o, d, bins, cam


def _samples(o, d, bins, cam):
    """this package's RaySamples (ray mode: they carry the [R, S+1] bin buffer)"""
    import sdfstudio_b200 as sb
    from sdfstudio_b200.rays import make_ray_samples

    R = o.shape[0]
    rb = sb.RayBundle(origins=o.cuda(), directions=d.cuda(), pixel_area=torch.ones(R, 1, device="cuda"), camera_indices=cam.view(R, 1).cuda())
    b = bins.cuda().contiguous()
    return make_ray_samples(rb, b, b, None)


def _spec(f):
    nb, nh = f.mlp_base, f.mlp_head
    return onf.NerfactoSpec(num_levels=nb.desc.n_levels, max_res=512, log2_hashmap_size=nb.desc.log2_hashmap_size, hidden_dim=nb.hidden_dim,
                            num_layers=nb.n_hidden_layers + 1, hidden_dim_color=nh.hidden_dim, num_layers_color=nh.n_hidden_layers + 1)


def _oracle(f, pos, dirs, app, dtype, norm):
    """the oracle in `dtype` on the fp32 normalised positions (the inputs the kernel hands to the grid), so that fp32 and fp64 share every
    grid cell and the difference between them is arithmetic rounding only"""
    spec = _spec(f)
    x01 = onf.normalize(pos.cpu().float(), torch.tensor(AABB) if norm == "aabb" else None, None if norm == "aabb" else norm)
    c = lambda t: t.detach().cpu().to(dtype)  # noqa: E731
    dens, pre, geo = onf.density(c(x01), c(f.mlp_base.params), spec)
    return {"density": dens, "pre": pre, "geo": geo, "rgb": onf.rgb(c(dirs), geo, c(app), c(f.mlp_head.params), spec)}


def _appearance(f, mode, cam_per_sample):
    emb = f.embedding_appearance.embedding.weight.detach().cpu()
    if mode == "train":
        return emb[cam_per_sample]
    if mode == "eval_mean":
        return emb.mean(0).expand(cam_per_sample.shape[0], -1)
    return torch.zeros(cam_per_sample.shape[0], emb.shape[1])


def _check(got, pos, dirs, app, f, norm, what, factor=4.0):
    """kernel vs fp64 oracle within `factor` x the fp32 oracle's own distance to fp64 (plus a small floor), every output finite.  Under the
    L-inf contraction and the aabb the kernel's normalised positions are those of the oracle bit for bit, so every sample must pass.  Under
    L2 the kernel's norm is rounded differently (fused multiply-adds), and a sample within an ulp of a grid-cell face may fall into the
    neighbouring cell; at most a few such samples are let through there."""
    r64 = _oracle(f, pos, dirs, app, torch.float64, norm)
    r32 = _oracle(f, pos, dirs, app, torch.float32, norm)
    n = r64["pre"].shape[0]
    allowed = max(2, n // 1000) if norm == "l2" else 0
    for key, floor in (("pre", 2e-5), ("rgb", 2e-6), ("density", 2e-5), ("geo", 2e-5)):
        if key not in got:
            continue
        cuda = got[key].detach().double().cpu().reshape(n, -1)
        assert bool(torch.isfinite(cuda).all()), f"{what} {key}: {int((~torch.isfinite(cuda)).sum())} non-finite outputs"
        exact = r64[key].reshape(n, -1)
        scale = exact.abs().clamp_min(1.0) if key == "density" else max(1.0, float(exact.abs().max()))
        noise = float(((r32[key].double().reshape(n, -1) - exact).abs() / scale).max())
        err = ((cuda - exact).abs() / scale).amax(dim=1)
        bound = max(floor, factor * noise)
        outliers = int((~(err <= bound)).sum())
        assert outliers <= allowed, f"{what} {key}: {outliers} samples with |cuda-exact| > {bound:.3e} (max {float(err.max()):.3e})"
    return r64


def _midpoints(o, d, bins):
    """Frustums.get_positions in fp32, exactly the reference's operation order"""
    R, S = bins.shape[0], bins.shape[1] - 1
    pos = onf.midpoints(o[:, None], d[:, None], bins[:, :-1, None], bins[:, 1:, None])
    return pos.reshape(-1, 3), d[:, None].expand(R, S, 3).reshape(-1, 3)


CASES = [  # (norm, hidden, hidden_color, layers, layers_color, mode)
    ("linf", 64, 64, 2, 3, "train"), ("l2", 64, 64, 2, 3, "train"), ("aabb", 64, 64, 2, 3, "train"),
    ("linf", 64, 64, 2, 3, "eval_zeros"), ("linf", 64, 64, 2, 3, "eval_mean"),
    ("linf", 16, 32, 3, 2, "train"), ("l2", 32, 16, 4, 4, "eval_mean"), ("aabb", 16, 16, 2, 2, "eval_zeros"), ("linf", 32, 64, 2, 3, "train"),
]


@pytest.mark.parametrize("norm,hidden,hidden_color,layers,layers_color,mode", CASES)
def test_eval_forward_matches_fp64_oracle(norm, hidden, hidden_color, layers, layers_color, mode):
    """forward() under no_grad (mode "train": train mode with camera indices) or in eval mode: one launch, vs the fp64 oracle on the
    same fp32 sample positions."""
    import sdfstudio_b200 as sb

    f = _field(norm, hidden, hidden_color, layers, layers_color, mean_app=mode == "eval_mean")
    f.train(mode == "train")
    R, S = 64, 48
    o, d, bins, cam = _rays(R, S)
    rs = _samples(o, d, bins, cam)
    n0 = sb._lib.launch_count()
    with torch.no_grad():
        out = f(rs)
    assert sb._lib.launch_count() - n0 == 1
    got = {"density": out[sb.FieldHeadNames.DENSITY], "rgb": out[sb.FieldHeadNames.RGB], "pre": f._density_before_activation}
    assert out[sb.FieldHeadNames.RGB].shape == (R, S, 3) and out[sb.FieldHeadNames.DENSITY].shape == (R, S, 1)
    pos, dirs = _midpoints(o, d, bins)
    _check(got, pos, dirs, _appearance(f, mode, cam[:, None].expand(R, S).reshape(-1)), f, norm, f"{norm} {hidden}/{hidden_color} {mode}")
    x01 = f._sample_locations
    assert x01.shape == (R, S, 3)


def _abi(f, origins, directions, bins, n_rows, app, stride, table_dtype="fp32", want_geo=True, want_rgb=True):
    """sdfb200_nerfacto_field_forward with explicit buffers (point mode when bins is None)."""
    from sdfstudio_b200 import _lib

    lib = _lib.load()
    nb, nh = f.mlp_base, f.mlp_head
    S = 0 if bins is None else bins.shape[1] - 1
    N = n_rows * S if S else n_rows
    p = nb.params.detach()
    table = p[nb.n_net:].half().contiguous() if table_dtype == "fp16" else p[nb.n_net:]
    desc = nb.desc
    desc.active_levels, desc.table_dtype = desc.n_levels, (_lib.DT_F16 if table_dtype == "fp16" else _lib.DT_F32)
    out = {"density": torch.full((N,), float("nan"), device="cuda"), "rgb": torch.full((N, 3), float("nan"), device="cuda"),
           "pre": torch.full((N,), float("nan"), device="cuda"), "geo": torch.full((N, f.geo_feat_dim), float("nan"), device="cuda")}
    code = f._contraction_code()
    aabb = f.aabb.detach().contiguous() if code == _lib.CONTRACT_NONE else None
    rc = lib.sdfb200_nerfacto_field_forward(desc, f._desc(S), table.data_ptr(), p.data_ptr(), nh.params.detach().data_ptr(), _lib.ptr(aabb),
                                            _lib.ptr(origins), _lib.ptr(directions), _lib.ptr(bins), n_rows, _lib.ptr(app), stride,
                                            out["density"].data_ptr(), out["rgb"].data_ptr() if want_rgb else None, out["pre"].data_ptr(),
                                            out["geo"].data_ptr() if want_geo else None, _lib.stream_ptr())
    desc.table_dtype = _lib.DT_F32
    _lib.check(rc, "sdfb200_nerfacto_field_forward")
    return out


@pytest.mark.parametrize("N", [0, 1, 127, 128, 129, 8192 * 48])
def test_point_mode_sizes(N):
    """point mode at the block-size edges and at the angelo workload's size (8192 rays x 48 samples), geometry feature included"""
    f = _field("linf").eval()
    g = torch.Generator().manual_seed(N)
    pos = (torch.rand(N, 3, generator=g) * 2 - 1) * 6.0
    dirs = torch.nn.functional.normalize(torch.randn(N, 3, generator=g), dim=-1)
    got = _abi(f, pos.cuda(), dirs.cuda(), None, N, None, 0)
    if N == 0:
        return
    _check(got, pos, dirs, torch.zeros(N, 32), f, "linf", f"N={N}")


def test_fp16_table():
    """an fp16 table (tiny-cuda-nn's storage precision) against the oracle on the fp16-representable table"""
    f = _field("linf").eval()
    with torch.no_grad():
        nb = f.mlp_base
        nb.params[nb.n_net:] = nb.params[nb.n_net:].half().float()
    R, S = 64, 48
    o, d, bins, cam = _rays(R, S, seed=4)
    got = _abi(f, o.cuda(), d.cuda(), bins.cuda(), R, None, 0, table_dtype="fp16")
    got32 = _abi(f, o.cuda(), d.cuda(), bins.cuda(), R, None, 0)
    assert torch.equal(got["rgb"], got32["rgb"]) and torch.equal(got["pre"], got32["pre"])
    pos, dirs = _midpoints(o, d, bins)
    _check(got, pos, dirs, torch.zeros(R * S, 32), f, "linf", "fp16 table")


@pytest.mark.parametrize("ray_mode", [True, False])
def test_density_half_alone_equals_full_call(ray_mode):
    """rgb = NULL skips the colour half (no head weights staged); density, pre-activation and geometry feature are those of the full call
    bit for bit, and the rgb buffer is left untouched"""
    f = _field("aabb").eval()
    R, S = 57, 48
    o, d, bins, cam = _rays(R, S, seed=8)
    if ray_mode:
        args = (o.cuda(), d.cuda(), bins.cuda(), R)
    else:
        pos, dirs = _midpoints(o, d, bins)
        args = (pos.cuda(), dirs.cuda(), None, R * S)
    full = _abi(f, *args, None, 0)
    half = _abi(f, *args, None, 0, want_rgb=False)
    for k in ("density", "pre", "geo"):
        assert bool(torch.isfinite(full[k]).all()) and torch.equal(half[k], full[k]), k
    assert bool(torch.isnan(half["rgb"]).all())
    if not ray_mode:   # point mode needs no directions without rgb
        nodir = _abi(f, args[0], None, None, R * S, None, 0, want_rgb=False)
        for k in ("density", "pre", "geo"):
            assert torch.equal(nodir[k], full[k]), k


def test_point_mode_equals_ray_mode_and_appearance_rows():
    """a RaySamples without this package's bin buffer runs in point mode: same outputs bit for bit; a per-ray appearance row equals
    the same rows per sample; stride 0 broadcasts"""
    import sdfstudio_b200 as sb

    f = _field("l2").train()
    R, S = 33, 48
    o, d, bins, cam = _rays(R, S, seed=7)
    rs = _samples(o, d, bins, cam)
    with torch.no_grad():
        ray = f(rs)
        object.__setattr__(rs, "_euclid_bins", None)
        n0 = sb._lib.launch_count()
        pt = f(rs)
        assert sb._lib.launch_count() - n0 == 1
    for k in (sb.FieldHeadNames.RGB, sb.FieldHeadNames.DENSITY):
        assert torch.equal(ray[k], pt[k]), k
    emb = f.embedding_appearance.embedding.weight.detach()
    per_ray = _abi(f, o.cuda(), d.cuda(), bins.cuda(), R, emb[cam.cuda()].contiguous(), 32)
    assert torch.equal(per_ray["rgb"].view(R, S, 3), ray[sb.FieldHeadNames.RGB])
    mean = emb.mean(0).contiguous()
    bcast = _abi(f, o.cuda(), d.cuda(), bins.cuda(), R, mean, 0)
    rows = _abi(f, o.cuda(), d.cuda(), bins.cuda(), R, mean.expand(R, -1).contiguous(), 32)
    assert torch.equal(bcast["rgb"], rows["rgb"])


def test_abi_misuse_returns_errors_without_launching():
    import sdfstudio_b200 as sb
    from sdfstudio_b200 import _lib

    lib = _lib.load()
    f = _field("linf")
    nb, nh = f.mlp_base, f.mlp_head
    x = torch.rand(10, 3, device="cuda")
    out = torch.empty(10, 3, device="cuda")
    p = nb.params.detach()

    bins = torch.rand(10, 49, device="cuda")

    def call(desc=None, grid=None, table=p[nb.n_net:].data_ptr(), base=p.data_ptr(), origins=x.data_ptr(), density=out.data_ptr(), n=10, bins=None,
             directions=x.data_ptr(), rgb=out.data_ptr(), head=nh.params.detach().data_ptr()):
        return lib.sdfb200_nerfacto_field_forward(nb.desc if grid is None else grid, f._desc(0) if desc is None else desc, table, base, head, None,
                                                  origins, directions, bins, n, None, 0, density, rgb, None, None, _lib.stream_ptr())

    n0 = sb._lib.launch_count()
    assert lib.sdfb200_nerfacto_field_forward(None, f._desc(0), None, None, None, None, None, None, None, 10, None, 0, None, None, None, None,
                                              None) == -1
    assert lib.sdfb200_nerfacto_field_forward(nb.desc, None, None, None, None, None, None, None, None, 10, None, 0, None, None, None, None,
                                              None) == -1
    for field, value in (("hidden_dim", 128), ("hidden_dim_color", 8), ("n_hidden_layers", 4), ("n_hidden_layers_color", 0), ("geo_feat_dim", 16),
                         ("appearance_dim", 40)):
        d = f._desc(0)
        setattr(d, field, value)
        assert call(desc=d) == -3, field
    torch_grid = sb.Encoding(3, {"otype": "HashGrid", "n_levels": 16, "n_features_per_level": 2, "log2_hashmap_size": 12, "base_resolution": 16,
                                 "per_level_scale": 1.3}, layout="torch")._desc_ref()
    assert call(grid=torch_grid) == -3
    assert call(table=None) == -1 and call(base=None) == -1 and call(origins=None) == -1 and call(density=None) == -1
    assert call(desc=f._desc(48), n=1) == -1                        # ray mode without bins
    assert call(desc=f._desc(48), n=1, bins=bins.data_ptr(), directions=None, rgb=None) == -1   # ray mode: the midpoints need directions
    assert call(directions=None) == -1 and call(head=None) == -1   # rgb needs directions and head weights
    assert call(n=-1) == -1
    assert call(table=None, base=None, origins=None, density=None, n=0) == 0   # n = 0: nothing to do
    assert sb._lib.launch_count() == n0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------ training
def _oracle_params64(f):
    ps = {"base": f.mlp_base.params, "head": f.mlp_head.params, "emb": f.embedding_appearance.embedding.weight}
    return {k: v.detach().double().cpu().requires_grad_(True) for k, v in ps.items()}


def _relu_margin(x01, dirs, app, base, head, spec):
    """per sample, the smallest |input| of any ReLU of either MLP (fp64): where it is within rounding of 0, fp32 and fp64 may take different
    sides of the kink and send that sample's gradient down different paths"""
    from oracle import hashgrid

    def walk(x, w, in_dim, hidden, n_hidden):
        in_pad = (in_dim + 15) // 16 * 16
        z = x @ w[: hidden * in_pad].view(hidden, in_pad)[:, :in_dim].t()
        m, o = z.abs().amin(1), hidden * in_pad
        for _ in range(n_hidden - 1):
            z = torch.relu(z) @ w[o: o + hidden * hidden].view(hidden, hidden).t()
            m, o = torch.minimum(m, z.abs().amin(1)), o + hidden * hidden
        return m, torch.relu(z) @ w[o: o + 16 * hidden].view(16, hidden).t()

    n_net = spec.n_base_net()
    feat = hashgrid.encode_tcnn_layout(x01, base[n_net:].view(-1, 2), spec.meta(), 2, False)
    m1, out = walk(feat, base[:n_net], spec.num_levels * 2, spec.hidden_dim, spec.num_layers - 1)
    h = torch.cat([onf.sh4_tcnn((dirs + 1.0) / 2.0 * 2 - 1), out[:, 1: 1 + spec.geo_feat_dim], app], dim=-1)
    m2, _ = walk(h, head, 16 + spec.geo_feat_dim + spec.appearance_embedding_dim, spec.hidden_dim_color, spec.num_layers_color - 1)
    return torch.minimum(m1, m2)


@pytest.mark.parametrize("norm", ["linf", "aabb"])
def test_training_composition_gradients(norm):
    """train mode with autograd: forward equals the kernel within fp32 noise; d loss / d (mlp_base.params, mlp_head.params, embedding) vs
    fp64 autograd over the oracle; the head's padded input columns get no gradient"""
    import sdfstudio_b200 as sb

    f = _field(norm, hidden=64, hidden_color=64).train()
    R, S = 48, 24
    o, d, bins, cam = _rays(R, S, seed=5)
    rs = _samples(o, d, bins, cam)
    out = f(rs)
    assert out[sb.FieldHeadNames.RGB].requires_grad
    g = torch.Generator().manual_seed(2)
    c_rgb, c_d = torch.randn(R, S, 3, generator=g), torch.randn(R, S, 1, generator=g)
    # samples sitting on a ReLU kink (within fp32 rounding) take no part in the loss
    spec = _spec(f)
    pos, dirs = _midpoints(o, d, bins)
    x01 = onf.normalize(pos, torch.tensor(AABB) if norm == "aabb" else None, None if norm == "aabb" else norm)   # fp32, as the composition
    p64 = _oracle_params64(f)
    app = p64["emb"][cam[:, None].expand(R, S).reshape(-1)]
    with torch.no_grad():
        keep = (_relu_margin(x01.double(), dirs.double(), app, p64["base"], p64["head"], spec) > 1e-4).double().view(R, S, 1)
    assert float(keep.mean()) > 0.95
    c_rgb, c_d = c_rgb * keep.float(), c_d * keep.float()
    dens, rgb = out[sb.FieldHeadNames.DENSITY], out[sb.FieldHeadNames.RGB]
    loss = (rgb * c_rgb.cuda()).sum() + (torch.log1p(dens) * c_d.cuda()).sum()
    params = [f.mlp_base.params, f.mlp_head.params, f.embedding_appearance.embedding.weight]
    grads = torch.autograd.grad(loss, params)
    with torch.no_grad():
        k = f(rs)
    assert _maxrel(rgb, k[sb.FieldHeadNames.RGB]) < 1e-5 and _maxrel(dens, k[sb.FieldHeadNames.DENSITY]) < 1e-5

    nb, nh = f.mlp_base, f.mlp_head
    dens64, _, geo64 = onf.density(x01.double(), p64["base"], spec)
    r = {"density": dens64, "rgb": onf.rgb(dirs.double(), geo64, app, p64["head"], spec)}
    loss64 = (r["rgb"].view(R, S, 3) * c_rgb.double()).sum() + (torch.log1p(r["density"].view(R, S, 1)) * c_d.double()).sum()
    g64 = torch.autograd.grad(loss64, [p64["base"], p64["head"], p64["emb"]])
    assert _maxrel(grads[0][: nb.n_net], g64[0][: nb.n_net]) < 2e-3
    assert _maxrel(grads[0][nb.n_net:], g64[0][nb.n_net:]) < 2e-3
    assert _maxrel(grads[1], g64[1]) < 2e-3
    assert _maxrel(grads[2], g64[2]) < 2e-3
    head_w0 = grads[1][: nh.hidden_dim * nh.in_pad].view(nh.hidden_dim, nh.in_pad)
    assert float(head_w0[:, nh.in_dim:].abs().max()) == 0.0


def test_angelo_shaped_step_with_background_merge():
    """SDFField (neus-facto case) + this field as the grid background, merged as forward_background_field_and_merge does
    (models/base_surface_model.py:266-290), weights, rgb render, L1 + eikonal, backward: loss and the gradients of both fields vs fp64"""
    import sdfstudio_b200 as sb

    spec, kw, o, d, cam, nears, fars, oracle, field = build_case("neusfacto_c1")
    R, S = 32, 24
    o, d, cam, nears, fars = o[:R], d[:R], cam[:R], nears[:R], fars[:R] * 2.5      # reach past the unit sphere
    if spec.contraction is not None:
        field.spatial_distortion = sb.SceneContraction(order=float("inf") if spec.contraction == "linf" else None)
    field.train()
    bg = _field("linf", hidden=64, hidden_color=64, seed=3, num_images=49).train()   # the case's camera indices reach 48
    bundle = make_bundle(o, d, cam, nears, fars)
    with torch.no_grad():
        rs = sb.UniformSampler(num_samples=S, train_stratified=False).eval()(bundle)
    target = torch.rand(R, 3, generator=torch.Generator().manual_seed(4))

    fo = field(rs, return_alphas=True)
    fb = bg(rs)
    inside = (rs.frustums.get_start_positions().norm(dim=-1, keepdim=True) < 1.0).float()
    alpha_bg = rs.get_alphas(fb[sb.FieldHeadNames.DENSITY])
    alpha = fo[sb.FieldHeadNames.ALPHA] * inside + (1.0 - inside) * alpha_bg
    rgb = fo[sb.FieldHeadNames.RGB] * inside + (1.0 - inside) * fb[sb.FieldHeadNames.RGB]
    assert 0 < float(inside.mean()) < 1
    w = sb.rays.weights_from_alphas(alpha)
    out_rgb = (w * rgb).sum(1)
    eik = ((fo[sb.FieldHeadNames.GRADIENT].norm(2, dim=-1) - 1) ** 2).mean()
    loss = (out_rgb - target.cuda()).abs().mean() + 0.1 * eik
    field.zero_grad()
    bg.zero_grad()
    loss.backward()

    # fp64 oracle of the same step
    of = OracleField(spec, {k: v for k, v in oracle.p.items()}, dtype=torch.float64)
    for v in of.p.values():
        if v.is_floating_point():
            v.requires_grad_(True)
    p64 = _oracle_params64(bg)
    bins = rs._euclid_bins.detach().double().cpu()
    starts, deltas = bins[:, :-1], bins[:, 1:] - bins[:, :-1]
    o64, d64 = o.double(), d.double()
    start_pos = (o64[:, None, :] + d64[:, None, :] * starts[..., None]).reshape(-1, 3)
    dirs = d64[:, None, :].expand(R, S, 3).reshape(-1, 3)
    x = scene_contraction(start_pos, spec.contraction).requires_grad_(True)
    h = of.forward_geonetwork(x)
    sdf, geo = h[:, :1], h[:, 1:]
    grads = torch.autograd.grad(sdf, x, torch.ones_like(sdf), create_graph=True)[0]
    of.training = True
    rgb_fg = of.get_colors(x, dirs, grads, geo, cam.reshape(R, 1).expand(R, S).reshape(-1))
    alpha_fg = of.get_alpha(dirs, deltas.reshape(-1, 1), sdf, grads)
    bspec = _spec(bg)
    mid = onf.midpoints(o.float()[:, None], d.float()[:, None], rs._euclid_bins.cpu()[:, :-1, None], rs._euclid_bins.cpu()[:, 1:, None])
    dens64, _, geo64 = onf.density(onf.normalize(mid.reshape(-1, 3), contraction="linf").double(), p64["base"], bspec)
    rb = {"density": dens64, "rgb": onf.rgb(dirs, geo64, p64["emb"][cam.reshape(R, 1).expand(R, S).reshape(-1)], p64["head"], bspec)}
    a64, rgb64 = onf.merge_background(alpha_fg, rgb_fg, start_pos, deltas.reshape(-1, 1), rb["density"][:, None], rb["rgb"])
    a64 = a64.view(R, S)
    T = torch.cumprod(torch.cat([torch.ones_like(a64[:, :1]), 1.0 - a64 + 1e-7], 1), 1)
    w64 = a64 * T[:, :-1]
    out64 = (w64[..., None] * rgb64.view(R, S, 3)).sum(1)
    loss64 = (out64 - target.double()).abs().mean() + 0.1 * ((grads.norm(2, dim=-1) - 1) ** 2).mean()
    loss64.backward()

    assert abs(float(loss.detach()) - float(loss64.detach())) < 5e-5 * max(1.0, abs(float(loss64.detach())))
    assert _maxrel(out_rgb, out64) < 5e-4
    for name, p in (("mlp_base.params", bg.mlp_base.params), ("mlp_head.params", bg.mlp_head.params),
                    ("embedding", bg.embedding_appearance.embedding.weight)):
        ref = {"mlp_base.params": p64["base"], "mlp_head.params": p64["head"], "embedding": p64["emb"]}[name].grad
        assert _maxrel(p.grad, ref) < 2e-3, (name, _maxrel(p.grad, ref))
    sd = dict(field.named_parameters())
    checked = 0
    for k, v in of.p.items():
        pk = {"hash_table": "encoding.hash_table" if spec.grid_layout == "torch" else "encoding.params"}.get(k, k)
        if not v.is_floating_point() or v.grad is None or pk not in sd or sd[pk].grad is None or float(v.grad.abs().max()) == 0.0:
            continue
        assert _maxrel(sd[pk].grad.reshape(v.grad.shape), v.grad) < 2e-3, k
        checked += 1
    assert checked >= 8, checked
    assert np.isfinite(float(loss.detach()))
