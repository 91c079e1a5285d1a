"""Training-path parity (GPU): the explicit backward kernels against fp64 autograd over the oracle restatement.

* hash-grid operator: first AND second-order backward (what `autograd.grad(..., create_graph=True)` + the eikonal loss need)
* alpha/density -> weights and the renderers: backward kernels vs torch autograd over the reference formulas
* one full SDFField training step (rgb + eikonal + normal-ish loss): parameter gradients vs the fp64 oracle
"""
import math

import pytest
import torch

from oracle import hashgrid
from oracle.field import FieldSpec, OracleField, init_params

from helpers import build_case, make_bundle, product_field

pytestmark = pytest.mark.gpu


def _maxrel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


# ------------------------------------------------------------------------------------------------------------------ grid
@pytest.mark.parametrize("layout,F", [("torch", 8), ("torch", 2), ("tcnn", 2), ("tcnn", 4)])
@pytest.mark.parametrize("delta", [1.0 / 4096.0, 0.03])
def test_grid_grouped_taps_equal_ungrouped(layout, F, delta):
    """Encoding.point_groups(7): the numerical-gradient batch (sample + six +-delta taps, tap g of sample s at row g * N + s) through the
    grouped kernels equals the ungrouped operator on the same points -- forward bit for bit, table gradient up to the order of the atomic
    sums -- both when the taps share their cell (delta = finest-level cell) and when they do not (delta = 0.03), with masked levels."""
    import sdfstudio_b200 as sb

    L, log2T, base, scale = 8, 12, 8, 1.5
    cfg = {"otype": "HashGrid", "n_levels": L, "n_features_per_level": F, "log2_hashmap_size": log2T, "base_resolution": base, "per_level_scale": scale,
           "interpolation": "Linear"}
    enc = sb.Encoding(3, cfg, layout=layout).cuda()
    enc.set_active_levels(6)
    g = torch.Generator().manual_seed(11)
    with torch.no_grad():
        enc.table.copy_(torch.randn(enc.table.shape, generator=g) * 0.3)
    N = 1000
    x = torch.rand(N, 3, generator=g) * 0.9 + 0.05
    offs = torch.tensor([[0, 0, 0], [delta, 0, 0], [-delta, 0, 0], [0, delta, 0], [0, -delta, 0], [0, 0, delta], [0, 0, -delta]], dtype=torch.float32)
    pts = (x[None] + offs[:, None, :]).reshape(-1, 3).cuda()
    r = torch.randn(7 * N, L * F, generator=g).cuda()

    def run(grouped):
        enc.zero_grad(set_to_none=True)
        if grouped:
            with enc.point_groups(7):
                out = enc(pts)
        else:
            out = enc(pts)
        (out * r).sum().backward()
        return out.detach(), enc.table.grad.detach().clone()

    out_u, gt_u = run(False)
    launches0 = sb._lib.launch_count()
    out_g, gt_g = run(True)
    assert sb._lib.launch_count() - launches0 == 2          # one grouped forward, one grouped backward
    assert torch.equal(out_g, out_u)
    assert float(out_u[:, 6 * F:].abs().max()) == 0.0 and float(out_u[:, : 6 * F].abs().max()) > 0
    scale_g = float(gt_u.abs().max())
    assert float((gt_g - gt_u).abs().max()) <= 2e-6 * scale_g, float((gt_g - gt_u).abs().max()) / scale_g
    # a batch that is not a multiple of the group size falls back to the ungrouped kernels
    with enc.point_groups(7):
        assert torch.equal(enc(pts[:-1]), out_u[:-1])


@pytest.mark.parametrize("layout", ["torch", "tcnn"])
@pytest.mark.parametrize("smooth", [True, False])
def test_grid_double_backward(layout, smooth):
    import sdfstudio_b200 as sb

    L, F, log2T, base, scale = 6, 2, 10, 4, 1.6
    cfg = {"otype": "HashGrid", "n_levels": L, "n_features_per_level": F, "log2_hashmap_size": log2T, "base_resolution": base,
           "per_level_scale": scale, "interpolation": "Smoothstep" if smooth else "Linear"}
    enc = sb.Encoding(3, cfg, layout=layout).cuda()
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        enc.table.copy_(torch.randn(enc.table.shape, generator=g) * 0.3)
    N = 513
    x = (torch.rand(N, 3, generator=g) * 0.96 + 0.02)
    r1, r2, q = torch.randn(N, L * F, generator=g), torch.randn(N, L * F, generator=g), torch.randn(N, 3, generator=g)

    def run(encode, x_, table_, cast):
        x_ = x_.clone().requires_grad_(True)
        out = encode(x_)
        first = torch.autograd.grad((out * cast(r1)).sum(), x_, create_graph=True)[0]
        loss = (first * cast(q)).sum() + 0.25 * (first * first).sum() + (out * cast(r2)).sum()
        gx, gt = torch.autograd.grad(loss, [x_, table_])
        return out, first, gx, gt

    out_c, first_c, gx_c, gt_c = run(lambda t: enc(t), x.cuda(), enc.table, lambda t: t.cuda())

    table64 = enc.table.detach().double().cpu().reshape(-1, F).requires_grad_(True)
    if layout == "torch":
        max_res = base * scale ** (L - 1)
        scal = hashgrid.torch_layout_scalings(L, base, max_res)
        ref = lambda t: hashgrid.encode_torch_layout(t, table64, scal, 1 << log2T, smooth)  # noqa: E731
    else:
        meta = hashgrid.tcnn_grid_meta(L, F, log2T, base, scale)
        ref = lambda t: hashgrid.encode_tcnn_layout(t, table64, meta, F, smooth)  # noqa: E731
    out_r, first_r, gx_r, gt_r = run(ref, x.double(), table64, lambda t: t.double())

    assert _maxrel(out_c, out_r) < 1e-5
    assert _maxrel(first_c, first_r) < 1e-4                      # first backward (dx)
    assert _maxrel(gt_c.reshape(-1, F), gt_r) < 2e-4             # d loss / d table incl. the second-order term
    if smooth:                                                    # linear interpolation: d2/dx2 has only cross terms, still checked
        assert _maxrel(gx_c, gx_r) < 5e-4
    else:
        assert _maxrel(gx_c, gx_r) < 5e-4


# ------------------------------------------------------------------------------------------------------------------ weights / render
def _ref_weights_alpha(a):
    T = torch.cumprod(torch.cat([torch.ones_like(a[:, :1]), 1.0 - a + 1e-7], 1), 1)
    return a * T[:, :-1], T


def test_weights_and_render_backward():
    import sdfstudio_b200 as sb
    from sdfstudio_b200.rays import weights_from_alphas, weights_from_density

    g = torch.Generator().manual_seed(11)
    R, S = 97, 77
    alphas = torch.rand(R, S, 1, generator=g) ** 3
    alphas[:5, 10] = 1.0                                            # saturated samples (f = 1e-7)
    rgb = torch.rand(R, S, 3, generator=g)
    nrm = torch.randn(R, S, 3, generator=g)
    bins = torch.cumsum(torch.rand(R, S + 1, generator=g) * 0.05 + 0.01, 1)
    bgc = torch.rand(R, 3, generator=g)
    c_rgb, c_d, c_n, c_a, c_w, c_t = (torch.randn(*s, generator=g) for s in [(R, 3), (R, 1), (R, 3), (R, 1), (R, S, 1), (R, 1)])

    # --- reference (fp64 autograd over the reference formulas)
    a64, rgb64, n64 = alphas.double().requires_grad_(True), rgb.double().requires_grad_(True), nrm.double().requires_grad_(True)
    w, T = _ref_weights_alpha(a64[..., 0])
    steps = ((bins[:, :-1] + bins[:, 1:]) / 2).double()
    acc = w.sum(1, keepdim=True)
    o_rgb = (w[..., None] * rgb64).sum(1) + bgc.double() * (1 - acc)
    o_depth = ((w * steps).sum(1, keepdim=True) / (acc + 1e-10)).clamp(steps.min(), steps.max())
    o_n = (w[..., None] * n64).sum(1)
    loss = (o_rgb * c_rgb.double()).sum() + (o_depth * c_d.double()).sum() + (o_n * c_n.double()).sum() + (acc * c_a.double()).sum() \
        + (w * c_w[..., 0].double()).sum() + (T[:, -1:] * c_t.double()).sum()
    ga_r, gr_r, gn_r = torch.autograd.grad(loss, [a64, rgb64, n64])

    # --- fused op
    class _RS:  # minimal ray_samples carrying the bin buffer
        _euclid_bins = bins.cuda()

    ac, rc, nc = alphas.cuda().requires_grad_(True), rgb.cuda().requires_grad_(True), nrm.cuda().requires_grad_(True)
    res = sb.render_from_alphas(ac, rc, nc, _RS, bgc.cuda(), training=True)
    loss_c = (res["rgb"] * c_rgb.cuda()).sum() + (res["depth"] * c_d.cuda()).sum() + (res["normal"] * c_n.cuda()).sum() \
        + (res["accumulation"] * c_a.cuda()).sum() + (res["weights"] * c_w.cuda()).sum() + (res["bg_transmittance"] * c_t.cuda()).sum()
    assert abs(float(loss_c.detach()) - float(loss.detach())) < 1e-3 * max(1.0, abs(float(loss)))
    ga, gr, gn = torch.autograd.grad(loss_c, [ac, rc, nc])
    sat = alphas[..., 0] >= 1.0                                     # d/dalpha through 1/(1e-7): compare those relatively
    assert _maxrel(gr, gr_r) < 1e-5 and _maxrel(gn, gn_r) < 1e-5
    assert _maxrel(ga[..., 0].cpu()[~sat], ga_r[..., 0][~sat]) < 2e-4
    assert _maxrel(ga[..., 0].cpu()[sat], ga_r[..., 0][sat]) < 2e-3

    # --- separate modules (RaySamples.get_weights_and_transmittance_from_alphas + the four renderers)
    ac2, rc2, nc2 = alphas.cuda().requires_grad_(True), rgb.cuda().requires_grad_(True), nrm.cuda().requires_grad_(True)
    w2, T2 = weights_from_alphas(ac2, True)
    o_rgb2 = sb.RGBRenderer(background_color=bgc.cuda()).train()(rc2, w2)
    o_d2 = sb.DepthRenderer("expected")(w2, _RS)
    o_n2 = sb.SemanticRenderer.forward(nc2, w2)
    o_a2 = sb.AccumulationRenderer.forward(w2)
    loss2 = (o_rgb2 * c_rgb.cuda()).sum() + (o_d2 * c_d.cuda()).sum() + (o_n2 * c_n.cuda()).sum() + (o_a2 * c_a.cuda()).sum() \
        + (w2 * c_w.cuda()).sum() + (T2[:, -1] * c_t.cuda()).sum()
    ga2, gr2, gn2 = torch.autograd.grad(loss2, [ac2, rc2, nc2])
    assert _maxrel(gr2, gr_r) < 1e-5 and _maxrel(gn2, gn_r) < 1e-5
    assert _maxrel(ga2[..., 0].cpu()[~sat], ga_r[..., 0][~sat]) < 2e-4

    # --- density -> weights (VolSDF)
    dens = (torch.rand(R, S, 1, generator=g) * 30.0)
    d64 = dens.double().requires_grad_(True)
    delta = (bins[:, 1:] - bins[:, :-1]).double()
    dd = delta * d64[..., 0]
    Tr = torch.exp(-torch.cat([torch.zeros(R, 1, dtype=torch.float64), torch.cumsum(dd, 1)[:, :-1]], 1))
    wd = (1 - torch.exp(-dd)) * Tr
    gd_r = torch.autograd.grad((wd * c_w[..., 0].double()).sum(), d64, retain_graph=True)[0]
    dc = dens.cuda().requires_grad_(True)
    wc = weights_from_density(bins.cuda(), dc)
    assert _maxrel(wc[..., 0], wd) < 1e-5
    gd = torch.autograd.grad((wc * c_w.cuda()).sum(), dc)[0]
    assert _maxrel(gd, gd_r) < 2e-4
    # transmittance gradient of the density form: VolSDF composites its background model with transmittance[:, -1]
    # (models/volsdf.py:67-68 + base_surface_model.py:329); every column must back-propagate, not only the weights
    c_T = torch.randn(R, S, generator=g)
    gd_rT = torch.autograd.grad((wd * c_w[..., 0].double()).sum() + (Tr * c_T.double()).sum() + 3.0 * Tr[:, -1].sum(), d64)[0]
    dc2 = dens.cuda().requires_grad_(True)
    wc2, Tc2 = weights_from_density(bins.cuda(), dc2, True)
    assert _maxrel(Tc2[..., 0], Tr) < 1e-5
    gdT = torch.autograd.grad((wc2 * c_w.cuda()).sum() + (Tc2[..., 0] * c_T.cuda()).sum() + 3.0 * Tc2[:, -1].sum(), dc2)[0]
    assert _maxrel(gdT, gd_rT) < 2e-4
    # ... and the alpha form through interior transmittance columns
    a64b = alphas.double().requires_grad_(True)
    wb, Tb = _ref_weights_alpha(a64b[..., 0])
    c_T1 = torch.randn(R, S + 1, generator=g)
    ga_rT = torch.autograd.grad((Tb * c_T1.double()).sum() + (wb * c_w[..., 0].double()).sum(), a64b)[0]
    ac3 = alphas.cuda().requires_grad_(True)
    w3, T3 = weights_from_alphas(ac3, True)
    gaT = torch.autograd.grad((T3[..., 0] * c_T1.cuda()).sum() + (w3 * c_w.cuda()).sum(), ac3)[0]
    assert _maxrel(gaT[..., 0].cpu()[~sat], ga_rT[..., 0][~sat]) < 2e-4


# ------------------------------------------------------------------------------------------------------------------ SDFField step
def _oracle_loss(of: OracleField, spec, o, d, cam, starts, deltas, bins, target, contraction_fn):
    """rgb L1 + eikonal + a normal term, differentiable fp64 composition of the oracle's restated methods."""
    R, S = starts.shape
    pos = (o[:, None, :] + d[:, None, :] * starts[..., None]).reshape(-1, 3)
    dirs = d[:, None, :].expand(R, S, 3).reshape(-1, 3)
    x = contraction_fn(pos).requires_grad_(True)
    h = of.forward_geonetwork(x)
    sdf, geo = h[:, :1], h[:, 1:]
    grads = torch.autograd.grad(sdf, x, torch.ones_like(sdf), create_graph=True)[0]
    of.training = True
    rgb = of.get_colors(x, dirs, grads, geo, cam.reshape(R, 1).expand(R, S).reshape(-1))
    alphas = of.get_alpha(dirs, deltas.reshape(-1, 1), sdf, grads).view(R, S)
    w, T = _ref_weights_alpha(alphas)
    acc = w.sum(1, keepdim=True)
    out_rgb = (w[..., None] * rgb.view(R, S, 3)).sum(1) + (1 - acc)            # white background
    normals = torch.nn.functional.normalize(grads, p=2, dim=-1).view(R, S, 3)
    out_n = (w[..., None] * normals).sum(1)
    steps = (bins[:, :-1] + bins[:, 1:]) / 2
    depth = (w * steps).sum(1, keepdim=True) / (acc + 1e-10)
    eik = ((grads.norm(2, dim=-1) - 1) ** 2).mean()
    loss = (out_rgb - target).abs().mean() + 0.1 * eik + 0.05 * (out_n * out_n).sum(-1).mean() + 0.01 * depth.mean() + 0.02 * T[:, -1].mean()
    return loss, out_rgb


@pytest.mark.parametrize("gemm", ["aten", "tc"])
@pytest.mark.parametrize("case", ["neusfacto_c1", "bakedsdf_small"])
def test_sdffield_training_step(case, gemm):
    """gemm="aten": dense layers through ATen (fp32, the reference's own arithmetic); gemm="tc": forward, input-gradient and
    weight-gradient GEMMs -- incl. the eikonal double backward -- on the tensor-core kernels (linear_ops.py, bf16x3)."""
    import sdfstudio_b200 as sb

    spec, kw, o, d, cam, nears, fars, oracle, field = build_case(case)
    field.config.train_gemm, field.config.precision = gemm, ("bf16x3" if gemm == "tc" else "fp32")
    R, S = 48, 12
    o, d, cam, nears, fars = o[:R], d[:R], cam[:R], nears[:R], fars[:R]
    if spec.contraction is not None:
        field.spatial_distortion = sb.SceneContraction(order=float("inf") if spec.contraction == "linf" else None)
    field.train()
    bundle = make_bundle(o, d, cam, nears, fars)
    with torch.no_grad():
        rs = sb.UniformSampler(num_samples=S, train_stratified=False).eval()(bundle)
    g = torch.Generator().manual_seed(3)
    target = torch.rand(R, 3, generator=g)

    # ---- product: one training step's loss + backward
    fo = field(rs, return_alphas=True)
    res = sb.render_from_alphas(fo[sb.FieldHeadNames.ALPHA], fo[sb.FieldHeadNames.RGB], fo[sb.FieldHeadNames.NORMAL], rs,
                                torch.ones(3, device="cuda"), training=True)
    grads_c = fo[sb.FieldHeadNames.GRADIENT]
    eik = ((grads_c.norm(2, dim=-1) - 1) ** 2).mean()
    loss_c = (res["rgb"] - target.cuda()).abs().mean() + 0.1 * eik + 0.05 * (res["normal"] ** 2).sum(-1).mean() \
        + 0.01 * res["depth"].mean() + 0.02 * res["bg_transmittance"].mean()
    field.zero_grad()
    loss_c.backward()

    # ---- oracle fp64
    params = {k: v for k, v in oracle.p.items()}
    of = OracleField(spec, params, dtype=torch.float64)
    if "mask_level" in kw:
        of.update_mask(kw["mask_level"])
    for k, v in of.p.items():
        if v.is_floating_point():
            v.requires_grad_(True)
    bins = rs._euclid_bins.detach().double().cpu()
    starts, deltas = bins[:, :-1], bins[:, 1:] - bins[:, :-1]
    from oracle.field import scene_contraction
    loss_r, rgb_r = _oracle_loss(of, spec, o.double(), d.double(), cam, starts, deltas, bins, target.double(),
                                 lambda p: scene_contraction(p, spec.contraction))
    loss_r.backward()

    assert abs(float(loss_c.detach()) - float(loss_r.detach())) < (5e-5 if gemm == "aten" else 2e-4) * max(1.0, abs(float(loss_r.detach())))
    assert _maxrel(res["rgb"], rgb_r) < 5e-4          # fp32 cancellation in the NeuS alpha (prev_cdf - next_cdf), same as the reference in fp32
    name_map = {"hash_table": "encoding.hash_table" if spec.grid_layout == "torch" else "encoding.params"}
    sd = dict(field.named_parameters())
    checked, errs = 0, {}
    for k, v in of.p.items():
        if not v.is_floating_point() or v.grad is None:
            continue
        pk = name_map.get(k, k)
        if pk not in sd or sd[pk].grad is None:
            continue
        gc, gr = sd[pk].grad, v.grad
        if float(gr.abs().max()) == 0.0:
            assert float(gc.abs().max()) < 1e-9, k
            continue
        err = _maxrel(gc.reshape(gr.shape), gr)
        errs[k] = err
        checked += 1
    bad = {k: f"{v:.2e}" for k, v in errs.items() if v >= 2e-3}
    assert not bad, f"grad max-rel errors: {bad} (all: { {k: f'{v:.1e}' for k, v in errs.items()} })"
    assert checked >= 8, checked

    # the no-grad path of the SAME module (fused kernels) agrees with the differentiable forward
    with torch.no_grad():
        fo2 = field(rs, return_alphas=True)
    for key in (sb.FieldHeadNames.RGB, sb.FieldHeadNames.SDF, sb.FieldHeadNames.GRADIENT, sb.FieldHeadNames.ALPHA):
        assert _maxrel(fo2[key], fo[key]) < (1e-4 if gemm == "aten" else 5e-4), key


# ------------------------------------------------------------------------------------------------------------------ training GEMMs
@pytest.mark.parametrize("P,N,K", [(1000, 256, 71), (4097, 257, 256), (333, 3, 256), (2500, 256, 321), (77, 16, 16)])
@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_training_gemm_primitives(P, N, K, precision):
    """sdfb200_gemm_nt / _nn / _tn (tensor cores) against fp64 matmuls: Y = X W^T, dX = dY W, dW = dY^T X."""
    from sdfstudio_b200 import linear_ops as lo

    g = torch.Generator().manual_seed(P + N + K)
    x = torch.randn(P, K, generator=g) * 0.5
    W = torch.randn(N, K, generator=g) / K**0.5
    gy = torch.randn(P, N, generator=g)
    xp, gyp = lo.pad_cols(x).cuda(), lo.pad_cols(gy).cuda()
    tol = 3e-5 if precision == "bf16x3" else 8e-3

    def relerr(a, ref, scale):
        return float((a.double().cpu() - ref).abs().max()) / scale

    y = lo.gemm_nt(xp, W.cuda(), precision)
    assert y.shape == (P, lo.pad16(N)) and float(y[:, N:].abs().max() if N % 16 else 0.0) == 0.0
    assert relerr(y[:, :N], x.double() @ W.double().t(), float((x.abs().double() @ W.abs().double().t()).max())) < tol
    dx = lo.gemm_nn(gyp, W.cuda(), precision)
    assert dx.shape == (P, lo.pad16(K))
    assert relerr(dx[:, :K], gy.double() @ W.double(), float((gy.abs().double() @ W.abs().double()).max())) < tol
    dW = lo.gemm_tn(gyp, xp, N, K, precision)
    assert dW.shape == (N, K)
    assert relerr(dW, gy.double().t() @ x.double(), float((gy.abs().double().t() @ x.abs().double()).max())) < tol
    # determinism of the weight gradient (fixed-order reduction of the per-SM partial sums)
    assert torch.equal(dW, lo.gemm_tn(gyp, xp, N, K, precision))


@pytest.mark.parametrize("act", [0, 1, 2])
def test_training_linear_first_and_second_order(act):
    """linear_ops.linear (fused bias + activation epilogue) under autograd, incl. create_graph=True double backward (the eikonal pattern:
    a loss on d out / d x), against the same composition in fp64 ATen."""
    import torch.nn.functional as F

    from sdfstudio_b200 import linear_ops as lo

    g = torch.Generator().manual_seed(5 + act)
    P, K, H = 777, 39, 256
    x0 = torch.randn(P, K, generator=g) * 0.3
    W0, b0 = torch.randn(H, K, generator=g) / K**0.5 * 0.3, torch.randn(H, generator=g) * 0.02
    W1, b1 = torch.randn(1, H, generator=g) / H**0.5, torch.randn(1, generator=g) * 0.1
    coef = torch.randn(P, generator=g)

    def run(lin, x, params, dt):
        W0_, b0_, W1_, b1_ = params
        h = lin(x, W0_, b0_, act)
        y = lin(h, W1_, b1_, 0)[:, :1]
        (gx,) = torch.autograd.grad(y.sum(), x, create_graph=True)
        loss = (y[:, 0] * coef.to(y.device, dt)).sum() + ((gx[:, :K].norm(dim=-1) - 1) ** 2).mean()
        return loss, torch.autograd.grad(loss, params)

    def ref_lin(x, W, b, a):
        z = F.linear(x, W, b)
        return F.softplus(z, beta=100) if a == 1 else (torch.relu(z) if a == 2 else z)

    p64 = [t.double().requires_grad_(True) for t in (W0, b0, W1, b1)]
    loss_r, grads_r = run(ref_lin, x0.double().requires_grad_(True), p64, torch.float64)
    pc = [t.cuda().requires_grad_(True) for t in (W0, b0, W1, b1)]
    xc = lo.pad_cols(x0).cuda().requires_grad_(True)
    loss_c, grads_c = run(lambda x, W, b, a: lo.linear(x, W, b, a, "bf16x3"), xc, pc, torch.float32)
    assert abs(float(loss_c) - float(loss_r)) < 1e-4 * max(1.0, abs(float(loss_r)))
    for gc, gr, name in zip(grads_c, grads_r, ("W0", "b0", "W1", "b1")):
        assert _maxrel(gc, gr) < 2e-3, (name, _maxrel(gc, gr))


# ------------------------------------------------------------------------------------------------------------------ proposal network
@pytest.mark.parametrize("contraction", [None, "linf"])
def test_density_field_training_gradients(contraction):
    """HashMLPDensityField in training mode: density and d loss / d params (grid tail + MLP head) vs fp64 autograd over the oracle."""
    import sdfstudio_b200 as sb
    from oracle.density import density_field

    aabb = torch.tensor([[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]])
    sd = sb.SceneContraction(order=float("inf")) if contraction else None
    f = sb.HashMLPDensityField(aabb, num_layers=2, hidden_dim=64, spatial_distortion=sd, num_levels=5, max_res=128, base_res=16, log2_hashmap_size=12).cuda().train()
    nb = f.mlp_base
    g = torch.Generator().manual_seed(9)
    with torch.no_grad():
        nb.params[nb.n_net:].copy_(torch.randn(nb.n_grid, generator=g) * 0.3)
    pos = (torch.rand(37, 11, 3, generator=g) * 2 - 1) * (1.8 if contraction else 0.98)
    coef = torch.randn(37, 11, 1, generator=g)
    dens = f.density_fn(pos.cuda())
    assert dens.requires_grad
    loss = (dens * coef.cuda()).sum() + 0.1 * (dens ** 2).mean()
    (gp,) = torch.autograd.grad(loss, [nb.params])

    p64 = nb.params.detach().double().cpu().requires_grad_(True)
    import numpy as np

    scale = float(np.exp((np.log(128) - np.log(16)) / 4))
    d64, _ = density_field(pos.double(), p64[: nb.n_net], p64[nb.n_net:], 64, 1, 5, 2, 12, 16, scale, aabb=None if contraction else aabb.double(),
                           contraction=contraction)
    loss64 = (d64 * coef.double()).sum() + 0.1 * (d64 ** 2).mean()
    (g64,) = torch.autograd.grad(loss64, [p64])
    assert _maxrel(dens, d64) < 2e-5
    assert _maxrel(gp[: nb.n_net], g64[: nb.n_net]) < 5e-4
    assert _maxrel(gp[nb.n_net:], g64[nb.n_net:]) < 5e-4
    # the no-grad path of the same module (fused kernel) agrees with the differentiable forward
    with torch.no_grad():
        assert _maxrel(f.density_fn(pos.cuda()), dens) < 1e-5
