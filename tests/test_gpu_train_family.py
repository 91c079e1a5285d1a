"""-m gpu: the SDFField training step (sdf_field_train.py: autograd over this package's grid operator and, at train_gemm="tc", the bf16x3
tensor-core GEMMs of linear_ops.py) against fp64 autograd over the oracle, one switch at a time from the presets' shapes, then at the size
of the angelo-train-8192 workload.

Numerical gradients divide sdf differences by 2 delta and the curvature term divides by delta^2, so no fixed relative bound fits every
quantity.  Each one is held to the repo's noise bound (helpers.assert_within_noise): |cuda - fp64 oracle| <= max(4 x |fp32 oracle - fp64
oracle|, floor x max|fp64 oracle|), per quantity and per parameter tensor, where the fp32 oracle is the same composition run in float32."""
import contextlib
import math
from dataclasses import replace

import pytest
import torch

from oracle import cases, hashgrid
from oracle.field import OracleField, init_params, scene_contraction

from helpers import assert_within_noise, make_bundle, product_field

pytestmark = pytest.mark.gpu

R, S = 48, 16
CURVATURE = 5e-4                                      # neuralangelo / bakedangelo curvature_loss_multi
FACTOR = 4.0
# floor of the noise bound, relative to the quantity's scale.  ATen fp32 does the oracle's own arithmetic.  A numerical gradient divides the
# bf16x3 rounding of the sdf by 2 delta = 0.004: measured on an H100 (700 W), up to 5e-3 of the gradients' scale and 3e-3 of a parameter
# gradient's, while the steps with analytic gradients stay within 2e-3.  The curvature term divides by delta^2: up to 1.6e-2 of glin0's
# weight gradient with it
FLOOR = {"aten": 1e-4, "tc": 2e-3}
FLOOR_TC_NUMERICAL = 1.5e-2
FLOOR_TC_CURVATURE = 4e-2

# name -> (case of oracle/cases.py, FieldSpec changes, kwargs changes, options).  Options: curvature (the curvature term on sampled_sdf),
# render "density" (alpha = 1 - exp(-sigma delta) from the Laplace density, as VolSDF composites), cos_anneal (NeuS get_alpha ratio)
CASES = {
    # numerical gradients, F = 8, mask at level 6 of 8, appearance in training, 4 colour layers, PE off
    "angelo_small": ("angelo_small", {}, {}, {}),
    "angelo_curvature": ("angelo_small", {}, {}, {"curvature": True}),
    # bakedangelo-shaped: ref-nerf heads, L-inf contraction and off-axis PE on the numerical path
    "bakedangelo": ("bakedsdf_small", {"use_numerical_gradients": True}, {"mask_level": 10, "num_grad_delta": 0.002}, {"curvature": True}),
    # 8 layers, skip at 4, no grid, inside-outside, weight norm: the double backward runs through 9 GEMMs
    "volsdf_stock": ("volsdf_stock", {}, {}, {"render": "density"}),
    # tcnn layout (encoding.params): dense coarse levels, hashed fine ones
    "neusfacto_tcnn": ("neusfacto_c1", {"grid_layout": "tcnn"}, {}, {}),
    "neusfacto_l2": ("neusfacto_l2", {}, {}, {}),
    # widths 128 / 192 / 96, 3 colour layers, F = 4, reflections + n.v without the diffuse / tint heads, appearance in training
    "mixed_heads": ("mixed_heads", {}, {}, {}),
    "neusfacto_anneal": ("neusfacto_c1", {}, {}, {"cos_anneal": 0.3}),
}


class _Case:
    """The product field of a case in training mode at one GEMM setting, and fp32 / fp64 oracles with the same parameters and switches."""

    def __init__(self, name, gemm):
        import sdfstudio_b200 as sb

        base, spec_changes, kw_changes, self.opt = CASES[name]
        spec, kw = cases.CASES[base] if base in cases.CASES else cases.CPU_CASES[base]
        self.name, self.gemm = name, gemm
        self.spec, self.kw = replace(spec, **spec_changes), {**kw, **kw_changes}
        _, _, o, d, cam, nears, fars = cases.case_inputs(base)
        self.o, self.d, self.cam, self.nears, self.fars = o[:R], d[:R], cam[:R], nears[:R], fars[:R]
        self.params = init_params(self.spec, **cases.init_kwargs(self.kw))
        f = product_field(self.spec, self.params, self.kw, precision="bf16x3" if gemm == "tc" else "fp32")
        f.config.train_gemm = gemm
        if self.spec.contraction is not None:
            f.spatial_distortion = sb.SceneContraction(order=float("inf") if self.spec.contraction == "linf" else None)
        f.set_cos_anneal_ratio(self.opt.get("cos_anneal", 1.0))
        self.field = f.train()

    def oracle(self, dtype):
        """OracleField in training mode whose floating-point parameters are autograd leaves"""
        of = OracleField(self.spec, self.params, dtype=dtype)
        if "mask_level" in self.kw:
            of.update_mask(self.kw["mask_level"])
        if "num_grad_delta" in self.kw:
            of.numerical_gradients_delta = self.kw["num_grad_delta"]
        of.cos_anneal_ratio = self.opt.get("cos_anneal", 1.0)
        of.training = True
        for k, v in of.p.items():
            if v.is_floating_point() and k != "laplace_density.beta_min":       # a constant of the reference (requires_grad=False)
                v.requires_grad_(True)
        return of

    def samples(self):
        import sdfstudio_b200 as sb

        with torch.no_grad():
            return sb.SpacedSampler(self.kw.get("spacing", "uniform"), None, num_samples=S).eval()(
                make_bundle(self.o, self.d, self.cam, self.nears, self.fars))

    def floor(self):
        if self.gemm == "tc" and self.spec.use_numerical_gradients:
            return FLOOR_TC_CURVATURE if self.opt.get("curvature") else FLOOR_TC_NUMERICAL
        return FLOOR[self.gemm]

    def table_name(self):
        return "encoding.hash_table" if self.spec.grid_layout == "torch" else "encoding.params"


def _target():
    return torch.rand(R, 3, generator=torch.Generator().manual_seed(3))


def _loss(out_rgb, target, grads, normal, depth, bg_t, sdf=None, sampled=None, delta=None):
    """rgb L1 + eikonal + normal, depth and background terms (+ the curvature term of neuralangelo / bakedangelo, models/bakedangelo.py:166-177)"""
    eik = ((grads.norm(2, dim=-1) - 1) ** 2).mean()
    loss = (out_rgb - target).abs().mean() + 0.1 * eik + 0.05 * (normal * normal).sum(-1).mean() + 0.01 * depth.mean() + 0.02 * bg_t.mean()
    if sampled is not None:
        curvature = (sampled.reshape(*sdf.shape[:2], 3, 2).sum(-1) - 2 * sdf) / (delta * delta)
        loss = loss + CURVATURE * curvature.abs().mean()
    return loss


def _oracle_step(c: _Case, of: OracleField, bins, target):
    """The training step of `c` composed from the oracle's restated methods under torch autograd, in the oracle's dtype: the geo network at x
    and, for numerical gradients, at the six taps x +- delta e_i in the reference's order (+x, -x, +y, -y, +z, -z: sdf_field.py:424-452,
    :640-645), the appearance embedding indexed by camera, the hash mask, the annealed NeuS alpha (or the density's), alpha compositing on a
    white background and the loss of _loss."""
    dt, spec = of.dtype, c.spec
    o, d, bins, target = c.o.to(dt), c.d.to(dt), bins.to(dt), target.to(dt)
    starts, deltas = bins[:, :-1], bins[:, 1:] - bins[:, :-1]
    pos = (o[:, None, :] + d[:, None, :] * starts[..., None]).reshape(-1, 3)
    dirs = d[:, None, :].expand(R, S, 3).reshape(-1, 3)
    x = scene_contraction(pos, spec.contraction)
    sampled = None
    if spec.use_numerical_gradients:
        h = of.forward_geonetwork(x)
        grads, ps = of.gradient(x, skip_spatial_distortion=True, return_sdf=True)
        sampled = ps.view(6, R, S).permute(1, 2, 0)
    else:
        x = x.requires_grad_(True)
        h = of.forward_geonetwork(x)
        grads = torch.autograd.grad(h[:, :1], x, torch.ones_like(h[:, :1]), create_graph=True)[0]
    sdf, geo = h[:, :1], h[:, 1:]
    rgb = of.get_colors(x, dirs, grads, geo, c.cam.reshape(R, 1).expand(R, S).reshape(-1))
    if c.opt.get("render") == "density":
        alphas = 1.0 - torch.exp(-deltas.reshape(-1, 1) * of.laplace_density(sdf))
    else:
        alphas = of.get_alpha(dirs, deltas.reshape(-1, 1), sdf, grads)
    alphas = alphas.view(R, S)
    T = torch.cumprod(torch.cat([torch.ones_like(alphas[:, :1]), 1.0 - alphas + 1e-7], 1), 1)
    w = alphas * T[:, :-1]
    acc = w.sum(1, keepdim=True)
    out_rgb = (w[..., None] * rgb.view(R, S, 3)).sum(1) + (1 - acc)
    normal = (w[..., None] * torch.nn.functional.normalize(grads, p=2, dim=-1).view(R, S, 3)).sum(1)
    depth = (w * (bins[:, :-1] + bins[:, 1:]) / 2).sum(1, keepdim=True) / (acc + 1e-10)
    sdf3 = sdf.view(R, S, 1)
    loss = _loss(out_rgb, target, grads, normal, depth, T[:, -1], sdf3, sampled if c.opt.get("curvature") else None, of.numerical_gradients_delta)
    loss.backward()
    out = {"loss": loss.detach().reshape(1), "rgb": out_rgb.detach(), "sdf": sdf3.detach(), "gradients": grads.detach().view(R, S, 3),
           "alphas": alphas.detach()[..., None]}
    if sampled is not None:
        out["sampled_sdf"] = sampled.detach()
    grads_p = {k: v.grad for k, v in of.p.items() if v.is_floating_point() and v.grad is not None}
    return out, grads_p


def _product_step(c: _Case, rs, target):
    import sdfstudio_b200 as sb

    H = sb.FieldHeadNames
    f = c.field
    f.zero_grad(set_to_none=True)
    fo = f(rs, return_alphas=True)
    alpha = rs.get_alphas(fo[H.DENSITY]) if c.opt.get("render") == "density" else fo[H.ALPHA]
    res = sb.render_from_alphas(alpha, fo[H.RGB], fo[H.NORMAL], rs, torch.ones(3, device="cuda"), training=True)
    loss = _loss(res["rgb"], target.cuda(), fo[H.GRADIENT], res["normal"], res["depth"], res["bg_transmittance"], fo[H.SDF],
                 fo["sampled_sdf"] if c.opt.get("curvature") else None, f.numerical_gradients_delta)
    loss.backward()
    out = {"loss": loss.detach().reshape(1), "rgb": res["rgb"].detach(), "sdf": fo[H.SDF].detach(), "gradients": fo[H.GRADIENT].detach(),
           "alphas": alpha.detach()}
    if fo["sampled_sdf"] is not None:
        out["sampled_sdf"] = fo["sampled_sdf"].detach()
    grads_p = {k: p.grad.detach().clone() for k, p in f.named_parameters() if p.grad is not None}
    return out, grads_p


class _Checks:
    """assert_within_noise over many quantities; every failing quantity is reported, not only the first"""

    def __init__(self, tag, floor):
        self.tag, self.floor, self.bad = tag, floor, []

    def __call__(self, what, cuda, r32, r64):
        assert tuple(cuda.shape) == tuple(r64.shape), f"{self.tag}/{what}: shape {tuple(cuda.shape)} != {tuple(r64.shape)}"
        scale = float(r64.detach().abs().max())
        try:
            assert_within_noise(cuda, r32, r64, f"{self.tag}/{what}", factor=FACTOR, floor=self.floor * scale)
        except AssertionError as e:
            self.bad.append(str(e))

    def done(self):
        assert not self.bad, "\n".join(self.bad)


def _check_params(chk, c: _Case, gp, g32, g64):
    """every parameter gradient within the noise bound; the same set of parameters has a nonzero gradient on both sides; the table rows of
    masked levels get exactly 0"""
    to_product = {"hash_table": c.table_name()}
    to_oracle = {v: k for k, v in to_product.items()}

    def nonzero(t):
        return t is not None and float(t.abs().max()) > 0.0

    nz_p = {to_oracle.get(k, k) for k, v in gp.items() if nonzero(v)}
    nz_o = {k for k, v in g64.items() if nonzero(v)}
    assert nz_p == nz_o, f"{c.name}/{c.gemm}: nonzero gradients only in the product {sorted(nz_p - nz_o)}, only in the oracle {sorted(nz_o - nz_p)}"
    expected = {f"{n}{l}.{w}" for n, k in (("glin", c.spec.num_layers + 1), ("clin", c.spec.num_layers_color + 1)) for l in range(k)
                for w in ("weight_g", "weight_v", "bias")}
    expected.add("laplace_density.beta" if c.opt.get("render") == "density" else "deviation_network.variance")
    if c.spec.use_grid_feature:
        expected.add("hash_table")
    if c.spec.use_appearance_embedding:
        expected.add("embedding_appearance.embedding.weight")
    assert expected <= nz_o, sorted(expected - nz_o)
    for k in sorted(nz_o):
        chk(f"d/d {k}", gp[to_product.get(k, k)].reshape(g64[k].shape), g32[k], g64[k])
    if "mask_level" in c.kw:
        assert c.spec.grid_layout == "torch"
        rows = c.kw["mask_level"] << c.spec.log2_hashmap_size
        gt = gp[c.table_name()]
        assert float(gt[rows:].abs().max()) == 0.0 and float(gt[:rows].abs().max()) > 0.0


_REF = {}


def _reference(c: _Case, rs, target):
    """fp32 and fp64 oracle steps on the product's own bins (cached per case: both GEMM settings sample the same bins)"""
    import sdfstudio_b200 as sb

    eu = sb.rays.bins_of(rs).detach().cpu()
    hit = _REF.get(c.name)
    if hit is not None and torch.equal(hit[0], eu):
        return hit[1]
    res = [_oracle_step(c, c.oracle(dt), eu, target) for dt in (torch.float32, torch.float64)]
    _REF[c.name] = (eu, res)
    return res


# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gemm", ["aten", "tc"])
@pytest.mark.parametrize("name", list(CASES))
def test_training_step_matches_fp64_oracle(name, gemm):
    """loss, rendered rgb, per-sample sdf / gradients / alpha (/ sampled_sdf) and every parameter gradient of one training step"""
    c = _Case(name, gemm)
    rs = c.samples()
    target = _target()
    out, gp = _product_step(c, rs, target)
    (e32, g32), (e64, g64) = _reference(c, rs, target)
    chk = _Checks(f"{name}/{gemm}", c.floor())
    assert ("sampled_sdf" in out) == c.spec.use_numerical_gradients == ("sampled_sdf" in e64)
    for k in e64:
        chk(k, out[k], e32[k], e64[k])
    _check_params(chk, c, gp, g32, g64)
    chk.done()


@pytest.mark.parametrize("gemm", ["aten", "tc"])
def test_angelo_step_grouped_equals_ungrouped(gemm, monkeypatch):
    """the seven taps of a sample through the grouped grid kernels (Encoding.point_groups(7)) against the same step with grouping off: the
    forward is bit for bit the same, every gradient the same up to the order of the atomic sums (table rows, appearance embedding rows)"""
    c = _Case("angelo_curvature", gemm)
    rs = c.samples()
    target = _target()
    out_g, gp_g = _product_step(c, rs, target)
    monkeypatch.setattr(c.field.encoding, "point_groups", lambda groups: contextlib.nullcontext())
    out_u, gp_u = _product_step(c, rs, target)
    for k in out_u:
        assert torch.equal(out_g[k], out_u[k]), k
    assert gp_g.keys() == gp_u.keys()
    for k, v in gp_u.items():
        scale = float(v.abs().max())
        assert float((gp_g[k] - v).abs().max()) <= 2e-6 * scale, (k, float((gp_g[k] - v).abs().max()) / max(scale, 1e-30))


@pytest.mark.parametrize("gemm", ["aten", "tc"])
@pytest.mark.parametrize("name", ["angelo_small", "bakedangelo"])
def test_numerical_gradient_in_training_mode(name, gemm):
    """field.gradient(x, return_sdf=True) of a numerical field in training mode (the six taps as one grouped batch, point_groups(6)) against
    oracle.gradient: the gradients and tap sdfs, then a loss on them back-propagated to the parameters"""
    c = _Case(name, gemm)
    g = torch.Generator().manual_seed(7)
    n = 600
    pts = (torch.rand(n, 3, generator=g) * 2 - 1) * (1.8 if c.spec.contraction else 0.9)
    cg, cs = torch.randn(n, 3, generator=g), torch.randn(6, n, generator=g)

    def loss_of(grads, psdf):
        return ((grads.norm(dim=-1) - 1) ** 2).mean() + 0.01 * (grads * cg.to(grads)).sum() + (psdf * cs.to(psdf)).mean()

    c.field.zero_grad(set_to_none=True)
    gr, ps = c.field.gradient(pts.cuda(), return_sdf=True)
    loss_of(gr, ps).backward()
    gp = {k: p.grad.detach().clone() for k, p in c.field.named_parameters() if p.grad is not None}
    ref = []
    for dt in (torch.float32, torch.float64):
        of = c.oracle(dt)
        gr_o, ps_o = of.gradient(pts.to(dt), return_sdf=True)
        loss_of(gr_o, ps_o).backward()
        ref.append((gr_o.detach(), ps_o.detach(), {k: v.grad for k, v in of.p.items() if v.is_floating_point() and v.grad is not None}))
    chk = _Checks(f"{name}/{gemm}/gradient()", c.floor())
    chk("gradients", gr, ref[0][0], ref[1][0])
    chk("points_sdf", ps, ref[0][1], ref[1][1])
    to_product = {"hash_table": c.table_name()}
    nz = {k for k, v in ref[1][2].items() if float(v.abs().max()) > 0}
    assert {"hash_table", "glin0.weight_v", "glin1.bias"} <= nz
    for k in sorted(nz):
        chk(f"d/d {k}", gp[to_product.get(k, k)].reshape(ref[1][2][k].shape), ref[0][2][k], ref[1][2][k])
    chk.done()


@pytest.mark.parametrize("layout,F", [("torch", 8), ("tcnn", 2)])
@pytest.mark.parametrize("delta", [1.0 / 4096.0, 0.03])
def test_grid_grouped_six_taps_equal_ungrouped(layout, F, delta):
    """Encoding.point_groups(6), the batch of SDFField.gradient() on a numerical field: the grouped kernels equal the ungrouped ones -- forward
    bit for bit, table gradient up to the order of the atomic sums -- with the taps inside one cell (delta = the finest cell) and across
    cells (delta = 0.03)"""
    import sdfstudio_b200 as sb

    L, log2T = 8, 12
    cfg = {"otype": "HashGrid", "n_levels": L, "n_features_per_level": F, "log2_hashmap_size": log2T, "base_resolution": 8, "per_level_scale": 1.5,
           "interpolation": "Linear"}
    enc = sb.Encoding(3, cfg, layout=layout).cuda()
    g = torch.Generator().manual_seed(12)
    with torch.no_grad():
        enc.table.copy_(torch.randn(enc.table.shape, generator=g) * 0.3)
    N = 1000
    x = torch.rand(N, 3, generator=g) * 0.9 + 0.05
    offs = torch.tensor([[delta, 0, 0], [-delta, 0, 0], [0, delta, 0], [0, -delta, 0], [0, 0, delta], [0, 0, -delta]])
    pts = (x[None] + offs[:, None, :]).reshape(-1, 3).cuda()
    r = torch.randn(6 * N, L * F, generator=g).cuda()

    def run(grouped):
        enc.zero_grad(set_to_none=True)
        with enc.point_groups(6) if grouped else contextlib.nullcontext():
            out = enc(pts)
        (out * r).sum().backward()
        return out.detach(), enc.table.grad.detach().clone()

    out_u, gt_u = run(False)
    launches0 = sb._lib.launch_count()
    out_g, gt_g = run(True)
    assert sb._lib.launch_count() - launches0 == 2          # one grouped forward, one grouped backward
    assert torch.equal(out_g, out_u)
    scale = float(gt_u.abs().max())
    assert float((gt_g - gt_u).abs().max()) <= 2e-6 * scale, float((gt_g - gt_u).abs().max()) / scale


def test_linear_padding_columns_are_not_part_of_the_function():
    """linear_ops.linear with softplus and N % 16 != 0: the padding columns of the result hold softplus(0) and are not part of the function,
    so a consumer that reads the whole padded result back-propagates only through the N real columns"""
    import torch.nn.functional as tF

    from sdfstudio_b200 import linear_ops as lo

    g = torch.Generator().manual_seed(8)
    P, K, N = 513, 39, 217                                # 217: the layer before the skip connection of an 8-layer geo network
    x = torch.randn(P, K, generator=g) * 0.3
    W, b = torch.randn(N, K, generator=g) / K**0.5, torch.randn(N, generator=g) * 0.02
    r = torch.randn(P, lo.pad16(N), generator=g)
    Wc, bc = W.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    y = lo.linear(lo.pad_cols(x).cuda(), Wc, bc, 1, "bf16x3")
    assert float(y[:, N:].min()) > 0.0                   # softplus(0) = log(2) / 100
    gW, gb = torch.autograd.grad((y * r.cuda()).sum(), [Wc, bc])
    W64, b64 = W.double().requires_grad_(True), b.double().requires_grad_(True)
    gW64, gb64 = torch.autograd.grad((tF.softplus(tF.linear(x.double(), W64, b64), beta=100) * r[:, :N].double()).sum(), [W64, b64])
    for a, e in ((gW, gW64), (gb, gb64)):
        assert float((a.double().cpu() - e).abs().max()) <= 2e-5 * float(e.abs().max())


# ---------------------------------------------------------------------------------------------------------------- the workload's size
P_WORKLOAD = 8192 * 48 * 7                             # rays x samples x (sample + six taps): rows of the angelo step's geo GEMMs


def _rowwise_error(a, ref_fn, chunks=8):
    """(max |a - ref|, max |ref_abs|) over row chunks without full-size float64 temporaries: ref_fn(lo, hi, absolute) -> float64 rows of
    the reference (absolute=True: the same product over |operands|, the scale a GEMM's rounding is relative to)"""
    n, step, err, scale = a.shape[0], (a.shape[0] + chunks - 1) // chunks, 0.0, 0.0
    for lo_ in range(0, n, step):
        hi = min(n, lo_ + step)
        err = max(err, float((a[lo_:hi].double() - ref_fn(lo_, hi, False)).abs().max()))
        scale = max(scale, float(ref_fn(lo_, hi, True).max()))
    return err, scale


@pytest.mark.parametrize("operands", ["nonnegative", "signed"])
@pytest.mark.parametrize("K,N", [(167, 256), (256, 257), (256, 256), (256, 3)])   # angelo geo 167 -> 256 -> 257, colour 256 -> 256 -> 3
def test_training_gemms_at_workload_rows(K, N, operands):
    """gemm_nt / gemm_nn / gemm_tn at bf16x3 over P = 2 752 512 rows against float64 matmuls on the GPU.  Non-negative operands (softplus /
    relu activations) are where the weight gradient's long fp32 reduction cannot cancel its rounding; gemm_tn must also be deterministic."""
    from sdfstudio_b200 import linear_ops as lo

    P = P_WORKLOAD
    g = torch.Generator(device="cuda").manual_seed(K * 1000 + N)
    if operands == "nonnegative":
        x = torch.rand(P, K, generator=g, device="cuda")
        W = torch.rand(N, K, generator=g, device="cuda") / K**0.5
        gy = torch.rand(P, N, generator=g, device="cuda")
    else:
        x = torch.randn(P, K, generator=g, device="cuda") * 0.5
        W = torch.randn(N, K, generator=g, device="cuda") / K**0.5
        gy = torch.randn(P, N, generator=g, device="cuda")
    xp, gyp = lo.pad_cols(x), lo.pad_cols(gy)
    del x, gy
    W64 = W.double()
    tol = 3e-5

    def ab(t, absolute):
        return t.abs() if absolute else t

    y = lo.gemm_nt(xp, W)
    err, scale = _rowwise_error(y[:, :N], lambda a, b, s: ab(xp[a:b, :K].double(), s) @ ab(W64, s).t())
    assert err <= tol * scale, ("nt", err / scale)
    del y
    dx = lo.gemm_nn(gyp, W)
    err, scale = _rowwise_error(dx[:, :K], lambda a, b, s: ab(gyp[a:b, :N].double(), s) @ ab(W64, s))
    assert err <= tol * scale, ("nn", err / scale)
    del dx
    dW = lo.gemm_tn(gyp, xp, N, K)
    ref = gyp[:, :N].double().t() @ xp[:, :K].double()
    scale = float((gyp[:, :N].abs().double().t() @ xp[:, :K].abs().double()).max())
    err = float((dW.double() - ref).abs().max()) / scale
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        err32 = float(((gyp[:, :N].t() @ xp[:, :K]).double() - ref).abs().max()) / scale
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    print(f"\n[wgrad P={P} K={K} N={N} {operands}] k_tc_wgrad bf16x3 {err:.2e}, fp32 cuBLAS (TF32 off) {err32:.2e} of max |dY|^T|X|")
    assert err <= max(tol, 4.0 * err32), ("tn", err, err32)
    assert torch.equal(dW, lo.gemm_tn(gyp, xp, N, K))


def test_grouped_grid_operator_at_workload_size():
    """the angelo workload's grid (L = 16, F = 8, T = 2^22: a 2.1 GB fp32 table, base 64, max 4096) over its 2 752 512 rows, seven taps of
    delta = 1/4096 per sample, level mask 8 applied as the training forward does (a multiply after the full encode): grouped forward bit for
    bit the ungrouped one, table gradients equal up to the order of the atomic sums, forward against the fp64 oracle on 4096 sampled rows"""
    import sdfstudio_b200 as sb

    L, F, log2T, base, max_res, mask = 16, 8, 22, 64, 4096, 8
    scale = hashgrid.growth_factor(L, base, max_res)
    cfg = {"otype": "HashGrid", "n_levels": L, "n_features_per_level": F, "log2_hashmap_size": log2T, "base_resolution": base, "per_level_scale": scale,
           "interpolation": "Linear"}
    enc = sb.Encoding(3, cfg, layout="torch").cuda()
    g = torch.Generator(device="cuda").manual_seed(21)
    with torch.no_grad():
        enc.table.copy_(torch.randn(enc.table.shape, generator=g, device="cuda") * 0.3)
    n = P_WORKLOAD // 7
    delta = 1.0 / 4096.0
    x = torch.rand(n, 3, generator=g, device="cuda") * 2 - 1
    offs = torch.tensor([[0, 0, 0], [delta, 0, 0], [-delta, 0, 0], [0, delta, 0], [0, -delta, 0], [0, 0, delta], [0, 0, -delta]], device="cuda")
    pts = ((x[None] + offs[:, None, :]).reshape(-1, 3) + 2.0) / 4.0          # SDFField's grid positions (x + 2) / 4
    del x
    level_mask = torch.ones(L * F, device="cuda")
    level_mask[mask * F:] = 0.0
    r = torch.randn(P_WORKLOAD, L * F, generator=g, device="cuda")

    def run(grouped):
        enc.zero_grad(set_to_none=True)
        with enc.point_groups(7) if grouped else contextlib.nullcontext():
            out = enc(pts)
        (out * level_mask * r).sum().backward()
        return out.detach(), enc.table.grad.detach().clone()

    out_u, gt_u = run(False)
    out_g, gt_g = run(True)
    assert torch.equal(out_g, out_u)
    del out_g
    gscale = float(gt_u.abs().max())
    assert float((gt_g - gt_u).abs().max()) <= 2e-6 * gscale, float((gt_g - gt_u).abs().max()) / gscale
    rows_masked = mask << log2T
    assert float(gt_g[rows_masked:].abs().max()) == 0.0 and float(gt_u[rows_masked:].abs().max()) == 0.0
    del gt_g, gt_u
    idx = torch.randperm(P_WORKLOAD, generator=torch.Generator().manual_seed(2))[:4096]
    xs = pts[idx.cuda()].cpu()
    table = enc.table.detach().cpu()
    scal = hashgrid.torch_layout_scalings(L, base, base * scale ** (L - 1))
    e32 = hashgrid.encode_torch_layout(xs, table, scal, 1 << log2T, False)
    e64 = hashgrid.encode_torch_layout(xs.double(), table, scal, 1 << log2T, False)      # fp32 table entries, float64 arithmetic
    assert_within_noise(out_u[idx.cuda()], e32, e64, "workload grid forward", factor=FACTOR, floor=1e-6 * float(e64.abs().max()))


def test_angelo_workload_step_tensor_core_gemms_match_fp32():
    """one full angelo-train-8192 step (tools/train_workload.py: 8192 rays x 48 uniform samples, the 2.1 GB table, level mask 8, delta =
    1/4096, rgb L1 + eikonal): the parameter gradients with the bf16x3 GEMMs against the same module and samples with ATen fp32 GEMMs
    (TF32 off).  Catches what only appears at size: chunking, index overflow, long reductions."""
    import sdfstudio_b200 as sb
    from sdfstudio_b200.synthetic import dtu_like_rays
    from tools.train_workload import R_TRAIN, S_TRAIN, Step, make_angelo_field

    dev = torch.device("cuda")
    field = make_angelo_field(dev, "bf16x3")
    o, d, cam, nears, fars = dtu_like_rays(R_TRAIN, 2000)
    with torch.no_grad():
        rs = sb.UniformSampler(num_samples=S_TRAIN, train_stratified=False).eval()(make_bundle(o, d, cam, nears, fars))
    target = torch.rand(R_TRAIN, 3, generator=torch.Generator().manual_seed(5)).to(dev)
    white = torch.ones(3, device=dev)
    step = Step(field)

    def run(gemm):
        field.config.train_gemm = gemm
        field.zero_grad(set_to_none=True)
        loss = step(rs, target, white)
        loss.backward()
        return float(loss), {k: p.grad.detach().clone() for k, p in field.named_parameters() if p.grad is not None}

    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        loss_tc, g_tc = run("tc")
        loss_32, g_32 = run("aten")
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    assert math.isfinite(loss_tc) and abs(loss_tc - loss_32) <= 1e-4 * abs(loss_32), (loss_tc, loss_32)
    assert g_tc.keys() == g_32.keys() and "encoding.hash_table" in g_32 and "embedding_appearance.embedding.weight" in g_32
    # the small angelo cases hold bf16x3 to FLOOR_TC_NUMERICAL at delta = 0.002; this delta is 8x smaller, and the bf16x3 GEMM noise in the
    # gradients grows with 1 / delta.  Compared in the L2 norm of each parameter tensor: the max-norm follows the few table rows with the
    # largest eikonal contributions, while a chunking or overflow bug moves the whole tensor.
    bound = FLOOR_TC_NUMERICAL * 0.002 / field.numerical_gradients_delta
    errs = {}
    for k, v in g_32.items():
        assert bool(torch.isfinite(g_tc[k]).all()), k
        errs[k] = (float((g_tc[k] - v).norm() / v.norm().clamp_min(1e-30)), float((g_tc[k] - v).abs().max() / v.abs().max().clamp_min(1e-30)))
    print("\n[angelo-train-8192 step, bf16x3 vs fp32 GEMMs] relative L2 / max-norm difference per parameter:",
          {k: f"{a:.1e}/{b:.1e}" for k, (a, b) in errs.items()})
    bad = {k: f"{a:.2e}" for k, (a, _) in errs.items() if not a <= bound}
    assert not bad, (bound, bad)
    assert float(g_tc["encoding.hash_table"][8 << 22:].abs().max()) == 0.0
