"""-m gpu: the hash-grid operator (csrc/grid_encode.cu over csrc/grid.cuh) against fp64 autograd of oracle/hashgrid.py, over its
whole configuration space: layout {torch, tcnn} x F {1, 2, 4, 8} x table {fp32, fp16} x {linear, smoothstep}.

The oracle evaluates each level at the kernels' own fp32 position (x*scale, or fma(x, scale, 0.5) for tcnn; `fp32_positions`), so it
blends the same cell with the same offset and only the kernels' arithmetic is measured.  An fp16 table is held by the oracle as
table.half().double(), the values the kernels gather.

Bounds are element-wise, a multiple of u = 2^-24 times the magnitude of the terms the element is made of, computed in fp64 from the
oracle's corner rows and per-axis weights with |.| on every factor.  Each per-axis weight factor of a corner (w or 1 - w) carries an
ABSOLUTE rounding error (1 - w is rounded from a rounded w), so the magnitude of a corner weight is |W_k| + the sum of its 2-factor
sub-products (`weight_mag`), and likewise for its derivatives.  The multiples:
  forward    FWD_K = 14: <= 4u per weight factor (3 roundings of smoothstep, 1 of 1 - w), 2u for the 3-factor product, <= 8u for the
             blend (torch: 3 lerp levels of one product and one sum; tcnn: 8 fma into the running sum)
  Jacobian   JAC_K = 20: the forward's 14u, one difference of two corner rows, dw = 6t(1 - t) (3u) and the two final products
  dx         JAC_K + F + L: one fma per feature, one fp32 atomic per level
  table grad (7 + m)u: the weight (6u) times dout (1u), m fp32 atomics into the row (m counted from the oracle's indices)
  g_dout     JAC_K + 4: a 3-term dot with g_dx and one fma per corner
  g_table    (JAC_K + m)u
  g_x        (HESS_K + L)u, HESS_K = 24 + F: d2w = (6 - 12t) s^2 (bounded with 6 + 12t), 4-factor products, the F-term dot with dout,
             the 3-term dot with g_dx and 8 fma over the corners
"""
import numpy as np
import pytest
import torch

from oracle import hashgrid

from helpers import corner_factors, geometry, kernel_positions, weight_mag

pytestmark = pytest.mark.gpu

U = 2.0**-24
FWD_K, JAC_K = 14, 20
DEV = "cuda"

# level sets.  "collide": log2T = 6, so corners of one cell share rows; tcnn level 0 is dense with res^3 = 27 rows (not a multiple of 8,
# padded to 32), level 1 is the first hashed one.  "wide": log2T = 14, tcnn levels 0-2 dense (27, 729, 13824 rows), level 3 the first
# hashed.  Both end at the angelo preset's finest scale (max_res 4096).  The torch layout hashes every level.
GRIDS = {"collide": dict(L=6, log2T=6, base=3, max_res=4096), "wide": dict(L=8, log2T=14, base=3, max_res=4096)}
CONFIGS = [(lay, F, dt, sm) for lay in ("torch", "tcnn") for F in (1, 2, 4, 8) for dt in ("fp32", "fp16") for sm in (False, True)]


def cid(c):
    return f"{c[0]}-F{c[1]}-{c[2]}-{'smooth' if c[3] else 'linear'}"


def make_enc(layout, F, table_dtype, smooth, L, log2T, base, max_res, seed=0):
    import sdfstudio_b200 as sb

    g = hashgrid.growth_factor(L, base, max_res)
    cfg = {"otype": "HashGrid", "n_levels": L, "n_features_per_level": F, "log2_hashmap_size": log2T, "base_resolution": base,
           "per_level_scale": g, "interpolation": "Smoothstep" if smooth else "Linear"}
    enc = sb.Encoding(3, cfg, layout=layout, table_dtype=table_dtype).to(DEV)
    gen = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        enc.table.copy_(((torch.rand(enc.table.shape, generator=gen) * 2 - 1)).to(DEV))
    return enc


def scales(enc):
    return torch.tensor([enc._desc.scale[l] for l in range(enc.n_levels)], dtype=torch.float32)


def oracle_table(enc):
    """[rows, F] fp64: what the kernels gather."""
    return enc.compute_table().double().view(-1, enc.n_features_per_level)


def oracle(enc, x64, t64):
    """fp64 oracle output [N, L*F] and the corner rows [N, L, 8] (corner k: bit 0 = x, 1 = y, 2 = z carries the per-axis weight w)."""
    F, smooth = enc.n_features_per_level, enc.interpolation == "Smoothstep"
    if enc.layout == "torch":
        scal = hashgrid.torch_layout_scalings(enc.n_levels, enc.base_resolution, enc.base_resolution * enc.per_level_scale ** (enc.n_levels - 1))
        assert torch.equal(scal.float(), scales(enc))
        out, idx = hashgrid.encode_torch_layout(x64, t64, scal, 1 << enc.log2_hashmap_size, smooth, return_indices=True, fp32_positions=True)
        # the reference's corners f0..f7 are (c,c,c)(c,f,c)(f,f,c)(f,c,c)(c,c,f)(c,f,f)(f,f,f)(f,c,f), c = ceil = a set bit
        order = [7, 5, 4, 6, 3, 1, 0, 2]
        rows = torch.empty_like(idx)
        for j, k in enumerate(order):
            rows[..., k] = idx[..., j]
        return out, rows
    meta = hashgrid.tcnn_grid_meta(enc.n_levels, F, enc.log2_hashmap_size, enc.base_resolution, enc.per_level_scale)
    return hashgrid.encode_tcnn_layout(x64, t64, meta, F, smooth, return_indices=True, fp32_positions=True)


def deriv_mag(a, dws):
    """[N, L, 8, 3]: magnitude of dW_k / dx_d (|dw_d s| times the other two factors, each with its absolute error)"""
    out = []
    for d in range(3):
        o1, o2 = [a[..., e] for e in range(3) if e != d]
        out.append(dws[:, :, None, d] * (o1 * o2 + o1 + o2))
    return torch.stack(out, -1)


def hess_mag(a, dws, d2m):
    """[N, L, 8, 3, 3]: magnitude of d2 W_k / dx_c dx_c'"""
    H = torch.zeros(*a.shape, 3, device=a.device, dtype=a.dtype)
    for c in range(3):
        for c2 in range(3):
            others = [e for e in range(3) if e not in (c, c2)]
            if c == c2:
                o1, o2 = a[..., others[0]], a[..., others[1]]
                H[..., c, c] = d2m[:, :, None, c] * (o1 * o2 + o1 + o2)
            else:
                H[..., c, c2] = dws[:, :, None, c] * dws[:, :, None, c2] * (a[..., others[0]] + 1)
    return H


class Ref:
    """The fp64 oracle of one (encoder, points) pair: values through autograd, magnitudes from the corner rows and weights."""

    def __init__(self, enc, x32):
        self.enc, self.x32 = enc, x32
        self.L, self.F = enc.n_levels, enc.n_features_per_level
        self.t64 = oracle_table(enc)
        self.x64 = x32.double().requires_grad_(True)
        self.tab = self.t64.clone().requires_grad_(True)
        self.out, self.rows = oracle(enc, self.x64, self.tab)
        w, dws, d2m = geometry(x32, scales(enc), enc.layout, enc.interpolation == "Smoothstep")
        self.a = corner_factors(w)
        self.dws, self.d2m = dws, d2m
        self.vabs = self.t64.abs()[self.rows]                        # [N, L, 8, F]
        self.fwd_mag = (weight_mag(self.a)[..., None] * self.vabs).sum(2)                    # [N, L, F]
        self.jm = deriv_mag(self.a, dws)                                                     # [N, L, 8, 3]
        self.jac_mag = torch.einsum("nlkd,nlkf->nlfd", self.jm, self.vabs)                   # [N, L, F, 3]

    def jacobian(self):
        """[N, L*F, 3] by autograd, one output column at a time"""
        cols = []
        for j in range(self.L * self.F):
            cols.append(torch.autograd.grad(self.out[:, j].sum(), self.x64, retain_graph=True)[0])
        return torch.stack(cols, 1)

    def row_terms(self, term_mag):
        """sum over the (point, level, corner) terms scattered into each row of term_mag [N, L, 8, F], and the number of terms per row"""
        nrows = self.t64.shape[0]
        flat = self.rows.reshape(-1)
        S = torch.zeros(nrows, self.F, dtype=torch.float64, device=DEV).index_add_(0, flat, term_mag.reshape(-1, self.F))
        m = torch.bincount(flat, minlength=nrows).double()
        return S, m


def check(what, got, ref, bound):
    got, ref, bound = got.double(), ref.double(), bound.double()
    err = (got - ref).abs()
    bad = err > bound
    if bool(bad.any()):
        i = int(torch.nonzero(bad.reshape(-1))[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements out of bound; first at flat index {i}: got {float(got.reshape(-1)[i])!r} "
                             f"ref {float(ref.reshape(-1)[i])!r} err {float(err.reshape(-1)[i]):.3e} bound {float(bound.reshape(-1)[i]):.3e}")


def lattice_points(enc, gen):
    """For every level, points whose kernel position is exactly an integer on one, two and three axes (a cell face, an edge and a
    corner), verified with the kernel's own fp32 rounding."""
    s = scales(enc).numpy()
    pts = []
    for l in range(enc.n_levels):
        for n_int in (1, 2, 3):
            p = np.float32(torch.rand(3, generator=gen).numpy())
            for d in range(n_int):
                # not every lattice coordinate i has an fp32 x with a rounded position of exactly i: try up to 64 of them
                for i in torch.randint(1, max(2, int(s[l])), (64,), generator=gen).tolist():
                    guess = np.float32((i - (0.0 if enc.layout == "torch" else 0.5)) / float(s[l]))
                    cands = guess + np.arange(-4, 5, dtype=np.float32) * np.spacing(guess)
                    if enc.layout == "torch":
                        hits = cands[cands * np.float32(s[l]) == np.float32(i)]
                    else:
                        hits = cands[(cands.astype(np.float64) * np.float64(s[l]) + 0.5).astype(np.float32) == np.float32(i)]
                    if len(hits):
                        p[d] = hits[0]
                        break
                else:
                    raise AssertionError(f"no fp32 lattice point for level {l}")
            pts.append(p)
    x = torch.tensor(np.stack(pts))
    q = kernel_positions(x, scales(enc), enc.layout)
    lv = torch.arange(enc.n_levels).repeat_interleave(3)
    qi = q[torch.arange(len(x)), lv]
    n_on = (qi == torch.floor(qi)).sum(1)
    assert bool((n_on >= torch.tensor([1, 2, 3] * enc.n_levels)).all()), "lattice points are not on the lattice"
    return x


def points(enc, n=1500, seed=1):
    gen = torch.Generator().manual_seed(seed)
    u = torch.rand(n, 3, generator=gen)
    out = (torch.rand(n // 3, 3, generator=gen) * 2 - 0.5)                      # [-0.5, 1.5]: AABB-normalised / uncontracted fields
    one_m = float(np.nextafter(np.float32(1), np.float32(0)))
    edges = torch.tensor([[0, 0, 0], [1, 1, 1], [one_m] * 3, [0, 1, one_m], [one_m, 0, 1], [1, one_m, 0]], dtype=torch.float32)
    return torch.cat([u, out, edges, lattice_points(enc, gen)]).to(DEV).contiguous()


def lib():
    import sdfstudio_b200 as sb

    return sb._lib.load()


def call(fn, *args):
    import sdfstudio_b200 as sb

    sb._lib.check(getattr(lib(), fn)(*args), fn)


def ptr(t):
    return None if t is None else t.data_ptr()


def level_rows(enc):
    """[rows] level index of each table row"""
    d = enc._desc
    sizes = [d.size[l] for l in range(enc.n_levels)]
    return torch.repeat_interleave(torch.arange(enc.n_levels, device=DEV), torch.tensor(sizes, device=DEV))


# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid", list(GRIDS))
@pytest.mark.parametrize("cfg", CONFIGS, ids=cid)
def test_forward_jacobian_and_backwards_match_fp64(cfg, grid):
    layout, F, dt, smooth = cfg
    enc = make_enc(layout, F, dt, smooth, **GRIDS[grid])
    L = enc.n_levels
    x = points(enc)
    n = x.shape[0]
    ref = Ref(enc, x)
    table = enc.compute_table()
    assert table.dtype == (torch.float16 if dt == "fp16" else torch.float32)
    if grid == "collide":   # corners of one cell that share a row: the table gradient sums them
        r = ref.rows.reshape(-1, 8)
        dup = (r[:, :, None] == r[:, None, :]).sum((1, 2)) > 8
        if layout == "tcnn":
            dup = dup.view(n, L)[:, 1:]   # hashed levels (level 0 is dense)
        assert int(dup.sum()) > 10, "expected colliding corners"

    # forward + dout_dx
    out = torch.empty(n, L * F, device=DEV)
    J = torch.empty(n, L * F, 3, device=DEV)
    call("sdfb200_grid_encode", enc._desc_ref(), table.data_ptr(), x.data_ptr(), n, out.data_ptr(), L * F, J.data_ptr(), None)
    torch.cuda.synchronize()
    check("out", out.view(n, L, F), ref.out.detach().view(n, L, F), FWD_K * U * ref.fwd_mag)
    check("dout_dx", J.view(n, L, F, 3), ref.jacobian().view(n, L, F, 3), JAC_K * U * ref.jac_mag)
    out_nj = torch.empty_like(out)
    call("sdfb200_grid_encode", enc._desc_ref(), table.data_ptr(), x.data_ptr(), n, out_nj.data_ptr(), L * F, None, None)
    assert torch.equal(out_nj, out)
    if layout == "torch":
        # the torch layout restates the reference's expression tree rounding by rounding: equal to the fp32 oracle bit for bit
        o32, _ = oracle(enc, x.clone(), table.float().view(-1, F))
        assert torch.equal(out, o32), f"torch layout differs from the fp32 reference at {int((out != o32).sum())} elements"

    # backward: dtable only, dx only, both
    gen = torch.Generator().manual_seed(11)
    go = torch.randn(n, L * F, generator=gen).to(DEV)
    dtab_ref, dx_ref = torch.autograd.grad((ref.out * go.double()).sum(), [ref.tab, ref.x64], retain_graph=True)
    S, m = ref.row_terms(weight_mag(ref.a)[..., None] * go.double().abs().view(n, L, 1, F))
    dtab_bound = (7 + m)[:, None] * U * S
    dx_bound = (JAC_K + F + L) * U * (go.double().abs().view(n, L, F, 1) * ref.jac_mag).sum((1, 2))
    rows = ref.t64.shape[0]
    for want_t, want_x in ((True, False), (False, True), (True, True)):
        dtab = torch.zeros(rows, F, device=DEV) if want_t else None
        dx = torch.zeros(n, 3, device=DEV) if want_x else None
        call("sdfb200_grid_encode_backward", enc._desc_ref(), table.data_ptr(), x.data_ptr(), go.data_ptr(), n, ptr(dtab), ptr(dx), None)
        torch.cuda.synchronize()
        if want_t:
            check("dtable", dtab, dtab_ref, dtab_bound)
        if want_x:
            check("dx", dx, dx_ref, dx_bound)

    # double backward: g_dout, g_table, g_x alone and together
    gdx = torch.randn(n, 3, generator=gen).to(DEV)
    go64 = go.double().requires_grad_(True)
    dx_o = torch.autograd.grad((ref.out * go64).sum(), ref.x64, create_graph=True)[0]
    g_do_ref, g_t_ref, g_x_ref = torch.autograd.grad((dx_o * gdx.double()).sum(), [go64, ref.tab, ref.x64], allow_unused=True)
    g_t_ref = torch.zeros_like(ref.t64) if g_t_ref is None else g_t_ref
    g_x_ref = torch.zeros_like(ref.x64) if g_x_ref is None else g_x_ref
    gdx_abs = gdx.double().abs()
    gdo_bound = (JAC_K + 4) * U * (ref.jac_mag * gdx_abs[:, None, None, :]).sum(-1).reshape(n, L * F)
    gW = (ref.jm * gdx_abs[:, None, None, :]).sum(-1)                                              # [N, L, 8]
    S2, m2 = ref.row_terms(gW[..., None] * go.double().abs().view(n, L, 1, F))
    gt_bound = (JAC_K + m2)[:, None] * U * S2
    H = hess_mag(ref.a, ref.dws, ref.d2m)                                                         # [N, L, 8, 3, 3]
    dot = (go.double().abs().view(n, L, 1, F) * ref.vabs).sum(-1)                                 # [N, L, 8]
    gx_bound = (24 + F + L) * U * torch.einsum("nlk,nlkcd,nc->nd", dot, H, gdx_abs)
    for sel in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1)):
        g_do = torch.full((n, L * F), float("nan"), device=DEV) if sel[0] else None
        g_t = torch.zeros(rows, F, device=DEV) if sel[1] else None
        g_x = torch.zeros(n, 3, device=DEV) if sel[2] else None
        call("sdfb200_grid_encode_backward_backward", enc._desc_ref(), table.data_ptr(), x.data_ptr(), go.data_ptr(), gdx.data_ptr(), n,
             ptr(g_do), ptr(g_t), ptr(g_x), None)
        torch.cuda.synchronize()
        if sel[0]:
            check("g_dout", g_do, g_do_ref, gdo_bound)
        if sel[1]:
            check("g_table", g_t, g_t_ref, gt_bound)
        if sel[2]:
            check("g_x", g_x, g_x_ref, gx_bound)


# ----------------------------------------------------------------------------------------------------------------
def tap_points(pattern, group, S, gen):
    """[group * S, 3], tap gi of sample s at row gi * S + s"""
    A = torch.rand(S, 3, generator=gen)
    if pattern == "same":
        taps = [A] * group
    elif pattern == "differ":
        taps = [torch.rand(S, 3, generator=gen) for _ in range(group)]
    else:   # A A B A A ...: the taps leave the cell and come back, the backward flushes twice
        B = torch.rand(S, 3, generator=gen)
        taps = [B if i % 4 == 2 else A for i in range(group)]
    return torch.cat(taps).to(DEV).contiguous()


@pytest.mark.parametrize("cfg", CONFIGS, ids=cid)
def test_grouped_kernels_match_ungrouped_and_fp64(cfg):
    layout, F, dt, smooth = cfg
    enc = make_enc(layout, F, dt, smooth, **GRIDS["collide"])
    L, table = enc.n_levels, enc.compute_table()
    rows = table.numel() // F
    gen = torch.Generator().manual_seed(5)
    S = 97
    for group in (1, 2, 6, 7):
        for pattern in ("same", "differ", "ABA"):
            x = tap_points(pattern, group, S, gen)
            n = x.shape[0]
            o_g, o_u = torch.empty(n, L * F, device=DEV), torch.empty(n, L * F, device=DEV)
            call("sdfb200_grid_encode_grouped", enc._desc_ref(), table.data_ptr(), x.data_ptr(), n, group, o_g.data_ptr(), L * F, None)
            call("sdfb200_grid_encode", enc._desc_ref(), table.data_ptr(), x.data_ptr(), n, o_u.data_ptr(), L * F, None, None)
            torch.cuda.synchronize()
            assert torch.equal(o_g, o_u), (group, pattern)
            go = torch.randn(n, L * F, generator=gen).to(DEV)
            d_g = torch.zeros(rows, F, device=DEV)
            call("sdfb200_grid_encode_backward_grouped", enc._desc_ref(), x.data_ptr(), go.data_ptr(), n, group, d_g.data_ptr(), None)
            torch.cuda.synchronize()
            ref = Ref(enc, x)
            d_ref = torch.autograd.grad((ref.out * go.double()).sum(), ref.tab)[0]
            S_, m = ref.row_terms(weight_mag(ref.a)[..., None] * go.double().abs().view(n, L, 1, F))
            check(f"grouped dtable G={group} {pattern}", d_g, d_ref, (7 + m)[:, None] * U * S_)
    # a batch that is not a multiple of the group runs the ungrouped kernels
    x = tap_points("ABA", 7, S, gen)[: 7 * S - 3].contiguous().requires_grad_(False)
    plain = enc(x)
    with enc.point_groups(7):
        grouped = enc(x)
        go = torch.randn_like(grouped)
        (grouped * go).sum().backward()
    assert torch.equal(grouped, plain)
    ref = Ref(enc, x)
    d_ref = torch.autograd.grad((ref.out * go.double()).sum(), ref.tab)[0]
    S_, m = ref.row_terms(weight_mag(ref.a)[..., None] * go.double().abs().view(-1, L, 1, F))
    check("fallback dtable", enc.table.grad.view(-1, F), d_ref, (7 + m)[:, None] * U * S_)


# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["torch", "tcnn"])
@pytest.mark.parametrize("F,dt", [(2, "fp32"), (8, "fp16")])
def test_encoding_autograd_inputs_only_and_eikonal(layout, F, dt):
    enc = make_enc(layout, F, dt, True, **GRIDS["wide"])
    L = enc.n_levels
    x = points(enc, n=700, seed=3)
    n = x.shape[0]
    gen = torch.Generator().manual_seed(2)
    go = torch.randn(n, L * F, generator=gen).to(DEV)
    gdx = torch.randn(n, 3, generator=gen).to(DEV)
    ref = Ref(enc, x)
    dx_bound = (JAC_K + F + L) * U * (go.double().abs().view(n, L, F, 1) * ref.jac_mag).sum((1, 2))
    # the autograd.grad(sdf, x) of SDFField: d/dx only
    xg = x.clone().requires_grad_(True)
    with enc.inputs_only_backward():
        dx = torch.autograd.grad((enc(xg) * go).sum(), xg)[0]
    dx_ref = torch.autograd.grad((ref.out * go.double()).sum(), ref.x64, create_graph=True)[0]
    check("inputs-only dx", dx, dx_ref, dx_bound)
    # eikonal pattern: create_graph, then a loss on dx back to the table and x
    xg = x.clone().requires_grad_(True)
    dx = torch.autograd.grad((enc(xg) * go).sum(), xg, create_graph=True)[0]
    check("create_graph dx", dx, dx_ref, dx_bound)
    (dx * gdx).sum().backward()
    g_t_ref, g_x_ref = torch.autograd.grad((dx_ref * gdx.double()).sum(), [ref.tab, ref.x64], allow_unused=True)
    gdx_abs = gdx.double().abs()
    gW = (ref.jm * gdx_abs[:, None, None, :]).sum(-1)
    S2, m2 = ref.row_terms(gW[..., None] * go.double().abs().view(n, L, 1, F))
    check("eikonal table grad", enc.table.grad.view(-1, F), g_t_ref, (JAC_K + m2)[:, None] * U * S2)
    H = hess_mag(ref.a, ref.dws, ref.d2m)
    dot = (go.double().abs().view(n, L, 1, F) * ref.vabs).sum(-1)
    check("eikonal x grad", xg.grad, g_x_ref, (24 + F + L) * U * torch.einsum("nlk,nlkcd,nc->nd", dot, H, gdx_abs))


# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", [c for c in CONFIGS if c[3]], ids=cid)
def test_masked_levels_are_exactly_zero(cfg):
    layout, F, dt, smooth = cfg
    enc = make_enc(layout, F, dt, smooth, **GRIDS["wide"])
    L, table = enc.n_levels, enc.compute_table()
    rows = table.numel() // F
    x = points(enc, n=500, seed=4)
    n = x.shape[0]
    gen = torch.Generator().manual_seed(6)
    go = torch.randn(n, L * F, generator=gen).to(DEV)
    gdx = torch.randn(n, 3, generator=gen).to(DEV)
    lvl = level_rows(enc)

    def run(active):
        enc.set_active_levels(active)
        d = enc._desc_ref()
        out, J = torch.empty(n, L * F, device=DEV), torch.empty(n, L * F, 3, device=DEV)
        call("sdfb200_grid_encode", d, table.data_ptr(), x.data_ptr(), n, out.data_ptr(), L * F, J.data_ptr(), None)
        dtab, dx = torch.zeros(rows, F, device=DEV), torch.zeros(n, 3, device=DEV)
        call("sdfb200_grid_encode_backward", d, table.data_ptr(), x.data_ptr(), go.data_ptr(), n, dtab.data_ptr(), dx.data_ptr(), None)
        dgrp = torch.zeros(rows, F, device=DEV)
        call("sdfb200_grid_encode_backward_grouped", d, x.data_ptr(), go.data_ptr(), n, 1, dgrp.data_ptr(), None)
        g_do, g_t = torch.full((n, L * F), float("nan"), device=DEV), torch.zeros(rows, F, device=DEV)
        call("sdfb200_grid_encode_backward_backward", d, table.data_ptr(), x.data_ptr(), go.data_ptr(), gdx.data_ptr(), n, g_do.data_ptr(),
             g_t.data_ptr(), None, None)
        torch.cuda.synchronize()
        return out, J, dtab, dgrp, g_do, g_t

    full = run(L)
    for active in (0, 1, L - 1, L):
        out, J, dtab, dgrp, g_do, g_t = run(active)
        k = active * F
        assert torch.equal(out[:, k:], torch.zeros_like(out[:, k:])) and torch.equal(J[:, k:], torch.zeros_like(J[:, k:]))
        assert torch.equal(g_do[:, k:], torch.zeros_like(g_do[:, k:]))
        assert torch.equal(out[:, :k], full[0][:, :k]) and torch.equal(J[:, :k], full[1][:, :k]) and torch.equal(g_do[:, :k], full[4][:, :k])
        masked = lvl >= active
        for what, d in (("dtable", dtab), ("grouped dtable", dgrp), ("g_table", g_t)):
            assert int(torch.count_nonzero(d[masked])) == 0, what
    enc.set_active_levels(L)


# ----------------------------------------------------------------------------------------------------------------
def test_past_2_31_elements():
    """n*L*F*3 (the Jacobian) and n*L*F (dout) past 2^31: the samples at the end of the batch equal a small call on the same points."""
    enc = make_enc("tcnn", 8, "fp32", True, L=16, log2T=16, base=16, max_res=2048)
    L, F, table = enc.n_levels, 8, enc.compute_table()
    gen = torch.Generator(device=DEV).manual_seed(1)
    n = (1 << 31) // (L * F * 3) + 4099
    x = torch.rand(n, 3, device=DEV, generator=gen)
    sample = torch.cat([torch.arange(0, 1000, device=DEV), torch.arange(n - 3000, n, device=DEV)])
    out = torch.empty(n, L * F, device=DEV)
    J = torch.empty(n, L * F, 3, device=DEV)
    call("sdfb200_grid_encode", enc._desc_ref(), table.data_ptr(), x.data_ptr(), n, out.data_ptr(), L * F, J.data_ptr(), None)
    xs = x[sample].contiguous()
    o_s, J_s = torch.empty(len(sample), L * F, device=DEV), torch.empty(len(sample), L * F, 3, device=DEV)
    call("sdfb200_grid_encode", enc._desc_ref(), table.data_ptr(), xs.data_ptr(), len(sample), o_s.data_ptr(), L * F, J_s.data_ptr(), None)
    torch.cuda.synchronize()
    assert torch.equal(out[sample], o_s) and torch.equal(J[sample], J_s)
    del out, J, x
    torch.cuda.empty_cache()
    n = (1 << 31) // (L * F) + 4099
    x = torch.rand(n, 3, device=DEV, generator=gen)
    go = torch.randn(n, L * F, device=DEV, generator=gen)
    dx = torch.zeros(n, 3, device=DEV)
    call("sdfb200_grid_encode_backward", enc._desc_ref(), table.data_ptr(), x.data_ptr(), go.data_ptr(), n, None, dx.data_ptr(), None)
    sample = torch.cat([torch.arange(0, 1000, device=DEV), torch.arange(n - 3000, n, device=DEV)])
    xs, gs = x[sample].contiguous(), go[sample].contiguous()
    del go
    torch.cuda.empty_cache()
    ref = Ref(enc, xs)
    dx_ref = torch.autograd.grad((ref.out * gs.double()).sum(), ref.x64)[0]
    check("dx past 2^31", dx[sample], dx_ref, (JAC_K + F + L) * U * (gs.double().abs().view(-1, L, F, 1) * ref.jac_mag).sum((1, 2)))


@pytest.mark.parametrize("dt", ["fp32", "fp16"])
def test_angelo_size(dt):
    """The angelo preset's grid (L = 16, F = 8, log2T = 22, base 64, max 4096) on 2^20 points: forward, backward and double backward
    against the fp64 oracle run on the GPU in chunks, with the element-wise bounds."""
    enc = make_enc("tcnn", 8, dt, False, L=16, log2T=22, base=64, max_res=4096)
    L, F, table = 16, 8, enc.compute_table()
    rows = table.numel() // F
    gen = torch.Generator(device=DEV).manual_seed(3)
    n = 1 << 20
    x = torch.rand(n, 3, device=DEV, generator=gen)
    go = torch.randn(n, L * F, device=DEV, generator=gen)
    gdx = torch.randn(n, 3, device=DEV, generator=gen)
    out = torch.empty(n, L * F, device=DEV)
    dtab, dx = torch.zeros(rows, F, device=DEV), torch.zeros(n, 3, device=DEV)
    g_do, g_t, g_x = torch.empty(n, L * F, device=DEV), torch.zeros(rows, F, device=DEV), torch.zeros(n, 3, device=DEV)
    d = enc._desc_ref()
    call("sdfb200_grid_encode", d, table.data_ptr(), x.data_ptr(), n, out.data_ptr(), L * F, None, None)
    call("sdfb200_grid_encode_backward", d, table.data_ptr(), x.data_ptr(), go.data_ptr(), n, dtab.data_ptr(), dx.data_ptr(), None)
    call("sdfb200_grid_encode_backward_backward", d, table.data_ptr(), x.data_ptr(), go.data_ptr(), gdx.data_ptr(), n, g_do.data_ptr(), g_t.data_ptr(),
         g_x.data_ptr(), None)
    torch.cuda.synchronize()
    dtab_ref, g_t_ref = torch.zeros(rows, F, dtype=torch.float64, device=DEV), torch.zeros(rows, F, dtype=torch.float64, device=DEV)
    S1, S2 = torch.zeros_like(dtab_ref), torch.zeros_like(dtab_ref)
    m = torch.zeros(rows, dtype=torch.float64, device=DEV)
    chunk = 1 << 16
    for c0 in range(0, n, chunk):
        sl = slice(c0, c0 + chunk)
        ref = Ref(enc, x[sl])
        k = ref.x64.shape[0]
        g = go[sl].double()
        check("angelo out", out[sl].view(k, L, F), ref.out.detach().view(k, L, F), FWD_K * U * ref.fwd_mag)
        g64 = g.clone().requires_grad_(True)
        dx_o = torch.autograd.grad((ref.out * g64).sum(), ref.x64, create_graph=True)[0]
        dt_c = torch.autograd.grad((ref.out * g).sum(), ref.tab, retain_graph=True)[0]
        check("angelo dx", dx[sl], dx_o.detach(), (JAC_K + F + L) * U * (g.abs().view(k, L, F, 1) * ref.jac_mag).sum((1, 2)))
        gd = gdx[sl].double()
        gdo_ref, gt_c, gx_ref = torch.autograd.grad((dx_o * gd).sum(), [g64, ref.tab, ref.x64], allow_unused=True)
        check("angelo g_dout", g_do[sl], gdo_ref, (JAC_K + 4) * U * (ref.jac_mag * gd.abs()[:, None, None, :]).sum(-1).reshape(k, L * F))
        if gx_ref is not None:   # linear interpolation: d2W has only the off-diagonal terms
            H = hess_mag(ref.a, ref.dws, ref.d2m)
            dot = (g.abs().view(k, L, 1, F) * ref.vabs).sum(-1)
            check("angelo g_x", g_x[sl], gx_ref, (24 + F + L) * U * torch.einsum("nlk,nlkcd,nc->nd", dot, H, gd.abs()))
        dtab_ref += dt_c
        g_t_ref += gt_c
        s1, mc = ref.row_terms(weight_mag(ref.a)[..., None] * g.abs().view(k, L, 1, F))
        s2, _ = ref.row_terms((ref.jm * gd.abs()[:, None, None, :]).sum(-1)[..., None] * g.abs().view(k, L, 1, F))
        S1 += s1
        S2 += s2
        m += mc
        del ref, dx_o
    check("angelo dtable", dtab, dtab_ref, (7 + m)[:, None] * U * S1)
    check("angelo g_table", g_t, g_t_ref, (JAC_K + m)[:, None] * U * S2)


# ----------------------------------------------------------------------------------------------------------------
# the fp16 copy of the table follows the fp32 parameter
# ----------------------------------------------------------------------------------------------------------------
def _fp16_pair():
    enc = make_enc("tcnn", 2, "fp16", False, L=4, log2T=10, base=4, max_res=64)
    x = torch.rand(257, 3, generator=torch.Generator().manual_seed(8)).to(DEV)
    return enc, x


def _fresh(enc):
    fresh = make_enc("tcnn", 2, "fp16", False, L=4, log2T=10, base=4, max_res=64, seed=99)
    with torch.no_grad():
        fresh.table.copy_(enc.table)
    return fresh


@pytest.mark.parametrize("how", ["adam-foreach", "adam-fused", "load_state_dict", "copy_"])
def test_fp16_copy_follows_the_table(how):
    enc, x = _fp16_pair()
    before = enc(x).detach()
    if how.startswith("adam"):
        opt = torch.optim.Adam(enc.parameters(), lr=1e-2, foreach=how == "adam-foreach", fused=how == "adam-fused")
        for _ in range(2):
            opt.zero_grad()
            (enc(x) ** 2).sum().backward()
            opt.step()
    elif how == "load_state_dict":
        enc.load_state_dict({k: v * 0.5 for k, v in enc.state_dict().items()})
    else:
        with torch.no_grad():
            enc.table.copy_(enc.table * -1.5)
    after = enc(x).detach()
    assert not torch.equal(after, before)
    assert torch.equal(after, _fresh(enc)(x).detach())


def test_fp16_copy_misses_writes_through_data():
    """`.data` has a version counter of its own: a write through it does not reach the parameter's, so the cached fp16 copy stays stale
    (documented in Encoding.compute_table)."""
    enc, x = _fp16_pair()
    before = enc(x).detach()
    enc.table.data.mul_(-1.5)
    assert torch.equal(enc(x).detach(), before)
    with torch.no_grad():
        enc.table.mul_(1.0)          # any in-place write under no_grad bumps the version: the copy is refreshed
    assert torch.equal(enc(x).detach(), _fresh(enc)(x).detach())


# ----------------------------------------------------------------------------------------------------------------
# the kernels that share the lookup
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("contraction", [False, True])
@pytest.mark.parametrize("F", [1, 4, 8])
def test_density_field_features_per_level(F, contraction):
    import sdfstudio_b200 as sb
    from helpers import assert_within_noise
    from oracle import density as odensity

    aabb = torch.tensor([[-1.0, -1, -1], [1, 1, 1]])
    sd = sb.SceneContraction(order=float("inf")) if contraction else None
    f = sb.HashMLPDensityField(aabb, num_layers=2, hidden_dim=16, spatial_distortion=sd, num_levels=5, max_res=256, log2_hashmap_size=12,
                               features_per_level=F).to(DEV)
    g = torch.Generator().manual_seed(F)
    nb = f.mlp_base
    with torch.no_grad():
        nb.params[nb.n_net:] = ((torch.rand(nb.n_grid, generator=g) * 2 - 1) * 0.5).to(DEV)
    pos = (torch.rand(37, 11, 3, generator=g) * 2 - 1) * (3.0 if contraction else 1.2)
    growth = hashgrid.growth_factor(5, 16, 256)
    p = nb.params.detach().cpu()

    def orc(params, dt):
        return odensity.density_field(pos.to(dt), params[: nb.n_net], params[nb.n_net:], 16, 1, 5, F, 12, 16, growth,
                                      aabb=None if contraction else aabb.to(dt), contraction="linf" if contraction else None)

    f.eval()
    dens, pre = f.density_from_positions(pos.to(DEV), return_pre_activation=True)
    o32, o64 = orc(p, torch.float32), orc(p.double(), torch.float64)
    assert_within_noise(pre, o32[1], o64[1], f"F={F} pre", floor=1e-6 * float(o64[1].abs().max()))
    assert_within_noise(dens, o32[0], o64[0], f"F={F} density", floor=1e-6 * float(o64[0].abs().max()))
    # fp16 table straight through the C-ABI (the module always passes fp32)
    t16 = nb.params.detach()[nb.n_net:].half().contiguous()
    desc = nb.desc
    desc.active_levels, desc.table_dtype = desc.n_levels, sb._lib.DT_F16
    code = sb.density_fields.contraction_code(sd)
    d16 = torch.empty(pos.numel() // 3, device=DEV)
    pq = pos.reshape(-1, 3).to(DEV).contiguous()
    aabb_d = aabb.to(DEV) if not contraction else None
    call("sdfb200_density_field_forward", desc, t16.data_ptr(), nb.params.detach()[: nb.n_net].data_ptr(), 16, 1, code, ptr(aabb_d), pq.data_ptr(),
         pq.shape[0], d16.data_ptr(), None, None)
    desc.table_dtype = sb._lib.DT_F32
    pq16 = torch.cat([p[: nb.n_net], t16.cpu().float()])
    assert_within_noise(d16.view(37, 11, 1), orc(pq16, torch.float32)[0], orc(pq16.double(), torch.float64)[0], f"F={F} fp16 density",
                        floor=1e-6 * float(o64[0].abs().max()))
    # training gradients (the interlevel loss path: grid operator + ATen MLP)
    f.train()
    w = torch.randn(37, 11, 1, generator=g)
    posd = pos.to(DEV)
    (f.density_from_positions(posd) * w.to(DEV)).sum().backward()
    p32 = p.clone().requires_grad_(True)
    p64 = p.double().requires_grad_(True)
    (orc(p32, torch.float32)[0] * w).sum().backward()
    (orc(p64, torch.float64)[0] * w.double()).sum().backward()
    assert_within_noise(nb.params.grad, p32.grad, p64.grad, f"F={F} param grad", floor=1e-6 * float(p64.grad.abs().max()))


def test_angelo_field_fp16_table_matches_oracle_on_the_same_quantised_table():
    """An angelo-shaped SDFField (F = 8, numerical gradients) with table_dtype="fp16" on the generic engine: the oracle holds the same
    fp16-representable table."""
    import sdfstudio_b200 as sb
    from helpers import build_case, make_bundle, oracle64, assert_within_noise

    spec, kw, o, d, cam, nears, fars, oracle_f, field = build_case("angelo_small", precision="fp32", table_dtype="fp16")
    assert field.encoding.n_features_per_level == 8 and field.encoding.compute_table().dtype == torch.float16
    rb = make_bundle(o, d, cam, nears, fars)
    rs = sb.UniformSampler(num_samples=kw["S"]).eval()(rb)
    out = field(rs, return_alphas=True)
    eu = sb.rays.bins_of(rs).cpu()
    oo = oracle_f.get_outputs(o, d, eu[:, :-1], eu[:, 1:] - eu[:, :-1], cam, return_alphas=True)
    o64 = oracle64(spec, oracle_f.p, kw)
    e64 = o64.get_outputs(o.double(), d.double(), eu[:, :-1].double(), (eu[:, 1:] - eu[:, :-1]).double(), cam, return_alphas=True)
    H = sb.FieldHeadNames
    for key, k in ((H.SDF, "sdf"), (H.RGB, "rgb"), (H.ALPHA, "alphas"), (H.GRADIENT, "gradients")):
        assert_within_noise(out[key], oo[k], e64[k], f"angelo fp16-table/{k}", factor=4.0, floor=1e-4 * float(e64[k].abs().max()))
