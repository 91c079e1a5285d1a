"""The compositing kernels (csrc/render.cu, csrc/render_backward.cu) against fp64 torch autograd over the reference formulas
(oracle/samplers.weights_from_{alphas,density}, oracle/render.py), at the shapes where the warp scans change shape (S = 1, 2, 31, 32, 33,
64, 65, 257, 1024), every background mode, every subset of per-ray gradients, the depth clip's edges, the segmented packed kernels and
the packed renderer branch under autograd.

Bounds.  u = 2^-24 (fp32 unit roundoff).  "Per element" bounds are |cuda - fp64| <= rel * M + tiny, where M is the element's magnitude
scale: |value| for a forward output, and for a gradient the same sum with every term taken in absolute value (computed in fp64), so that
a gradient that cancels to ~0 is held to the rounding of the terms it is made of, not to 0.  `tiny` = 2^-126 (fp32's smallest normal)
covers transmittances that underflow in fp32 exactly as in the reference's own fp32.
* alpha weights / transmittance: (S + 8) * 2u relative -- the S factors (1 - alpha + 1e-7) are rounded to fp32 once each (the kernels
  multiply them in double), as in the reference's fp32 cumprod.  k_weights_bwd forms its suffix sums as (row total - prefix) in double,
  which adds an absolute S * 2^-50 * row total / f to the gradients.
* alpha-mode gradients at and after a saturated sample (alpha = 1: the gradient divides by f = 1e-7): within 4x the fp32 oracle's own
  error against fp64 (helpers.assert_within_noise), with a floor of 2e-6 x the gradient tensor's max.
* density weights / gradients: 1.2e-5 relative -- delta * sigma summed over a ray stays below 12 by construction, and each of delta, f
  and T carries at most 4 fp32 roundings of a quantity of that size (12 * 4 * u = 2.9e-6, 4x margin); plus an absolute 4u T per
  weight, because 1 - exp(-delta sigma) cancels and expf is within 2 ulp, as in the reference's own fp32.
* rendered rgb / depth / normal / accumulation and their gradients: (S + 8) * 2u relative to the sum of the absolute terms (the
  classic bound of recursive fp32 summation; the weights themselves are inputs there).  d/dalpha through the renderers composes two
  such stages: 4 (S + 8) * 2u.
* segmented packed kernels: double sums and products rounded once or twice: 4u relative to the magnitude.
* median depth: bit-exact against the reference's fp32 cumsum (CPU cumsum accumulates in double, as the kernel does, so the same
  prefixes round to the same floats and the tie at exactly 0.5 resolves the same way; no flip was allowed or needed).
* steps_minmax: exact (min / max are exact operations on dyadic bins).
None of these bounds rests on a measurement except the noise-relative one, whose factor 4 follows the rest of the suite.
"""
import math

import pytest
import torch

from oracle import render as orender
from oracle import samplers as osamp

from helpers import assert_within_noise

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TINY = 2.0 ** -126
S_SET = [1, 2, 31, 32, 33, 64, 65, 257, 1024]
R_SET = [1, 7, 129, 4097]
BG_MODES = ["color", "per_ray", "last_sample"]


def _sb():
    import sdfstudio_b200 as sb

    return sb


def _lib():
    return _sb()._lib


def _assert_elem(cuda, ref, scale, rel, what, tiny=TINY):
    """|cuda - ref| <= rel * scale + tiny, element-wise (ref, scale in fp64 on the CPU)."""
    c = cuda.detach().double().cpu()
    err = (c - ref).abs()
    lim = rel * scale.abs() + tiny
    bad = ~(err <= lim)
    if bool(bad.any()):
        i = int(torch.nonzero(bad.reshape(-1))[0])
        raise AssertionError(f"{what}: {int(bad.sum())} elements out of bound; first flat index {i}: cuda {c.reshape(-1)[i].item():.9g} "
                             f"ref {ref.reshape(-1)[i].item():.9g} scale {scale.reshape(-1)[i].item():.3g} rel {rel:.3g}")


def _canary(t, slack):
    """t flattened into a buffer followed by `slack` NaNs: a kernel that reads past the columns it was given picks up NaN."""
    buf = torch.full((t.numel() + slack,), float("nan"), device="cuda")
    buf[: t.numel()] = t.reshape(-1).cuda()
    return buf


# ------------------------------------------------------------------------------------------------------------------------------ inputs
def _alphas(R, S, g):
    a = torch.rand(R, S, generator=g) ** 3
    if R >= 7:
        a[1] = 0.0                                  # nothing absorbs: T = (1 + 1e-7)^i
        a[2] = 1.0                                  # every sample saturated: T underflows in fp32 after 6 samples
        a[3, S // 2] = 1.0                          # one saturated sample
        a[4, S // 3: S // 3 + 3] = 1.0              # a run of three
        a[5, -1] = 1.0
    return a


def _bins(R, S, g, zero_len=False):
    """[R, S+1] euclidean bins, spacing ~ 2/S (so delta * sigma summed over a ray stays moderate), optionally zero-length bins."""
    d = (torch.rand(R, S, generator=g) + 0.5) * (2.0 / S)
    if zero_len and R >= 7:
        d[6, ::3] = 0.0
    return torch.cat([torch.full((R, 1), 0.5), 0.5 + torch.cumsum(d, 1)], 1)


def _density(R, S, g):
    s = torch.rand(R, S, generator=g) * 5.0
    if R >= 7:
        s[1] = 0.0                                  # density 0
        s[2, S // 2] = 1e6                          # f = exp(-delta sigma) = 0: T after it is 0
        s[3, :] = 1e6 if S <= 2 else s[3, :]
    return s


def _wbwd(x, bins, from_density, g_w, g_T, cols):
    """sdfb200_weights_backward called directly, g_T behind a NaN canary (cols = 0: NULL)."""
    lib = _lib().load()
    R, S = x.shape
    g_in = torch.full((R, S), float("nan"), device="cuda")
    gt = _canary(g_T, S + 2) if cols else None
    _lib().check(lib.sdfb200_weights_backward(_lib().ptr(x), _lib().ptr(bins), from_density, R, S, _lib().ptr(g_w), _lib().ptr(gt), cols,
                                              _lib().ptr(g_in), _lib().stream_ptr()), "sdfb200_weights_backward")
    return g_in


# ------------------------------------------------------------------------------------------------------------ A. weights fwd + bwd
def _alpha_scale(a64, w64, T64, gw, gT, cols):
    """per-element magnitude of d/dalpha: |gw_i| T_i + (sum_{k>i} |gw_k| w_k + |gT_k| T_k + |gT_S| T_S) / f_i; and the absolute slack of
    the kernel's suffix sums, which it forms as (row total - prefix) in double: S * 2^-50 * row total / f_i (8x the 2^-53 per add)."""
    R, S = a64.shape
    f = 1.0 - a64 + 1e-7
    terms = gw.abs() * w64
    tail = torch.zeros(R, S, dtype=torch.float64)
    if cols == S + 1:
        terms = terms + gT[:, :S].abs() * T64[:, :S]
    if cols:
        tail = tail + (gT[:, -1:].abs() * T64[:, -1:])
    suffix = terms.flip(1).cumsum(1).flip(1) - terms            # sum over k > i
    total = terms.sum(1, keepdim=True) + tail
    return gw.abs() * T64[:, :S] + (suffix + tail) / f, S * 2.0 ** -50 * total / f + TINY


@pytest.mark.parametrize("S", S_SET)
def test_weights_from_alphas_forward_backward(S):
    """Forward weights / every transmittance column, and d/dalpha through the weights with gt_cols = 0, 1 (the last column only, what
    RenderAlphasFn passes) and S + 1 (every column, WeightsFromAlphasFn), for R in {1, 7, 129, 4097}."""
    sb = _sb()
    g = torch.Generator().manual_seed(100 + S)
    for R in R_SET:
        a = _alphas(R, S, g)
        ac = a.cuda()
        w, T = sb.rays.weights_from_alphas(ac[..., None], True)
        a64 = a.double().requires_grad_(True)
        w64, T64 = osamp.weights_from_alphas(a64)
        rel = (S + 8) * 2 * U
        _assert_elem(w[..., 0], w64.detach(), w64.detach(), rel, f"weights R={R} S={S}")
        _assert_elem(T[..., 0], T64.detach(), T64.detach(), rel, f"transmittance R={R} S={S}")
        a32 = a.clone().requires_grad_(True)
        w32, T32 = osamp.weights_from_alphas(a32)
        gw = torch.randn(R, S, generator=g)
        gT = torch.randn(R, S + 1, generator=g)
        sat = (a >= 1.0).int().cumsum(1) > 0                    # at or after a saturated sample
        for cols in (0, 1, S + 1):
            gTc = gT[:, -1:] if cols == 1 else gT
            loss64 = (w64 * gw.double()).sum()
            loss32 = (w32 * gw).sum()
            if cols:
                loss64 = loss64 + (T64[:, -cols:] * gTc.double()).sum()
                loss32 = loss32 + (T32[:, -cols:] * gTc).sum()
            ref = torch.autograd.grad(loss64, a64, retain_graph=True)[0]
            ref32 = torch.autograd.grad(loss32, a32, retain_graph=True)[0]
            got = _wbwd(ac, None, 0, gw.cuda(), gTc, cols).cpu()
            scale, slack = _alpha_scale(a.double(), w64.detach(), T64.detach(), gw.double(), gT.double() if cols == S + 1 else gTc.double(), cols)
            what = f"d/dalpha R={R} S={S} gt_cols={cols}"
            _assert_elem(got[~sat], ref[~sat], scale[~sat], (S + 8) * 2 * U, what, tiny=slack[~sat])
            if bool(sat.any()):
                assert_within_noise(got[sat], ref32[sat], ref[sat], what + " (saturated)", floor=2e-6 * float(ref.abs().max()))
        # the autograd Function (full-width transmittance gradient) is the same kernel
        ag = ac.clone().requires_grad_(True)
        wg, Tg = sb.rays.weights_from_alphas(ag[..., None], True)
        gfn = torch.autograd.grad((wg[..., 0] * gw.cuda()).sum() + (Tg[..., 0] * gT.cuda()).sum(), ag)[0]
        assert torch.equal(gfn, _wbwd(ac, None, 0, gw.cuda(), gT, S + 1))


def _density_ref(dens, bins):
    d64 = dens.double().requires_grad_(True)
    deltas = (bins[:, 1:] - bins[:, :-1]).double()
    w64, T64 = osamp.weights_from_density(deltas, d64)
    return d64, deltas, w64, T64


@pytest.mark.parametrize("S", S_SET)
def test_weights_from_density_forward_backward(S):
    """density -> weights / transmittance [R,S] and d/dsigma with gt_cols = 0 and S (every column), including density 0, density 1e6
    (f = 0) and zero-length bins (delta = 0)."""
    sb = _sb()
    g = torch.Generator().manual_seed(200 + S)
    for R in R_SET:
        dens, bins = _density(R, S, g), _bins(R, S, g, zero_len=True)
        dc, bc = dens.cuda(), bins.cuda()
        w, T = sb.rays.weights_from_density(bc, dc[..., None], True)
        d64, deltas, w64, T64 = _density_ref(dens, bins)
        rel = 1.2e-5
        # 1 - exp(-delta sigma) cancels: expf's 2-ulp error near 1 (2u) becomes an absolute error of the weight of 2u T (4u T: 2x margin)
        _assert_elem(w[..., 0], w64.detach(), w64.detach(), rel, f"density weights R={R} S={S}", tiny=4 * U * T64.detach() + TINY)
        _assert_elem(T[..., 0], T64.detach(), T64.detach(), rel, f"density transmittance R={R} S={S}")
        gw, gT = torch.randn(R, S, generator=g), torch.randn(R, S, generator=g)
        f64 = torch.exp(-deltas * dens.double())
        for cols in (0, S):
            loss = (w64 * gw.double()).sum() + ((T64 * gT.double()).sum() if cols else 0.0)
            ref = torch.autograd.grad(loss, d64, retain_graph=True)[0]
            terms = gw.double().abs() * w64.detach() + (gT.double().abs() * T64.detach() if cols else 0.0)
            suffix = terms.flip(1).cumsum(1).flip(1) - terms
            scale = deltas * (gw.double().abs() * T64.detach() * f64 + suffix)
            # suffix = row total - prefix, in double; and each w_k = (1 - expf(-dd)) T_k carries an absolute 2u T_k (4u: 2x margin)
            tw = gw.double().abs() * T64.detach()
            slack = deltas * (S * 2.0 ** -50 * terms.sum(1, keepdim=True) + 4 * U * (tw.flip(1).cumsum(1).flip(1) - tw)) + TINY
            got = _wbwd(dc, bc, 1, gw.cuda(), gT, cols)
            _assert_elem(got, ref, scale, rel, f"d/dsigma R={R} S={S} gt_cols={cols}", tiny=slack)
            if R >= 7:
                assert float(got[6, ::3].abs().max()) == 0.0            # delta = 0: no gradient


# ------------------------------------------------------------------------------------------------------- B / C. render, render_alphas
def _render_inputs(R, S, g, bg_mode):
    w = (torch.rand(R, S, generator=g) ** 2) * (1.5 / S)
    rgb = torch.rand(R, S, 3, generator=g) * 1.2 - 0.1                  # rgb_padding pushes colours outside [0, 1]
    nrm = torch.randn(R, S, 3, generator=g)
    bins = _bins(R, S, g)
    if R >= 4:
        w[0] = 0.0                                                     # accumulation 0: depth 0, clipped; no gradient through the clip
        w[1] = w[1] * (1.0 / w[1].sum().clamp_min(1e-30)) * 1.3        # accumulation > 1: 1 - acc < 0
        rgb[2], rgb[3] = 1.1, -0.1                                     # composites outside [0, 1] in every background mode
    bg = {"color": torch.tensor([1.3, -0.2, 0.5]), "per_ray": torch.rand(R, 3, generator=g) * 1.4 - 0.2, "last_sample": "last_sample"}[bg_mode]
    return w, rgb, nrm, bins, bg


def _ref_outputs(w, rgb, nrm, bins, bg, clip=True):
    """fp64 reference (oracle/render.py): rgb (unclamped), depth (clipped or not), normal, accumulation."""
    steps = ((bins[:, :-1] + bins[:, 1:]) / 2)[..., None]
    o_rgb = orender.render_rgb(rgb, w[..., None], bg if isinstance(bg, str) else bg.double(), training=True)
    acc = orender.render_accumulation(w[..., None])
    if clip:
        o_d = orender.render_depth(w[..., None], steps, steps)
    else:
        o_d = torch.sum(w[..., None] * steps, dim=-2) / (acc + 1e-10)
    o_n = orender.render_semantics(nrm, w[..., None])
    return o_rgb, o_d, o_n, acc


def _abs_scale(w, rgb, nrm, bins, bg):
    """per-ray magnitudes: sum |w c| + |bg| |1 - acc|, sum |w step|, sum |w n|, sum |w|."""
    wa = w.abs()[..., None]
    acc = w.sum(1, keepdim=True)
    b = rgb[:, -1] if isinstance(bg, str) else bg.double().expand(w.shape[0], 3)
    steps = ((bins[:, :-1] + bins[:, 1:]) / 2).double()
    return ((wa * rgb.abs()).sum(1) + b.abs() * (1 - acc).abs(), (w.abs() * steps.abs()).sum(1, keepdim=True), (wa * nrm.abs()).sum(1),
            wa.sum(1))


@pytest.mark.parametrize("bg_mode", BG_MODES)
@pytest.mark.parametrize("S", [1, 33, 257])
def test_render_forward_every_background_and_clamp(bg_mode, S):
    """k_render (no-grad renderers) and RenderFn: rgb in every background mode with clamp01 on and off, expected depth with the batch
    clip, normal and accumulation, against fp64; rays with accumulation 0 and above 1."""
    sb = _sb()
    g = torch.Generator().manual_seed(300 + S)
    R = 129
    w, rgb, nrm, bins, bg = _render_inputs(R, S, g, bg_mode)
    o_rgb, o_d, o_n, acc = _ref_outputs(w.double(), rgb.double(), nrm.double(), bins.double(), bg)
    s_rgb, s_d, s_n, s_a = _abs_scale(w.double(), rgb.double(), nrm.double(), bins, bg)
    rel = (S + 8) * 2 * U
    bgc = bg if isinstance(bg, str) else bg.cuda()
    for clamp in (False, True):
        got = sb.renderers._render(w.cuda()[..., None], rgb=rgb.cuda(), normals=nrm.cuda(), bins=bins.cuda(), background=bgc, clamp01=clamp,
                                   depth_method="expected", want_acc=True, want_normal=True)
        ref_rgb = o_rgb.clamp(0, 1) if clamp else o_rgb
        _assert_elem(got["rgb"], ref_rgb, s_rgb, rel, f"rgb clamp01={clamp}")
        if clamp:
            assert float(got["rgb"].min()) >= 0.0 and float(got["rgb"].max()) <= 1.0
            assert bool(((o_rgb < 0) | (o_rgb > 1)).any())              # the clamp binds somewhere
        _assert_elem(got["depth"], o_d, s_d / acc.abs().clamp_min(1e-10) + o_d.abs(), rel, "depth")
        _assert_elem(got["normal"], o_n, s_n, rel, "normal")
        _assert_elem(got["accumulation"], acc, s_a, rel, "accumulation")
    assert float(got["depth"][0]) == float(((bins[:, :-1] + bins[:, 1:]) / 2).min())   # acc 0: depth 0 clipped to the batch minimum


_SUBSETS = [tuple(bool(m >> k & 1) for k in range(4)) for m in range(16)]   # (rgb, depth, normal, acc) used in the loss


def _render_bwd_direct(w, rgb, nrm, bins, bg, bg_mode, acc, depth, grads, g_w_in=None):
    """sdfb200_render_backward with NULL for every absent per-ray gradient; the per-sample outputs start as NaN to see the zero-fill."""
    lib = _lib().load()
    R, S = w.shape
    g_rgb, g_d, g_n, g_a = grads
    g_w = torch.full((R, S), float("nan"), device="cuda")
    g_rgb_s = torch.full((R, S, 3), float("nan"), device="cuda")
    g_n_s = torch.full((R, S, 3), float("nan"), device="cuda")
    p = _lib().ptr
    _lib().check(lib.sdfb200_render_backward(p(w), p(rgb), p(nrm), p(bins), p(bg), bg_mode, R, S, p(acc), p(depth), p(g_rgb), p(g_d), p(g_n),
                                             p(g_a), p(g_w_in), p(g_w), p(g_rgb_s), p(g_n_s), _lib().stream_ptr()), "sdfb200_render_backward")
    return g_w, g_rgb_s, g_n_s


def _bg_args(bg, R):
    L = _lib()
    if isinstance(bg, str):
        return L.BG_LAST_SAMPLE, None
    return (L.BG_PER_RAY if bg.dim() == 2 else L.BG_COLOR), bg.cuda().contiguous()


@pytest.mark.parametrize("bg_mode", BG_MODES)
@pytest.mark.parametrize("S", [1, 2, 77])
def test_render_backward_every_gradient_subset(bg_mode, S):
    """k_render_bwd for each of the 16 subsets of (rgb, depth, normal, accumulation) in the loss, with absent gradients passed as NULL
    (the kernel zero-fills g_rgb_samples / g_normal_samples) and, through RenderFn, as autograd hands them over; against fp64 autograd
    over the unclipped reference formulas.  BG_LAST_SAMPLE adds g (1 - acc) to the last sample's colour."""
    sb = _sb()
    g = torch.Generator().manual_seed(400 + S)
    R = 97
    w, rgb, nrm, bins, bg = _render_inputs(R, S, g, bg_mode)
    bmode, bg_t = _bg_args(bg, R)
    wc, rgbc, nrmc, binsc = w.cuda(), rgb.cuda(), nrm.cuda(), bins.cuda()
    o_rgb, o_d, o_n, o_acc, _ = sb.autograd_ops.RenderFn.apply(wc, rgbc, nrmc, binsc, bg_t, bmode)
    c = [torch.randn(R, 3, generator=g), torch.randn(R, generator=g), torch.randn(R, 3, generator=g), torch.randn(R, generator=g)]
    w64, rgb64, n64 = (t.double().requires_grad_(True) for t in (w, rgb, nrm))
    r_rgb, r_d, r_n, r_a = _ref_outputs(w64, rgb64, n64, bins.double(), bg, clip=False)
    refs = [r_rgb, r_d[:, 0], r_n, r_a[:, 0]]
    rel = (S + 8) * 2 * U
    steps = ((bins[:, :-1] + bins[:, 1:]) / 2).double()
    accd = w.double().sum(1, keepdim=True)
    b64 = rgb.double()[:, -1] if isinstance(bg, str) else bg.double().expand(R, 3)
    for sub in _SUBSETS:
        loss = sum((refs[k] * c[k].double()).sum() for k in range(4) if sub[k]) + 0.0 * w64.sum() + 0.0 * rgb64.sum() + 0.0 * n64.sum()
        gw_r, grgb_r, gn_r = torch.autograd.grad(loss, [w64, rgb64, n64], retain_graph=True)
        # scale of d/dw: |g_rgb| |c - bg| + |g_n| |n| + |g_acc| + |g_d| (|step| + |depth|) / (acc + 1e-10)
        sc = torch.zeros(R, S, dtype=torch.float64)
        if sub[0]:
            sc += (c[0].double().abs()[:, None] * (rgb.double() - b64[:, None]).abs()).sum(-1)
        if sub[1]:
            sc += c[1].double().abs()[:, None] * (steps.abs() + r_d.detach().abs()) / (accd + 1e-10)
        if sub[2]:
            sc += (c[2].double().abs()[:, None] * nrm.double().abs()).sum(-1)
        if sub[3]:
            sc += c[3].double().abs()[:, None]
        grads = [c[k].cuda() if sub[k] else None for k in range(4)]
        g_w, g_rgb_s, g_n_s = _render_bwd_direct(wc, rgbc, nrmc, binsc, bg_t, bmode, o_acc, o_d, grads)
        what = f"{bg_mode} S={S} subset={sub}"
        _assert_elem(g_w, gw_r, sc, rel, "d/dw " + what)
        s_rgb_s = grgb_r.abs() + c[0].double().abs()[:, None] * accd[..., None].abs()   # g (1 - acc) at the last sample: acc's rounding
        _assert_elem(g_rgb_s, grgb_r, s_rgb_s, rel, "d/drgb " + what)
        _assert_elem(g_n_s, gn_r, gn_r, 4 * U, "d/dnormal " + what)
        if any(sub):     # through autograd (unused outputs arrive as zero tensors)
            wa, ra, na = (t.clone().requires_grad_(True) for t in (wc, rgbc, nrmc))
            outs = sb.autograd_ops.RenderFn.apply(wa, ra, na, binsc, bg_t, bmode)
            lc = sum((outs[k] * c[k].cuda()).sum() for k in range(4) if sub[k])
            ga = torch.autograd.grad(lc, [wa, ra, na])
            _assert_elem(ga[0], gw_r, sc, rel, "RenderFn d/dw " + what)
            _assert_elem(ga[1], grgb_r, s_rgb_s, rel, "RenderFn d/drgb " + what)


def test_render_depth_clip_gradient_and_median():
    """Training path of the renderers: the clipped expected depth of a ray with accumulation 0 has gradient 0 (clamp at the batch
    minimum), like the reference's torch.clip; median depth is bit-exact against the reference's fp32 cumsum at an exact 0.5 tie, when
    the cumsum never reaches 0.5 (index clamped to S - 1) and on random rays."""
    sb = _sb()
    g = torch.Generator().manual_seed(7)
    R, S = 300, 40
    w, rgb, nrm, bins, bg = _render_inputs(R, S, g, "color")

    class _RS:
        _euclid_bins = bins.cuda()

    wc = w.cuda()[..., None].requires_grad_(True)
    d = sb.DepthRenderer("expected")(wc, _RS)
    cd = torch.randn(R, 1, generator=g)
    gw = torch.autograd.grad((d * cd.cuda()).sum(), wc)[0][..., 0].cpu()
    w64 = w.double().requires_grad_(True)
    steps = ((bins[:, :-1] + bins[:, 1:]) / 2).double()[..., None]
    ref = torch.autograd.grad((orender.render_depth(w64[..., None], steps, steps) * cd.double()).sum(), w64)[0]
    assert float(gw[0].abs().max()) == 0.0 and float(ref[0].abs().max()) == 0.0
    sc = cd.double().abs() * (steps[..., 0].abs() + float(steps.abs().max())) / (w.double().sum(1, keepdim=True) + 1e-10)
    _assert_elem(gw[1:], ref[1:], sc[1:], (S + 8) * 2 * U, "clipped depth d/dw")

    wm = torch.rand(R, S, generator=g) * (1.0 / S)
    wm[2] = 0.0
    wm[2, :4] = torch.tensor([0.25, 0.125, 0.125, 0.5])     # cumsum 0.25, 0.375, 0.5 (exact tie at index 2), 1.0
    wm[3] = 1e-3                                            # cumsum never reaches 0.5: index clamped to S - 1
    wm[4, :2] = 0.5                                         # tie at the first step
    for med_w in (wm, w):
        got = sb.DepthRenderer("median")(med_w.cuda()[..., None], _RS).cpu()
        st32 = ((bins[:, :-1] + bins[:, 1:]) / 2)[..., None]
        ref32 = orender.render_depth(med_w[..., None], st32, st32, method="median")
        assert torch.equal(got, ref32), int((got != ref32).sum())
    got = sb.DepthRenderer("median")(wm.cuda()[..., None], _RS).cpu()
    assert float(got[2]) == float(st32[2, 2]) and float(got[3]) == float(st32[3, -1]) and float(got[4]) == float(st32[4, 0])


@pytest.mark.parametrize("bg_mode", BG_MODES)
@pytest.mark.parametrize("S", S_SET)
def test_render_alphas_forward_backward(bg_mode, S):
    """k_render_alphas / RenderAlphasFn: weights, rgb (clamp01 on and off), clipped expected depth, normal, accumulation,
    bg_transmittance and every input gradient against fp64 autograd, on alphas with saturated samples; and the fused launch agrees with
    weights -> k_render on the same inputs to within the rounding of the summation order."""
    sb = _sb()
    g = torch.Generator().manual_seed(500 + S)
    R = 129
    a = _alphas(R, S, g)
    _, rgb, nrm, bins, bg = _render_inputs(R, S, g, bg_mode)

    class _RS:
        _euclid_bins = bins.cuda()

    bgc = bg if isinstance(bg, str) else bg.cuda()
    c = [torch.randn(R, 3, generator=g), torch.randn(R, 1, generator=g), torch.randn(R, 3, generator=g), torch.randn(R, 1, generator=g),
         torch.randn(R, 1, generator=g), torch.randn(R, S, 1, generator=g)]
    ac, rc, nc = (t.cuda().requires_grad_(True) for t in (a[..., None], rgb, nrm))
    res = sb.render_from_alphas(ac, rc, nc, _RS, bgc, training=True)
    keys = ["rgb", "depth", "normal", "accumulation", "bg_transmittance", "weights"]
    loss_c = sum((res[k] * c[i].cuda()).sum() for i, k in enumerate(keys))
    ga, gr, gn = torch.autograd.grad(loss_c, [ac, rc, nc])

    def ref_loss(aa, rr, nn_, dt):
        w, T = osamp.weights_from_alphas(aa)
        o_rgb, o_d, o_n, acc = _ref_outputs(w, rr, nn_, bins.to(dt), bg if isinstance(bg, str) else bg.to(dt))
        outs = [o_rgb, o_d, o_n, acc, T[:, -1:], w[..., None]]
        return sum((o * ci.to(dt)).sum() for o, ci in zip(outs, c)), outs

    a64, r64, n64 = (t.double().requires_grad_(True) for t in (a, rgb, nrm))
    l64, outs64 = ref_loss(a64, r64, n64, torch.float64)
    ga_r, gr_r, gn_r = torch.autograd.grad(l64, [a64, r64, n64])
    a32, r32, n32 = (t.clone().requires_grad_(True) for t in (a, rgb, nrm))
    l32, _ = ref_loss(a32, r32, n32, torch.float32)
    ga_32 = torch.autograd.grad(l32, [a32])[0]

    rel = (S + 8) * 2 * U
    w64 = outs64[5][..., 0].detach()
    s_rgb, s_d, s_n, s_a = _abs_scale(w64, rgb.double(), nrm.double(), bins, bg)
    _assert_elem(res["weights"][..., 0], w64, w64, rel, "weights")
    _assert_elem(res["bg_transmittance"], outs64[4].detach(), outs64[4].detach(), rel, "bg_transmittance")
    _assert_elem(res["rgb"], outs64[0].detach(), s_rgb + rel * s_a, 2 * rel, "rgb")
    _assert_elem(res["depth"], outs64[1].detach(), s_d / s_a.clamp_min(1e-10) + outs64[1].detach().abs(), 2 * rel, "depth")
    _assert_elem(res["normal"], outs64[2].detach(), s_n, 2 * rel, "normal")
    _assert_elem(res["accumulation"], outs64[3].detach(), s_a, 2 * rel, "accumulation")
    _assert_elem(gr, gr_r, gr_r.abs() + c[0].double().abs()[:, None] * s_a[..., None], 2 * rel, "d/drgb")
    _assert_elem(gn, gn_r, gn_r.abs(), 2 * rel, "d/dnormal")
    # d/dalpha away from saturation: the per-sample d/dw magnitude (every term of k_render_bwd in absolute value; the depth term
    # (step - depth) / acc is ill-conditioned at small accumulation in the reference's own fp32 too) pushed through the alpha scale
    steps = ((bins[:, :-1] + bins[:, 1:]) / 2).double()
    b64 = rgb.double()[:, -1] if isinstance(bg, str) else bg.double().expand(R, 3)
    acc64 = outs64[3].detach()
    sc_w = (c[0].double().abs()[:, None] * (rgb.double() - b64[:, None]).abs()).sum(-1) + (c[2].double().abs()[:, None] * nrm.double().abs()).sum(-1) \
        + c[1].double().abs() * (steps.abs() + outs64[1].detach().abs()) / (acc64 + 1e-10) + c[3].double().abs() + c[5][..., 0].double().abs()
    T64 = osamp.weights_from_alphas(a.double())[1]
    sc_a, slack = _alpha_scale(a.double(), w64, T64, sc_w, c[4].double(), 1)
    sat = (a >= 1.0).int().cumsum(1) > 0
    ga = ga[..., 0].cpu()
    scale = float(ga_r.abs().max())
    _assert_elem(ga[~sat], ga_r[~sat], sc_a[~sat], 4 * rel, f"d/dalpha {bg_mode} S={S}", tiny=slack[~sat])
    if bool(sat.any()):
        assert_within_noise(ga[sat], ga_32[sat], ga_r[sat], f"d/dalpha saturated {bg_mode} S={S}", floor=2e-6 * scale)

    # the same inputs through weights -> k_render (the unfused renderers, no grad)
    with torch.no_grad():
        fused = sb.render_from_alphas(a.cuda()[..., None], rgb.cuda(), nrm.cuda(), _RS, bgc, training=False)
        w2 = sb.rays.weights_from_alphas(a.cuda()[..., None])
        sep = sb.renderers.render_all(w2, rgb.cuda(), nrm.cuda(), _RS, bgc, training=False)
    wf = fused["weights"][..., 0]
    assert float(((wf - w2[..., 0]).abs() - 2 * 2 * U * w2[..., 0].abs()).max()) <= TINY      # <= 2 ulp (different product order)
    wabs = w2[..., 0].double().abs().cpu()
    s_sum = (S + math.log2(S) + 4) * U
    for k, sc in (("rgb", (wabs[..., None] * rgb.double().abs()).sum(1) + 3.0 * (1 + wabs.sum(1, keepdim=True))), ("normal", (wabs[..., None] * nrm.double().abs()).sum(1)),
                  ("accumulation", wabs.sum(1, keepdim=True))):
        d = (fused[k].double().cpu() - sep[k].double().cpu()).abs()
        assert bool((d <= s_sum * sc + 2 * U * fused[k].double().abs().cpu() + TINY).all()), (k, float(d.max()))


# ------------------------------------------------------------------------------------------------------------ D. depth clip / minmax
@pytest.mark.parametrize("R", [1, 31, 33, 127, 129])
def test_steps_minmax_exact(R):
    """steps_minmax of k_render, k_render_alphas and the packed render equals the fp64 min / max of the steps exactly when R is not a
    multiple of 32 or 128 (lanes past R join the shuffle reduction with +-inf), with the extremes on the last ray, then on the first."""
    sb = _sb()
    g = torch.Generator().manual_seed(600 + R)
    S = 9
    for last in (True, False):
        q = torch.randint(1, 64, (R, S + 1), generator=g).float().cumsum(1) / 1024.0 + 2.0   # dyadic: (a + b) / 2 is exact in fp32
        edge = R - 1 if last else 0
        q[edge] = q[edge] - q[edge, 0] + 0.25                    # the smallest step
        q[edge, -1] = 50.0                                       # the largest
        steps64 = (q[:, :-1].double() + q[:, 1:].double()) / 2
        lo, hi = float(steps64.min()), float(steps64.max())
        w = torch.rand(R, S, generator=g) * 0.1
        _, _, _, _, mm = sb.autograd_ops.RenderFn.apply(w.cuda(), None, None, q.cuda(), None, _lib().BG_COLOR)
        assert mm.tolist() == [lo, hi]
        a = torch.rand(R, S, generator=g) * 0.3
        outs = sb.autograd_ops.RenderAlphasFn.apply(a.cuda(), torch.rand(R, S, 3).cuda(), torch.rand(R, S, 3).cuda(), q.cuda(),
                                                    torch.zeros(3).cuda(), _lib().BG_COLOR)
        assert outs[6].tolist() == [lo, hi]
        ri = torch.arange(R).repeat_interleave(S)
        st, en = q[:, :-1].reshape(-1).cuda(), q[:, 1:].reshape(-1).cuda()
        outs = sb.autograd_ops.PackedRenderFn.apply(w.reshape(-1).cuda(), None, None, st, en, ri.cuda(), R, None, _lib().BG_COLOR)
        assert outs[4].tolist() == [lo, hi]

        class _Fr:
            starts, ends = st[:, None], en[:, None]

        class _RSp:
            frustums = _Fr

        wz = torch.zeros(R * S, 1)                                 # every ray accumulation 0: packed depth = clip(0) = batch min
        dep = sb.DepthRenderer("expected")(wz.cuda(), _RSp, ray_indices=ri.cuda(), num_rays=R)
        assert dep.reshape(-1).tolist() == [lo] * R


# ------------------------------------------------------------------------------------------------------------ E. packed, segmented
def _segments(g, lens):
    """ray_indices of segments with the given lengths (sorted, so the segmented kernels take them), alphas with runs of 0 and 1."""
    lens = torch.tensor(lens)
    ri = torch.repeat_interleave(torch.arange(len(lens)), lens)
    a = torch.rand(int(lens.sum()), generator=g) ** 2
    off = torch.cat([torch.zeros(1, dtype=torch.int64), lens.cumsum(0)])
    for r, n in enumerate(lens.tolist()):
        b = int(off[r])
        if n >= 33:
            a[b + 3: b + 7] = 0.0                  # a run of alpha 0
            a[b + 20: b + 23] = 1.0                # a run of alpha 1: T = 0 after it
    return ri, a, off


def _packed_weights64(a, off):
    """nerfacc 0.3.5 render_weight_from_alpha in fp64 autograd: w = alpha * exclusive cumprod(1 - alpha) per segment."""
    parts = []
    for r in range(off.numel() - 1):
        s = a[int(off[r]): int(off[r + 1])]
        T = torch.cumprod(torch.cat([torch.ones(1, dtype=s.dtype), 1.0 - s[:-1]]), 0) if s.numel() else s
        parts.append(s * T)
    return torch.cat(parts)


LENS = [0, 1, 31, 32, 33, 4096, 0, 65, 2, 257]


def test_packed_weights_forward_backward_deterministic():
    """k_packed_weights / k_packed_weights_bwd over segments of length {0, 1, 31, 32, 33, 4096, 65, 2, 257} with runs of alpha 0 and 1:
    the forward exclusive product scan and the backward's reverse affine scan (which starts from the last 32-sample row) against fp64
    autograd, bit-identical on a rerun."""
    sb = _sb()
    g = torch.Generator().manual_seed(800)
    ri, a, off = _segments(g, LENS)
    ac = a.cuda().requires_grad_(True)
    w = sb.packed.render_weight_from_alpha(ac, ray_indices=ri.cuda(), n_rays=len(LENS))
    gw = torch.randn(a.shape[0], generator=g)
    ga = torch.autograd.grad((w * gw.cuda()).sum(), ac)[0]
    a64 = a.double().requires_grad_(True)
    w64 = _packed_weights64(a64, off)
    ga64 = torch.autograd.grad((w64 * gw.double()).sum(), a64)[0]
    w64 = w64.detach()
    _assert_elem(w, w64, w64, 4 * U, "packed weights")
    # magnitude of d/dalpha_k = T_k g_k - sum_{j>k} g_j w_j / (1 - alpha_k):  T_k |g_k| + sum_{j>k} |g_j| w_j
    sc = torch.zeros_like(w64)
    for r in range(len(LENS)):
        b, e = int(off[r]), int(off[r + 1])
        if e > b:
            Tseg = torch.cumprod(torch.cat([torch.ones(1, dtype=torch.float64), 1.0 - a.double()[b:e - 1]]), 0)
            t = (gw.double()[b:e].abs() * w64[b:e])
            suf = t.flip(0).cumsum(0).flip(0) - t
            sc[b:e] = Tseg * gw.double()[b:e].abs() + suf
    _assert_elem(ga, ga64, sc, 8 * U, "packed d/dalpha")
    ac2 = a.cuda().requires_grad_(True)
    w2 = sb.packed.render_weight_from_alpha(ac2, ray_indices=ri.cuda(), n_rays=len(LENS))
    assert torch.equal(w2, w) and torch.equal(torch.autograd.grad((w2 * gw.cuda()).sum(), ac2)[0], ga)


@pytest.mark.parametrize("C", [None, 1, 2, 3, 4, 5, 6, 7, 8, 9])
def test_packed_accumulate_every_channel_count(C):
    """k_packed_accumulate / _bwd for C = 1 to 9 (the c0 += 4 loop's partial last group) and values = None, over the same segments:
    index_add in fp64 forward and autograd backward, bit-identical reruns."""
    sb = _sb()
    g = torch.Generator().manual_seed(900 + (C or 0))
    ri, a, off = _segments(g, LENS)
    N, R = a.shape[0], len(LENS)
    w = torch.rand(N, 1, generator=g)
    v = torch.randn(N, C, generator=g) if C else None
    wc = w.cuda().requires_grad_(True)
    vc = v.cuda().requires_grad_(True) if C else None
    out = sb.packed.accumulate_along_rays(wc, ri.cuda(), vc, n_rays=R)
    go = torch.randn(R, C or 1, generator=g)
    grads = torch.autograd.grad((out * go.cuda()).sum(), [wc] + ([vc] if C else []))
    w64 = w.double().requires_grad_(True)
    v64 = v.double().requires_grad_(True) if C else None
    ref = orender.accumulate_along_rays(w64, ri, v64, R)
    ref_g = torch.autograd.grad((ref * go.double()).sum(), [w64] + ([v64] if C else []))
    vabs = v.double().abs() if C else torch.ones(N, 1, dtype=torch.float64)
    sc = orender.accumulate_along_rays(w.double(), ri, vabs, R)
    _assert_elem(out, ref.detach(), sc, 2 * U, f"packed accumulate C={C}")
    _assert_elem(grads[0], ref_g[0], (go.double().abs()[ri] * vabs).sum(1, keepdim=True), 2 * U, f"packed accumulate d/dw C={C}")
    if C:
        _assert_elem(grads[1], ref_g[1], ref_g[1], U, f"packed accumulate d/dvalues C={C}")
    out2 = sb.packed.accumulate_along_rays(w.cuda(), ri.cuda(), v.cuda() if C else None, n_rays=R)
    assert torch.equal(out2, out.detach())
    assert float(out[0].abs().max()) == 0.0 and float(out[6].abs().max()) == 0.0      # empty segments


# ------------------------------------------------------------------------------------------------------------ F. packed renderer branch
class _Frustums:
    def __init__(self, starts, ends):
        self.starts, self.ends = starts, ends


class _PackedSamples:
    def __init__(self, starts, ends):
        self.frustums = _Frustums(starts, ends)


def _packed_inputs(g, R=301, Smax=40):
    counts = torch.randint(0, Smax + 1, (R,), generator=g)
    counts[5] = 0
    counts[R - 1] = 0
    ri = torch.repeat_interleave(torch.arange(R), counts)
    ri = ri[torch.randperm(ri.numel(), generator=g)]           # unsorted: the scatter-add branch takes any order
    N = ri.numel()
    w = torch.rand(N, 1, generator=g) * 0.1
    rgb = torch.rand(N, 3, generator=g) * 1.2 - 0.1
    nrm = torch.randn(N, 3, generator=g)
    starts = torch.rand(N, 1, generator=g) * 3 + 0.5
    ends = starts + torch.rand(N, 1, generator=g) * 0.1
    return ri, w, rgb, nrm, starts, ends


@pytest.mark.parametrize("bg_kind", ["color", "per_ray"])
def test_packed_renderers_forward_and_autograd(bg_kind):
    """The ray_indices / num_rays branch of RGBRenderer, AccumulationRenderer and DepthRenderer on unsorted samples with empty rays:
    forward (eval, clamp01) within bound of the fp64 index_add restatement (float atomics: not bit-identical), and in training the
    outputs carry gradients to weights, rgb and starts / ends equal to fp64 autograd over nerfacc.accumulate_along_rays."""
    sb = _sb()
    g = torch.Generator().manual_seed(1000)
    ri, w, rgb, nrm, starts, ends = _packed_inputs(g)
    R = 301
    bg = torch.tensor([1.2, -0.1, 0.4]) if bg_kind == "color" else torch.rand(R, 3, generator=g)
    Rc = ri.cuda()
    # scale of the sums: per-ray sum |w| |x|
    wd = w.double()
    s_acc = orender.accumulate_along_rays(wd, ri, None, R)
    s_rgb = orender.accumulate_along_rays(wd, ri, rgb.double().abs(), R) + bg.double().abs() * (1 - s_acc).abs()
    steps64 = (starts.double() + ends.double()) / 2
    rel = 64 * 2 * U                                            # <= 40 samples per ray, summed in any order

    with torch.no_grad():
        o_rgb = sb.RGBRenderer(background_color=bg.cuda()).eval()(rgb.cuda(), w.cuda(), ray_indices=Rc, num_rays=R)
        o_acc = sb.AccumulationRenderer.forward(w.cuda(), ray_indices=Rc, num_rays=R)
        o_dep = sb.DepthRenderer("expected")(w.cuda(), _PackedSamples(starts.cuda(), ends.cuda()), ray_indices=Rc, num_rays=R)
    r_rgb = orender.render_rgb_packed(rgb.double(), wd, ri, R, bg.double(), training=True)
    _assert_elem(o_rgb, r_rgb.clamp(0, 1), s_rgb, rel, "packed rgb (eval)")
    _assert_elem(o_acc, s_acc, s_acc, rel, "packed accumulation")
    r_dep = orender.render_depth_packed(wd, starts.double(), ends.double(), ri, R)
    _assert_elem(o_dep, r_dep, torch.full_like(r_dep, float(steps64.max())), rel, "packed depth")
    assert float(o_acc[5]) == 0.0 and torch.equal(o_rgb[5].cpu(), bg.clamp(0, 1)[5] if bg.dim() == 2 else bg.clamp(0, 1))

    # training: gradients through the packed branch
    wc, rc, sc_, ec = (t.cuda().requires_grad_(True) for t in (w, rgb, starts, ends))
    c_rgb, c_acc, c_dep = torch.randn(R, 3, generator=g), torch.randn(R, 1, generator=g), torch.randn(R, 1, generator=g)
    p_rgb = sb.RGBRenderer(background_color=bg.cuda()).train()(rc, wc, ray_indices=Rc, num_rays=R)
    p_acc = sb.AccumulationRenderer.forward(wc, ray_indices=Rc, num_rays=R)
    p_dep = sb.DepthRenderer("expected")(wc, _PackedSamples(sc_, ec), ray_indices=Rc, num_rays=R)
    assert p_rgb.requires_grad and p_acc.requires_grad and p_dep.requires_grad
    loss = (p_rgb * c_rgb.cuda()).sum() + (p_acc * c_acc.cuda()).sum() + (p_dep * c_dep.cuda()).sum()
    gw, grgb, gs, ge = torch.autograd.grad(loss, [wc, rc, sc_, ec])
    w64, rgb64, s64, e64 = (t.double().requires_grad_(True) for t in (w, rgb, starts, ends))
    l64 = (orender.render_rgb_packed(rgb64, w64, ri, R, bg.double(), training=True) * c_rgb.double()).sum() \
        + (orender.accumulate_along_rays(w64, ri, None, R) * c_acc.double()).sum() \
        + (orender.render_depth_packed(w64, s64, e64, ri, R) * c_dep.double()).sum()
    rw, rrgb, rs, re = torch.autograd.grad(l64, [w64, rgb64, s64, e64])
    acc_i = s_acc[ri]
    b_i = bg.double().expand(R, 3)[ri]
    sc_w = (c_rgb.double()[ri].abs() * (rgb.double() - b_i).abs()).sum(1, keepdim=True) + c_acc.double()[ri].abs() \
        + c_dep.double()[ri].abs() * (steps64.abs() + float(steps64.max())) / (acc_i + 1e-10)
    _assert_elem(gw, rw, sc_w, rel, "packed d/dw")
    _assert_elem(grgb, rrgb, rrgb, 4 * U, "packed d/drgb")
    _assert_elem(gs, rs, rs.abs() + 1e-6 * float(rs.abs().max()), 8 * U, "packed d/dstarts")
    _assert_elem(ge, re, re.abs() + 1e-6 * float(re.abs().max()), 8 * U, "packed d/dends")

    # the smallest training use: the sum of the rendered colour
    w1, c1 = w.cuda().requires_grad_(True), rgb.cuda().requires_grad_(True)
    sb.RGBRenderer(torch.ones(3).cuda()).train()(c1, w1, ray_indices=Rc, num_rays=R).sum().backward()
    w1r, c1r = w.double().requires_grad_(True), rgb.double().requires_grad_(True)
    orender.render_rgb_packed(c1r, w1r, ri, R, torch.ones(3, dtype=torch.float64), training=True).sum().backward()
    _assert_elem(w1.grad, w1r.grad, (rgb.double() - 1).abs().sum(1, keepdim=True), 4 * U, "RGBRenderer(...).sum() d/dw")
    _assert_elem(c1.grad, c1r.grad, c1r.grad, U, "RGBRenderer(...).sum() d/drgb")
    with pytest.raises(NotImplementedError):
        sb.RGBRenderer(background_color="last_sample").train()(rc, wc, ray_indices=Rc, num_rays=R)


# ------------------------------------------------------------------------------------------------------------ G. C-ABI refusals
def test_c_abi_refusals_launch_nothing():
    """Bad arguments are refused before any launch: n_samples = 0, a g_transmittance_cols that is neither 1 nor the transmittance's
    width, 'last_sample' with packed samples, and a requested output whose input is missing."""
    L = _lib()
    lib = L.load()
    p, sp = L.ptr, L.stream_ptr()
    R, S = 4, 3
    x = torch.rand(R, S, device="cuda")
    bins = torch.rand(R, S + 1, device="cuda").cumsum(1)
    o = torch.empty(R, 3, device="cuda")
    o1 = torch.empty(R, device="cuda")
    mm = torch.empty(2, device="cuda")
    ri = torch.zeros(R * S, dtype=torch.int64, device="cuda")
    ws = torch.empty(R * 8, device="cuda")
    n0 = L.launch_count()
    calls = {
        "weights_from_alphas S=0": lambda: lib.sdfb200_weights_from_alphas(p(x), R, 0, p(x), None, sp),
        "weights_from_density S=0": lambda: lib.sdfb200_weights_from_density(p(x), p(bins), R, 0, p(x), None, sp),
        "render S=0": lambda: lib.sdfb200_render(p(x), None, None, None, None, L.BG_COLOR, 0, 0, R, 0, L.render_out(accumulation=o1), sp),
        "render_alphas S=0": lambda: lib.sdfb200_render_alphas(p(x), None, None, None, None, L.BG_COLOR, 0, R, 0, None, None,
                                                                L.render_out(accumulation=o1), sp),
        "render_backward S=0": lambda: lib.sdfb200_render_backward(p(x), None, None, None, None, L.BG_COLOR, R, 0, None, None, None, None, None,
                                                                    None, None, p(x), None, None, sp),
        "weights_backward S=0": lambda: lib.sdfb200_weights_backward(p(x), None, 0, R, 0, p(x), None, 0, p(x), sp),
        "alpha gt_cols=2": lambda: lib.sdfb200_weights_backward(p(x), None, 0, R, S, p(x), p(bins), 2, p(x), sp),
        "alpha gt_cols=S": lambda: lib.sdfb200_weights_backward(p(x), None, 0, R, S, p(x), p(bins), S, p(x), sp),
        "density gt_cols=1": lambda: lib.sdfb200_weights_backward(p(x), p(bins), 1, R, S, p(x), p(bins), 1, p(x), sp),
        "density gt_cols=S+1": lambda: lib.sdfb200_weights_backward(p(x), p(bins), 1, R, S, p(x), p(bins), S + 1, p(x), sp),
        "density without bins": lambda: lib.sdfb200_weights_backward(p(x), None, 1, R, S, p(x), None, 0, p(x), sp),
        "packed last_sample": lambda: lib.sdfb200_render_packed(p(x), p(x), None, None, None, p(ri), R * S, R, None, L.BG_LAST_SAMPLE, 0,
                                                                L.render_out(accumulation=o1), p(ws), ws.numel() * 4, sp),
        "packed backward last_sample": lambda: lib.sdfb200_render_packed_backward(p(x), None, None, None, None, p(ri), R * S, R, None,
                                                                                   L.BG_LAST_SAMPLE, None, None, None, None, None, p(o1), p(x), None,
                                                                                   None, None, sp),
        "packed small workspace": lambda: lib.sdfb200_render_packed(p(x), None, None, None, None, p(ri), R * S, R, None, L.BG_COLOR, 0,
                                                                    L.render_out(accumulation=o1), p(ws), 4, sp),
        "render rgb without rgb": lambda: lib.sdfb200_render(p(x), None, None, None, p(o1), L.BG_COLOR, 0, 0, R, S, L.render_out(rgb=o), sp),
        "render rgb without bg": lambda: lib.sdfb200_render(p(x), p(x), None, None, None, L.BG_COLOR, 0, 0, R, S, L.render_out(rgb=o), sp),
        "render depth without bins": lambda: lib.sdfb200_render(p(x), None, None, None, None, L.BG_COLOR, 0, 0, R, S,
                                                                L.render_out(depth=o1, steps_minmax=mm), sp),
        "render normal without normals": lambda: lib.sdfb200_render(p(x), None, None, None, None, L.BG_COLOR, 0, 0, R, S, L.render_out(normal=o), sp),
        "render_alphas depth without bins": lambda: lib.sdfb200_render_alphas(p(x), None, None, None, None, L.BG_COLOR, 0, R, S, None, None,
                                                                              L.render_out(depth=o1), sp),
        "render_backward g_depth without depth": lambda: lib.sdfb200_render_backward(p(x), None, None, p(bins), None, L.BG_COLOR, R, S, p(o1),
                                                                                      None, None, p(o1), None, None, None, p(x), None, None, sp),
        "render_backward g_rgb without rgb": lambda: lib.sdfb200_render_backward(p(x), None, None, None, p(o1), L.BG_COLOR, R, S, p(o1), None,
                                                                                  p(o), None, None, None, None, p(x), None, None, sp),
        "packed depth without starts": lambda: lib.sdfb200_render_packed(p(x), None, None, None, None, p(ri), R * S, R, None, L.BG_COLOR, 0,
                                                                         L.render_out(depth=o1, steps_minmax=mm), p(ws), ws.numel() * 4, sp),
        "packed backward g_depth without depth": lambda: lib.sdfb200_render_packed_backward(p(x), None, None, p(x), p(x), p(ri), R * S, R, None,
                                                                                             L.BG_COLOR, p(o1), None, None, p(o1), None, None,
                                                                                             p(x), None, None, None, sp),
        "packed_accumulate C=2 without values": lambda: lib.sdfb200_packed_accumulate(p(x), None, 2, p(ri), R, p(o), sp),
    }
    for what, call in calls.items():
        assert call() != 0, what
        assert L.launch_count() == n0, what


# ------------------------------------------------------------------------------------------------------------ H. size
def _free_gb():
    return torch.cuda.mem_get_info()[0] / 2 ** 30


def test_render_backward_past_int32_samples():
    """One k_render_bwd call with R * S just above 2^31 (weights, bins and per-ray g_acc / g_depth only, ~26 GB): its element index and
    grid are 64-bit / unsigned; a slice at each end is checked against fp64."""
    need = 30.0
    if _free_gb() < need:
        pytest.skip(f"needs {need:.0f} GiB of free device memory, {_free_gb():.1f} GiB free (the device is shared)")
    S = 1024
    R = (1 << 31) // S + 1                                       # R * S = 2^31 + 1024
    w = torch.rand(R, S, device="cuda")
    bins = torch.arange(S + 1, device="cuda", dtype=torch.float32).mul_(1.0 / 256).expand(R, S + 1).contiguous()
    bins += torch.arange(R, device="cuda", dtype=torch.float32)[:, None].remainder_(97.0)
    acc = torch.rand(R, device="cuda") + 0.5
    depth = torch.rand(R, device="cuda") * 4
    g_acc, g_d = torch.randn(R, device="cuda"), torch.randn(R, device="cuda")
    L = _lib()
    g_w = torch.empty(R, S, device="cuda")
    p = L.ptr
    L.check(L.load().sdfb200_render_backward(p(w), None, None, p(bins), None, L.BG_COLOR, R, S, p(acc), p(depth), None, p(g_d), None,
                                             p(g_acc), None, p(g_w), None, None, L.stream_ptr()), "sdfb200_render_backward")
    for rows in (slice(0, 3), slice(R - 3, R)):
        bb, ww = bins[rows].double().cpu(), g_w[rows].double().cpu()
        steps = (bb[:, :-1] + bb[:, 1:]) / 2
        ref = g_acc[rows].double().cpu()[:, None] + g_d[rows].double().cpu()[:, None] * (steps - depth[rows].double().cpu()[:, None]) \
            / (acc[rows].double().cpu()[:, None] + 1e-10)
        sc = g_acc[rows].double().cpu().abs()[:, None] + g_d[rows].double().cpu().abs()[:, None] * (steps.abs() + 4) / acc[rows].double().cpu()[:, None]
        _assert_elem(ww, ref, sc, 8 * U, f"k_render_bwd rows {rows}")
    del w, bins, g_w


def test_warp_per_ray_kernels_past_2_16_blocks():
    """R > 2^16 * 8 rays in one call of the warp-per-ray kernels (k_render_alphas, k_weights_bwd, k_packed_weights{,_bwd},
    k_packed_accumulate): the last rays, in blocks past 2^16, are checked against fp64."""
    sb = _sb()
    g = torch.Generator().manual_seed(1200)
    R, S = (1 << 16) * 8 + 37, 3
    a = torch.rand(R, S, generator=g)
    ac = a.cuda().requires_grad_(True)
    outs = sb.autograd_ops.RenderAlphasFn.apply(ac, torch.rand(R, S, 3).cuda(), torch.rand(R, S, 3).cuda(), _bins(R, S, g).cuda(),
                                                torch.zeros(3).cuda(), _lib().BG_COLOR)
    gw = torch.randn(R, S, generator=g)
    ga = torch.autograd.grad((outs[0] * gw.cuda()).sum(), ac)[0]
    tail = slice(R - 40, R)
    a64 = a[tail].double().requires_grad_(True)
    w64, _ = osamp.weights_from_alphas(a64)
    ga64 = torch.autograd.grad((w64 * gw[tail].double()).sum(), a64)[0]
    _assert_elem(outs[0][tail], w64.detach(), w64.detach(), 32 * U, "render_alphas weights, last rays")
    _assert_elem(ga[tail], ga64, ga64.abs() + float(ga64.abs().max()) * 1e-6, 64 * U, "weights_bwd, last rays")
    ri = torch.arange(R).repeat_interleave(S).cuda()
    ap = a.reshape(-1).cuda()
    wp = sb.packed.render_weight_from_alpha(ap, ray_indices=ri, n_rays=R)
    acc = sb.packed.accumulate_along_rays(wp, ri, None, n_rays=R)
    a_t = a[tail].double()
    T = torch.cumprod(torch.cat([torch.ones(40, 1, dtype=torch.float64), 1 - a_t[:, :-1]], 1), 1)
    w_ref = a_t * T
    _assert_elem(wp.reshape(R, S)[tail], w_ref, w_ref, 4 * U, "packed weights, last rays")
    _assert_elem(acc[tail, 0], w_ref.sum(1), w_ref.sum(1), 8 * U, "packed accumulate, last rays")
