"""Differentiable forms of the weights / compositing operators (training path).

The reference trains through ATen autograd over rays.py:131-230 and renderers.py:42-295; here every op keeps its forward
kernel and gets an explicit backward kernel (csrc/render_backward.cu: sdfb200_render_backward, sdfb200_weights_backward).
Used automatically by rays.py / renderers.py when an input requires grad.  Each dense compositing op has one launch function here
(launch_*): it allocates the outputs, builds the RenderOut and launches the kernel.  The no-grad (rendering) path calls it directly, with
its in-kernel clamp / median and only the outputs it asks for; the Function's forward calls it and keeps what its backward needs.
"""
import torch

from . import _lib


def needs_grad(*ts) -> bool:
    return torch.is_grad_enabled() and any(t is not None and torch.is_tensor(t) and t.requires_grad for t in ts)


def training_step(module, params) -> bool:
    """True when autograd is recording a training step of `module` through `params`: the fields then take their differentiable path."""
    return torch.is_grad_enabled() and module.training and any(p.requires_grad for p in params)


def launch_weights_from_alphas(a, with_transmittance: bool):
    """alphas [R,S] (fp32, contiguous) -> weights [R,S], transmittance [R,S+1] | None (sdfb200_weights_from_alphas)."""
    R, S = a.shape
    w = torch.empty_like(a)
    T = a.new_empty(R, S + 1) if with_transmittance else None
    _lib.check(_lib.load().sdfb200_weights_from_alphas(_lib.ptr(a), R, S, _lib.ptr(w), _lib.ptr(T), _lib.stream_ptr()), "sdfb200_weights_from_alphas")
    return w, T


def launch_weights_from_density(d, bins, with_transmittance: bool):
    """densities [R,S] (fp32, contiguous), euclidean bins [R,S+1] -> weights [R,S], transmittance [R,S] | None
    (sdfb200_weights_from_density)."""
    R, S = d.shape
    w = torch.empty_like(d)
    T = torch.empty_like(d) if with_transmittance else None
    _lib.check(_lib.load().sdfb200_weights_from_density(_lib.ptr(d), _lib.ptr(bins), R, S, _lib.ptr(w), _lib.ptr(T), _lib.stream_ptr()),
               "sdfb200_weights_from_density")
    return w, T


def launch_render(w, rgb, normals, bins, bg, bg_mode, clamp01=False, median=False, want_acc=True):
    """weights [R,S] (+ rgb, normals [R,S,3], bins [R,S+1], all fp32 contiguous or None) -> rgb [R,3], depth [R], normal [R,3],
    accumulation [R], steps_minmax [2] (sdfb200_render).  An output whose input is None (accumulation: want_acc False) is not computed
    and comes back as None; the depth is the unclipped one."""
    R, S = w.shape
    dev = w.device
    o_rgb = w.new_empty(R, 3) if rgb is not None else None
    o_nrm = w.new_empty(R, 3) if normals is not None else None
    o_depth = w.new_empty(R) if bins is not None else None
    o_acc = w.new_empty(R) if want_acc else None
    mm = _lib.steps_minmax_seed(dev).clone() if bins is not None else None
    out = _lib.render_out(o_rgb, o_depth, o_nrm, o_acc, mm)
    _lib.check(_lib.load().sdfb200_render(_lib.ptr(w), _lib.ptr(rgb), _lib.ptr(normals), _lib.ptr(bins), _lib.ptr(bg), bg_mode, int(clamp01),
                                          int(median), R, S, out, _lib.stream_ptr()), "sdfb200_render")
    return o_rgb, o_depth, o_nrm, o_acc, mm


def launch_render_alphas(a, rgb, normals, bins, bg, bg_mode, clamp01=False, want_weights=True):
    """alphas [R,S] (+ rgb, normals [R,S,3], bins [R,S+1], fp32 contiguous) -> weights [R,S] | None, rgb [R,3], unclipped depth [R],
    normal [R,3], accumulation [R], bg_transmittance [R], steps_minmax [2] in one launch (sdfb200_render_alphas)."""
    R, S = a.shape
    dev = a.device
    w = a.new_empty(R, S) if want_weights else None
    o_rgb, o_depth, o_nrm = a.new_empty(R, 3), a.new_empty(R), a.new_empty(R, 3)
    o_acc, o_bgT = a.new_empty(R), a.new_empty(R)
    mm = _lib.steps_minmax_seed(dev).clone()
    out = _lib.render_out(o_rgb, o_depth, o_nrm, o_acc, mm)
    _lib.check(_lib.load().sdfb200_render_alphas(_lib.ptr(a), _lib.ptr(rgb), _lib.ptr(normals), _lib.ptr(bins), _lib.ptr(bg), bg_mode, int(clamp01), R, S,
                                                 _lib.ptr(w), _lib.ptr(o_bgT), out, _lib.stream_ptr()), "sdfb200_render_alphas")
    return w, o_rgb, o_depth, o_nrm, o_acc, o_bgT, mm


def launch_render_packed(w, rgb, normals, starts, ends, ray_indices, R, bg, bg_mode, clamp01=False, want_acc=True):
    """packed samples: weights [N] (+ rgb, normals [N,3], starts, ends [N], fp32 contiguous or None), int64 ray_indices [N] in any order ->
    rgb [R,3], unclipped depth [R], normal [R,3], accumulation [R], steps_minmax [2] (sdfb200_render_packed).  An output whose input is
    None (accumulation: want_acc False) is not computed and comes back as None."""
    N, dev = w.shape[0], w.device
    o_rgb = w.new_empty(R, 3) if rgb is not None else None
    o_nrm = w.new_empty(R, 3) if normals is not None else None
    o_depth = w.new_empty(R) if starts is not None else None
    o_acc = w.new_empty(R) if want_acc else None
    mm = _lib.steps_minmax_seed(dev).clone() if starts is not None else None
    out = _lib.render_out(o_rgb, o_depth, o_nrm, o_acc, mm)
    ws = w.new_empty(max(R, 1) * 8)
    _lib.check(_lib.load().sdfb200_render_packed(_lib.ptr(w), _lib.ptr(rgb), _lib.ptr(normals), _lib.ptr(starts), _lib.ptr(ends), _lib.ptr(ray_indices),
                                                 N, R, _lib.ptr(bg), bg_mode, int(clamp01), out, _lib.ptr(ws), ws.numel() * 4, _lib.stream_ptr()),
               "sdfb200_render_packed")
    return o_rgb, o_depth, o_nrm, o_acc, mm


def _or_zeros(t, like, *shape):
    """an output the launch did not compute (its input was None): zeros, so that the Function returns a tensor in every place"""
    return t if t is not None else like.new_zeros(shape)


class WeightsFromAlphasFn(torch.autograd.Function):
    """alphas [R,S] -> weights [R,S], transmittance [R,S+1] (rays.py:194-230).  Gradients flow back through the weights and
    through every transmittance column (bg_transmittance = transmittance[:, -1], models/neus.py:101)."""

    @staticmethod
    def forward(ctx, alphas):
        a = _lib.f32c(alphas)
        w, T = launch_weights_from_alphas(a, True)
        ctx.save_for_backward(a)
        return w, T

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_w, g_T):
        lib = _lib.load()
        (a,) = ctx.saved_tensors
        R, S = a.shape
        g_w = _lib.f32c(g_w) if g_w is not None else torch.zeros_like(a)
        g_T = _lib.f32c(g_T) if g_T is not None else None
        g_a = torch.empty_like(a)
        _lib.check(lib.sdfb200_weights_backward(_lib.ptr(a), None, 0, R, S, _lib.ptr(g_w), _lib.ptr(g_T), S + 1, _lib.ptr(g_a), _lib.stream_ptr()),
                   "sdfb200_weights_backward")
        return g_a


class WeightsFromDensityFn(torch.autograd.Function):
    """densities [R,S], euclidean bins [R,S+1] -> weights [R,S], transmittance [R,S] (rays.py:131-192).  Gradients flow to the
    densities through the weights AND the transmittance (VolSDF composites the background model with transmittance[:, -1],
    models/volsdf.py:67-68 + base_surface_model.py:329)."""

    @staticmethod
    def forward(ctx, density, bins):
        d = _lib.f32c(density)
        w, T = launch_weights_from_density(d, bins, True)
        ctx.save_for_backward(d, bins)
        return w, T

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_w, g_T):
        lib = _lib.load()
        d, bins = ctx.saved_tensors
        R, S = d.shape
        g_w = _lib.f32c(g_w) if g_w is not None else torch.zeros_like(d)
        g_T = _lib.f32c(g_T) if g_T is not None else None
        g_d = torch.empty_like(d)
        _lib.check(lib.sdfb200_weights_backward(_lib.ptr(d), _lib.ptr(bins), 1, R, S, _lib.ptr(g_w), _lib.ptr(g_T), S, _lib.ptr(g_d), _lib.stream_ptr()),
                   "sdfb200_weights_backward")
        return g_d, None


def _render_backward(ctx_t, bg_mode, grads, g_weights_in, want_rgb_s, want_nrm_s):
    """shared by RenderFn / RenderAlphasFn: per-ray output gradients -> (g_weights, g_rgb_samples, g_normal_samples)."""
    lib = _lib.load()
    w, rgb, nrm, bins, bg, acc, depth = ctx_t
    R, S = w.shape
    g_rgb, g_depth, g_nrm, g_acc = grads
    g_rgb = _lib.f32c(g_rgb) if (g_rgb is not None and rgb is not None) else None
    g_depth = _lib.f32c(g_depth) if (g_depth is not None and bins is not None) else None
    g_nrm = _lib.f32c(g_nrm) if (g_nrm is not None and nrm is not None) else None
    g_acc = _lib.f32c(g_acc) if g_acc is not None else None
    g_w = torch.empty_like(w)
    g_rgb_s = torch.empty(R, S, 3, device=w.device, dtype=torch.float32) if (want_rgb_s and rgb is not None) else None
    g_nrm_s = torch.empty(R, S, 3, device=w.device, dtype=torch.float32) if (want_nrm_s and nrm is not None) else None
    _lib.check(lib.sdfb200_render_backward(_lib.ptr(w), _lib.ptr(rgb), _lib.ptr(nrm), _lib.ptr(bins), _lib.ptr(bg), bg_mode, R, S, _lib.ptr(acc),
                                           _lib.ptr(depth), _lib.ptr(g_rgb), _lib.ptr(g_depth), _lib.ptr(g_nrm), _lib.ptr(g_acc),
                                           _lib.ptr(g_weights_in), _lib.ptr(g_w), _lib.ptr(g_rgb_s), _lib.ptr(g_nrm_s), _lib.stream_ptr()),
               "sdfb200_render_backward")
    return g_w, g_rgb_s, g_nrm_s


class RenderFn(torch.autograd.Function):
    """weights [R,S] (+ rgb, normals [R,S,3], bins [R,S+1]) -> rgb [R,3], UNCLIPPED expected depth [R], normal [R,3],
    accumulation [R], steps_minmax [2] (sdfb200_render).  Absent inputs are passed as None and yield zero-filled outputs."""

    @staticmethod
    def forward(ctx, weights, rgb, normals, bins, bg, bg_mode):
        w = _lib.f32c(weights)
        R = w.shape[0]
        rgb = _lib.f32c(rgb) if rgb is not None else None
        normals = _lib.f32c(normals) if normals is not None else None
        o_rgb, o_depth, o_nrm, o_acc, mm = launch_render(w, rgb, normals, bins, bg, bg_mode)
        o_rgb, o_depth, o_nrm = _or_zeros(o_rgb, w, R, 3), _or_zeros(o_depth, w, R), _or_zeros(o_nrm, w, R, 3)
        mm = mm if mm is not None else _lib.steps_minmax_seed(w.device).clone()
        ctx.tensors = (w, rgb, normals, bins, bg, o_acc, o_depth)
        ctx.bg_mode = bg_mode
        ctx.mark_non_differentiable(mm)
        return o_rgb, o_depth, o_nrm, o_acc, mm

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_rgb, g_depth, g_nrm, g_acc, _g_mm):
        g_w, g_rgb_s, g_nrm_s = _render_backward(ctx.tensors, ctx.bg_mode, (g_rgb, g_depth, g_nrm, g_acc), None,
                                                 ctx.needs_input_grad[1], ctx.needs_input_grad[2])
        return g_w, g_rgb_s, g_nrm_s, None, None, None


class RenderAlphasFn(torch.autograd.Function):
    """alphas [R,S] -> weights, rgb, UNCLIPPED depth, normal, accumulation, bg_transmittance, steps_minmax in one forward launch
    (sdfb200_render_alphas); backward = sdfb200_render_backward -> sdfb200_weights_backward."""

    @staticmethod
    def forward(ctx, alphas, rgb, normals, bins, bg, bg_mode):
        a = _lib.f32c(alphas)
        rgb, normals = _lib.f32c(rgb), _lib.f32c(normals)
        w, o_rgb, o_depth, o_nrm, o_acc, o_bgT, mm = launch_render_alphas(a, rgb, normals, bins, bg, bg_mode)
        ctx.tensors = (w, rgb, normals, bins, bg, o_acc, o_depth)
        ctx.alphas = a
        ctx.bg_mode = bg_mode
        ctx.mark_non_differentiable(mm)
        return w, o_rgb, o_depth, o_nrm, o_acc, o_bgT, mm

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_w_in, g_rgb, g_depth, g_nrm, g_acc, g_bgT, _g_mm):
        lib = _lib.load()
        a = ctx.alphas
        R, S = a.shape
        g_w_in = _lib.f32c(g_w_in) if g_w_in is not None else None
        g_w, g_rgb_s, g_nrm_s = _render_backward(ctx.tensors, ctx.bg_mode, (g_rgb, g_depth, g_nrm, g_acc), g_w_in,
                                                 ctx.needs_input_grad[1], ctx.needs_input_grad[2])
        g_a = None
        if ctx.needs_input_grad[0]:
            g_a = torch.empty_like(a)
            g_last = _lib.f32c(g_bgT) if g_bgT is not None else None
            _lib.check(lib.sdfb200_weights_backward(_lib.ptr(a), None, 0, R, S, _lib.ptr(g_w), _lib.ptr(g_last), 1, _lib.ptr(g_a), _lib.stream_ptr()),
                       "sdfb200_weights_backward")
        return g_a, g_rgb_s, g_nrm_s, None, None, None


class PackedRenderFn(torch.autograd.Function):
    """packed samples: weights [N] (+ rgb, normals [N,3], starts, ends [N]), ray_indices [N] in any order -> rgb [R,3], UNCLIPPED expected
    depth [R], normal [R,3], accumulation [R], steps_minmax [2] (sdfb200_render_packed; backward sdfb200_render_packed_backward).  What
    nerfacc.accumulate_along_rays gives the reference's renderers (renderers.py:78-79, 194, 251-252), differentiable like it.  Absent inputs
    are passed as None and yield zero-filled outputs."""

    @staticmethod
    def forward(ctx, weights, rgb, normals, starts, ends, ray_indices, num_rays, bg, bg_mode):
        w = _lib.f32c(weights)
        R = int(num_rays)
        rgb = _lib.f32c(rgb) if rgb is not None else None
        normals = _lib.f32c(normals) if normals is not None else None
        st, en = (_lib.f32c(starts), _lib.f32c(ends)) if starts is not None else (None, None)
        o_rgb, o_depth, o_nrm, o_acc, mm = launch_render_packed(w, rgb, normals, st, en, ray_indices, R, bg, bg_mode)
        o_rgb, o_depth, o_nrm = _or_zeros(o_rgb, w, R, 3), _or_zeros(o_depth, w, R), _or_zeros(o_nrm, w, R, 3)
        mm = mm if mm is not None else _lib.steps_minmax_seed(w.device).clone()
        ctx.tensors = (w, rgb, normals, st, en, ray_indices, bg, o_acc, o_depth)
        ctx.bg_mode = bg_mode
        ctx.mark_non_differentiable(mm)
        return o_rgb, o_depth, o_nrm, o_acc, mm

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_rgb, g_depth, g_nrm, g_acc, _g_mm):
        lib = _lib.load()
        w, rgb, nrm, st, en, ri, bg, acc, depth = ctx.tensors
        N, R = w.shape[0], acc.shape[0]
        g_rgb = _lib.f32c(g_rgb) if (g_rgb is not None and rgb is not None) else None
        g_depth = _lib.f32c(g_depth) if (g_depth is not None and st is not None) else None
        g_nrm = _lib.f32c(g_nrm) if (g_nrm is not None and nrm is not None) else None
        g_acc = _lib.f32c(g_acc) if g_acc is not None else None
        g_w = torch.empty_like(w)
        g_rgb_s = torch.empty(N, 3, device=w.device) if (ctx.needs_input_grad[1] and rgb is not None) else None
        g_nrm_s = torch.empty(N, 3, device=w.device) if (ctx.needs_input_grad[2] and nrm is not None) else None
        want_steps = st is not None and (ctx.needs_input_grad[3] or ctx.needs_input_grad[4])
        g_steps = torch.empty(N, device=w.device) if want_steps else None
        _lib.check(lib.sdfb200_render_packed_backward(_lib.ptr(w), _lib.ptr(rgb), _lib.ptr(nrm), _lib.ptr(st), _lib.ptr(en), _lib.ptr(ri), N, R,
                                                      _lib.ptr(bg), ctx.bg_mode, _lib.ptr(acc), _lib.ptr(depth), _lib.ptr(g_rgb), _lib.ptr(g_depth),
                                                      _lib.ptr(g_nrm), _lib.ptr(g_acc), _lib.ptr(g_w), _lib.ptr(g_rgb_s), _lib.ptr(g_nrm_s),
                                                      _lib.ptr(g_steps), _lib.stream_ptr()), "sdfb200_render_packed_backward")
        g_half = g_steps * 0.5 if want_steps else None          # step = (starts + ends) / 2
        return g_w, g_rgb_s, g_nrm_s, g_half, g_half, None, None, None, None


class PackedWeightsFn(torch.autograd.Function):
    """alphas [N] of segmented packed samples (ray r = [offsets[r], offsets[r+1])) -> weights [N] = alpha * exclusive prod(1 - alpha)
    (nerfacc 0.3.5 render_weight_from_alpha; sdfb200_packed_weights / sdfb200_packed_weights_backward)."""

    @staticmethod
    def forward(ctx, alphas, offsets):
        lib = _lib.load()
        a = _lib.f32c(alphas)
        w = torch.empty_like(a)
        R = offsets.numel() - 1
        _lib.check(lib.sdfb200_packed_weights(_lib.ptr(a), _lib.ptr(offsets), R, _lib.ptr(w), _lib.stream_ptr()), "sdfb200_packed_weights")
        ctx.save_for_backward(a, offsets)
        return w

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_w):
        lib = _lib.load()
        a, offsets = ctx.saved_tensors
        g_a = torch.zeros_like(a)
        _lib.check(lib.sdfb200_packed_weights_backward(_lib.ptr(a), _lib.ptr(offsets), offsets.numel() - 1, _lib.ptr(_lib.f32c(g_w)), _lib.ptr(g_a),
                                                       _lib.stream_ptr()), "sdfb200_packed_weights_backward")
        return g_a, None


class PackedAccumulateFn(torch.autograd.Function):
    """weights [N], values [N,C] | None -> [R,C] per-segment sums of weights * values (nerfacc 0.3.5 accumulate_along_rays;
    sdfb200_packed_accumulate / sdfb200_packed_accumulate_backward)."""

    @staticmethod
    def forward(ctx, weights, values, offsets, ray_indices):
        lib = _lib.load()
        w = _lib.f32c(weights)
        v = _lib.f32c(values) if values is not None else None
        C = v.shape[1] if v is not None else 1
        R = offsets.numel() - 1
        out = torch.empty(R, C, device=w.device, dtype=torch.float32)
        _lib.check(lib.sdfb200_packed_accumulate(_lib.ptr(w), _lib.ptr(v), C, _lib.ptr(offsets), R, _lib.ptr(out), _lib.stream_ptr()),
                   "sdfb200_packed_accumulate")
        ctx.save_for_backward(w, v, ray_indices)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_out):
        lib = _lib.load()
        w, v, ray_indices = ctx.saved_tensors
        C = v.shape[1] if v is not None else 1
        g_w = torch.empty_like(w) if ctx.needs_input_grad[0] else None
        g_v = torch.empty_like(v) if (v is not None and ctx.needs_input_grad[1]) else None
        _lib.check(lib.sdfb200_packed_accumulate_backward(_lib.ptr(w), _lib.ptr(v), C, _lib.ptr(ray_indices), w.shape[0], _lib.ptr(_lib.f32c(g_out)),
                                                          _lib.ptr(g_w), _lib.ptr(g_v), _lib.stream_ptr()), "sdfb200_packed_accumulate_backward")
        return g_w, g_v, None, None


class InterlevelLossFn(torch.autograd.Function):
    """One proposal level of the interlevel loss (losses.py:38-172): proposal weights [R,Sp] -> the mean over all elements (0-dim).
    form = _lib.INTERLEVEL_OUTER or _lib.INTERLEVEL_ZIP (blur_radius is read by the latter only).  The forward kernel writes
    d (a ray's sum) / d proposal weights next to the loss, so the backward is one scale by grad / count.  Only the proposal weights
    are differentiable: the bin edges and the fine weights are constants here, as they are in the reference."""

    @staticmethod
    def forward(ctx, proposal_weights, proposal_bins, fine_bins, fine_weights, form, blur_radius):
        lib = _lib.load()
        wp = _lib.f32c(proposal_weights)
        R, sp = wp.shape
        sf = fine_weights.shape[1]
        per_ray = torch.empty(R, device=wp.device, dtype=torch.float32)
        loss = torch.empty((), device=wp.device, dtype=torch.float32)
        grad = torch.empty_like(wp) if ctx.needs_input_grad[0] else None
        _lib.check(lib.sdfb200_interlevel_loss(_lib.ptr(fine_bins), _lib.ptr(fine_weights), sf, _lib.ptr(proposal_bins), _lib.ptr(wp), sp, R, form,
                                               float(blur_radius), _lib.ptr(per_ray), _lib.ptr(loss), _lib.ptr(grad), _lib.stream_ptr()),
                   "sdfb200_interlevel_loss")
        ctx.save_for_backward(grad)
        ctx.count = R * (sp if form == _lib.INTERLEVEL_ZIP else sf)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_loss):
        (grad,) = ctx.saved_tensors
        return grad * (g_loss / ctx.count), None, None, None, None, None
