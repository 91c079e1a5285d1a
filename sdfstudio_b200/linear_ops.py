"""Dense-layer GEMMs of the TRAINING path on the tensor-core (wgmma) kernels (sdfb200_gemm_nt / _nn / _tn), as autograd Functions.

The reference trains through ATen autograd over ``nn.Linear`` (nerfstudio/fields/sdf_field.py:400-409 via engine/trainer.py:319-323),
including the double backward of the eikonal term (``torch.autograd.grad(..., create_graph=True)``, sdf_field.py:646-655).  The three
primitives below are closed under differentiation -- the backward of each is made of the other two -- so first- and second-order
autograd run entirely on this package's kernels:

    nt(x [P,Kp], W [N,K])        -> x W^T   [P,Np]      d/dx = nn(g, W)        d/dW = tn(g, x)
    nn(g [P,Np], W [N,K])        -> g W     [P,Kp]      d/dg = nt(gy, W)       d/dW = tn(g, gy)
    tn(a [P,Np], b [P,Kp], N, K) -> a^T b   [N,K]       d/da = nt(b, gC)       d/db = nn(a, gC)

Activations travel with their feature dimension padded to a multiple of 16 (``pad16``): padding columns of outputs are zero, padding
columns of inputs are ignored by the kernels.  fp32 in / out, bf16x3 (parity grade) or bf16 arithmetic.
"""
import torch

from . import _lib

_ws = {}


def pad16(n: int) -> int:
    return (n + 15) // 16 * 16


def _workspace(dev):
    w = _ws.get(dev)
    if w is None:
        w = torch.empty(_lib.load().sdfb200_gemm_workspace_bytes(), dtype=torch.uint8, device=dev)
        _ws[dev] = w
    return w


def _prec(precision: str) -> int:
    return _lib.PRECISION["bf16" if precision == "bf16" else "bf16x3"]


def _c(t):
    t = t if t.dtype == torch.float32 else t.float()
    return t if t.is_contiguous() else t.contiguous()


def pad_cols(x: torch.Tensor) -> torch.Tensor:
    """[P, K] -> [P, pad16(K)] (zero padded copy; no-op when already aligned)."""
    k = x.shape[-1]
    return x if k % 16 == 0 else torch.nn.functional.pad(x, (0, pad16(k) - k))


def _raw_nt(x, W, bias, epilogue, precision):
    lib = _lib.load()
    P, N, K = x.shape[0], W.shape[0], W.shape[1]
    assert x.shape[1] == pad16(K), (x.shape, W.shape)
    y = torch.empty(P, pad16(N), device=x.device, dtype=torch.float32)
    ws = _workspace(x.device)
    _lib.check(lib.sdfb200_gemm_nt(_prec(precision), _lib.ptr(x), x.shape[1], _lib.ptr(W), W.shape[1], N, K, _lib.ptr(bias), epilogue, _lib.ptr(y), y.shape[1], P,
                                   _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "sdfb200_gemm_nt")
    return y


def _raw_nn(g, W, precision):
    lib = _lib.load()
    P, N, K = g.shape[0], W.shape[0], W.shape[1]
    assert g.shape[1] == pad16(N), (g.shape, W.shape)
    y = torch.empty(P, pad16(K), device=g.device, dtype=torch.float32)
    ws = _workspace(g.device)
    _lib.check(lib.sdfb200_gemm_nn(_prec(precision), _lib.ptr(g), g.shape[1], _lib.ptr(W), W.shape[1], N, K, _lib.ptr(y), y.shape[1], P, _lib.ptr(ws), ws.numel(),
                                   _lib.stream_ptr()), "sdfb200_gemm_nn")
    return y


def _raw_tn(a, b, N, K, precision):
    lib = _lib.load()
    P = a.shape[0]
    assert a.shape[1] >= N and b.shape[1] >= K and b.shape[0] == P
    c = torch.empty(N, K, device=a.device, dtype=torch.float32)
    ws = _workspace(a.device)
    _lib.check(lib.sdfb200_gemm_tn(_prec(precision), _lib.ptr(a), a.shape[1], _lib.ptr(b), b.shape[1], _lib.ptr(c), K, P, N, K, _lib.ptr(ws), ws.numel(),
                                   _lib.stream_ptr()), "sdfb200_gemm_tn")
    return c


class _NT(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, W, precision):
        x, W = _c(x), _c(W)
        ctx.save_for_backward(x, W)
        ctx.precision = precision
        return _raw_nt(x, W, None, 0, precision)

    @staticmethod
    def backward(ctx, gy):
        x, W = ctx.saved_tensors
        gx = _NN.apply(gy, W, ctx.precision) if ctx.needs_input_grad[0] else None
        gW = _TN.apply(gy, x, W.shape[0], W.shape[1], ctx.precision) if ctx.needs_input_grad[1] else None
        return gx, gW, None


class _NN(torch.autograd.Function):
    @staticmethod
    def forward(ctx, g, W, precision):
        g, W = _c(g), _c(W)
        ctx.save_for_backward(g, W)
        ctx.precision = precision
        return _raw_nn(g, W, precision)

    @staticmethod
    def backward(ctx, gy):
        g, W = ctx.saved_tensors
        gg = _NT.apply(gy, W, ctx.precision) if ctx.needs_input_grad[0] else None
        gW = _TN.apply(g, gy, W.shape[0], W.shape[1], ctx.precision) if ctx.needs_input_grad[1] else None
        return gg, gW, None


class _TN(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b, N, K, precision):
        a, b = _c(a), _c(b)
        ctx.save_for_backward(a, b)
        ctx.precision = precision
        return _raw_tn(a, b, N, K, precision)

    @staticmethod
    def backward(ctx, gC):
        a, b = ctx.saved_tensors
        gC = _c(gC)
        ga = _NT.apply(b, gC, ctx.precision) if ctx.needs_input_grad[0] else None      # b [P,Kp] gC[N,K]^T -> [P,Np]
        gb = _NN.apply(a, gC, ctx.precision) if ctx.needs_input_grad[1] else None      # a [P,Np] gC[N,K]   -> [P,Kp]
        return ga, gb, None, None, None


def gemm_nt(x, W, precision="bf16x3"):
    return _NT.apply(x, W, precision)


def gemm_nn(g, W, precision="bf16x3"):
    return _NN.apply(g, W, precision)


def gemm_tn(a, b, N, K, precision="bf16x3"):
    return _TN.apply(a, b, N, K, precision)


class _LinearAct(torch.autograd.Function):
    """y = act(x W^T + b) with bias and activation fused into the GEMM epilogue (act: 0 none, 1 softplus(beta=100), 2 relu).
    backward: gz = gy * act'(.) expressed through the OUTPUT (softplus' = 1 - exp(-100 y), relu' = [y > 0]) with differentiable torch
    ops, then the nn / tn GEMMs -- so the op is differentiable to any order."""

    @staticmethod
    def forward(ctx, x, W, b, act, precision):
        x, W = _c(x), _c(W)
        n = W.shape[0]
        bp = _c(b if n % 16 == 0 else torch.nn.functional.pad(b, (0, pad16(n) - n)))
        y = _raw_nt(x, W, bp, act, precision)
        ctx.save_for_backward(x, W, y)
        ctx.act, ctx.precision = act, precision
        return y

    @staticmethod
    def backward(ctx, gy):
        x, W, y = ctx.saved_tensors
        n = W.shape[0]
        if ctx.act == 1:
            gz = gy * (1.0 - torch.exp(-100.0 * y))
        elif ctx.act == 2:
            gz = gy * (y > 0).to(gy.dtype)
        else:
            gz = gy
        if n % 16 != 0:                       # padding columns carry act(0) != 0 for softplus: they are not part of the function
            mask = torch.zeros(gz.shape[1], device=gz.device, dtype=gz.dtype)
            mask[:n] = 1.0
            gz = gz * mask
        gx = _NN.apply(gz, W, ctx.precision) if ctx.needs_input_grad[0] else None
        gW = _TN.apply(gz, x, n, W.shape[1], ctx.precision) if ctx.needs_input_grad[1] else None
        gb = gz.sum(0)[:n] if ctx.needs_input_grad[2] else None
        return gx, gW, gb, None, None


def linear(x, weight, bias, act: int = 0, precision="bf16x3"):
    """``act(F.linear(x, weight, bias))`` on the tensor-core GEMMs: x [P, pad16(K)] (padding columns ignored), weight [N, K], bias [N]
    -> [P, pad16(N)].  For act = 0 / relu the padding columns of the result are zero; for softplus they hold softplus(0) and must be
    sliced off or ignored by the consumer (the next layer's GEMM ignores them).  Differentiable to any order."""
    return _LinearAct.apply(x, weight, bias, act, precision)
