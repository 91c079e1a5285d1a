"""-m gpu: the three training GEMMs (sdfb200_gemm_nt / _nn / _tn) against fp64, element by element, at every chunk, tile and slice
boundary they cross, through the C ABI (strides, padding and canaries under the test's control) and through linear_ops' autograd.

Oracles (fp64 on the GPU).  Let x0 = bf16(x) and x1 = bf16(x - x0) (the kernels' split2 / k_tc_pack; x - x0 is exact in fp32), the same
for w.  bf16x3 computes S = sum(x0 w0 + x1 w0 + x0 w1), bf16 computes S = sum(x0 w0).  Every product is exact in fp32 (8 x 8 significant
bits), so against S the kernel's only error is the accumulation; T = the same sum over |terms| bounds every partial sum.
  * The wgmma accumulator is not documented to round to nearest (tc_wgrad.cu reports it does not), so each addition inside a wgmma
    chain is taken to truncate: relative error <= ut = 2^-23.  A chain of n products then errs by at most n ut T (recursive summation).
  * nt / nn: one chain per 256-wide K chunk, n = planes_terms * min(K, 256) (3 terms for bf16x3, 1 for bf16; zero padding adds exact
    zeros), and the partial sums round-trip through Y in fp32 round-to-nearest (u = 2^-24 each):  E = (n ut + (chunks - 1) u) T.
  * tn: one chain per slice of kWgSlice stages of kWgPts points (n = terms * 1024), each slice added into the CTA's workspace slot in
    fp32 (one u per spill), then k_wgrad_reduce sums the G slots in a fixed order (G u):  E = (n ut + (spills + G) u) T.
  * The epilogue: bias adds u (|S| + |b|); ReLU is 1-Lipschitz; softplus(beta = 100) through fast_ex2 / fast_lg2 (relative error
    <= 2^-22 each, PTX ISA) is 1-Lipschitz in z plus at most 2^-20 |h| + 2^-24 of its own (for z < -0.87 e flushes to 0 and h = 0
    where the true h < 1e-37).  dsoftplus100_fast_from_h = 1 - ex2(-144.27 h) has an ABSOLUTE error <= 2^-21 (ex2, the rounding of 1 - e
    and of the product): for h < ~1e-9 the derivative 100 h is below that and has no relative precision left, by design.
  E is 2^-23 * 768 = 9e-5 of T at most for nt / nn and 3.7e-4 for tn: far below the 2^-9 .. 2^-8 of T that a dropped or mis-paired
  plane, a K block counted twice or left out, or a lost slice costs.  The value pattern "lo1" (values in [1, 2) whose low planes are
  all positive, 0.3 .. 0.45 of 2^-8) makes a dropped low plane cost ~1e-3 T, 10x the largest E.  Where one fp32 rounding (the bias
  add) dominates, it may come within a few per cent of its u |result| bound (measured worst ratio 0.99).
True fp64 product: bf16x3 is also held to X W^T in fp64 with the split's own error added, |x w - (x0 w0 + x1 w0 + x0 w1)| <=
3.1 * 2^-16 |x||w| (|x - x0| <= 2^-8 |x|, |x - x0 - x1| <= 2^-16 |x|).

Shapes (the constants are read from the sources: kKBL, the 256-wide chunks, n64 blocks, the 128-row tile, kWgPts, kWgRowsA / B,
kWgSlice): every N and K in DIMS, the layer shapes the package runs, P for nt / nn in P_LINEAR, and for tn P = 0 (C exactly 0), fewer
stages than CTAs, as many and one more, 32 * 32 * CTAs points and that +-1 point and +-1 stage, and two slices + 1, with CTAs =
min(multiProcessorCount, 132) (persistent_ctas()).  One call per primitive past 2^31 elements (P = 2^23 + 129 at 256 x 256) checks
sampled rows; it needs about 17 GB of device memory.  Inputs carry NaN in every column past the real width and every row past P (read
canaries), outputs a sentinel in every spare row and column (write canaries).

Mutants, each applied alone to a scratch build, each killed by the test named:
  accumulate forced to 0 ........................ test_nt_table / test_nn_table (K > 256)
  final_chunk forced to 1 ....................... test_nt_table (bias over three K chunks)
  lo plane of k_tc_linear's A staging zeroed .... test_nt_table / test_nn_table (pattern lo1, bf16x3)
  `w - hi` -> 0 in k_tc_pack .................... test_nt_table / test_nn_table (pattern lo1, bf16x3)
  `k + 8 <= a.Kvalid` -> `<= a.Kc32` ............ test_nt_table (NaN canaries; every X row carries >= 32 spare columns)
  spill stores instead of adding ................ test_tn_table (P past one slice)
  k_wgrad_reduce sums G - 1 slots ............... test_tn_table
  aux_cols compared without a.n0 ................ test_dsoftplus_epilogue_across_n_chunks

Run time on one H100 80GB HBM3 (700 W): about 35 s.  The measured error / bound ratios are in DESIGN §4.
"""
import ctypes
import math
import os
import re

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "sdfstudio_b200", "csrc")


def _const(fname, name):
    src = open(os.path.join(CSRC, fname)).read()
    return int(re.search(rf"constexpr\s+\w+\s+{name}\s*=\s*(\d+)", src).group(1))


KBL = _const("tc_linear.cu", "kKBL")              # K per streamed weight block
WG_PTS = _const("tc_wgrad.cu", "kWgPts")          # points per tn stage
WG_ROWS_A = _const("tc_wgrad.cu", "kWgRowsA")     # tn N chunk
WG_ROWS_B = _const("tc_wgrad.cu", "kWgRowsB")     # tn K chunk
WG_SLICE = _const("tc_wgrad.cu", "kWgSlice")      # stages per slice
CHUNK = 256                                       # tc_gemm_ex's N / K chunk (and the wgmma n256 / K-tile limit)
TILE = 128                                        # rows per k_tc_linear CTA
assert (KBL, WG_PTS, WG_ROWS_A, WG_ROWS_B, WG_SLICE) == (32, 32, 128, CHUNK, 32)

U, UT = 2.0**-24, 2.0**-23
SPLIT = 3.1 * 2.0**-16
SENT = -1.2345e30
TERMS = {"bf16x3": 3, "bf16": 1}
_RATIOS = {}


def pad16(n):
    return (n + 15) // 16 * 16


def _ctas():
    return min(torch.cuda.get_device_properties(0).multi_processor_count, 132)


def _lib():
    from sdfstudio_b200 import _lib as L

    return L


def _ws():
    from sdfstudio_b200 import linear_ops

    return linear_ops._workspace(torch.device("cuda", torch.cuda.current_device()))


def _record(key, err, bound):
    """error / bound, kept per (primitive, precision, oracle); the test fails on > 1"""
    err, bound = err.detach(), bound.detach()
    r = float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0
    m = err > bound
    if bool(m.any()):
        i = int(m.flatten().nonzero()[0])
        raise AssertionError(f"{key}: element {i} err {float(err.flatten()[i]):.3e} > bound {float(bound.flatten()[i]):.3e} ({int(m.sum())} elements)")
    _RATIOS[key] = max(_RATIOS.get(key, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(_RATIOS):
        print(f"max err/bound {k}: {_RATIOS[k]:.3f}")


# ---------------------------------------------------------------------------------------------------------------
# buffers with canaries
# ---------------------------------------------------------------------------------------------------------------
class Buf:
    """[1 + rows + 2, ld] fp32, one spare row before and two after; `v` is the [rows, cols] region the call sees (pointer p)."""

    def __init__(self, rows, cols, ld, fill):
        self.b = torch.full((rows + 3, ld), fill, device="cuda")
        self.rows, self.cols, self.ld = rows, cols, ld
        self.v = self.b[1:1 + rows, :cols]
        self.p = self.b[1].data_ptr()

    def outside(self, cols=None):
        """everything outside rows [0, rows) x columns [0, cols)"""
        m = torch.ones_like(self.b, dtype=torch.bool)
        m[1:1 + self.rows, :self.cols if cols is None else cols] = False
        return self.b[m]


def _values(pattern, rows, cols, g, rowscale=True):
    if pattern == "randn":
        x = torch.randn(rows, cols, generator=g)
    elif pattern == "nonneg":
        x = torch.rand(rows, cols, generator=g)
    elif pattern == "scaled":                       # rows (or, for tn, columns) 1e6, 1, 1e-6
        x = torch.randn(rows, cols, generator=g)
        s = torch.tensor([1e6, 1.0, 1e-6]).repeat(rows // 3 + 1)[:rows, None] if rowscale else \
            torch.tensor([1e6, 1.0, 1e-6]).repeat(cols // 3 + 1)[None, :cols]
        x = x * s
    elif pattern == "zeros":                        # half exact zeros, plus zero rows / columns
        x = torch.randn(rows, cols, generator=g) * (torch.rand(rows, cols, generator=g) < 0.5)
        x[::5] = 0.0
        x[:, ::7] = 0.0
    elif pattern == "lo0":                          # the low plane is exactly 0
        x = torch.randn(rows, cols, generator=g).bfloat16().float()
    elif pattern == "lo1":                          # in [1, 2), low planes all positive: 0.3 .. 0.45 of half a bf16 ulp (2^-8)
        x0 = (1.0 + torch.rand(rows, cols, generator=g)).bfloat16().float()
        x = x0 + 2.0**-8 * (0.3 + 0.15 * torch.rand(rows, cols, generator=g))
    else:
        raise ValueError(pattern)
    return x.cuda()


PATTERNS = ["randn", "nonneg", "scaled", "zeros", "lo0", "lo1"]


def _pow2_rsqrt(n):
    """a power of two near 1 / sqrt(n): scales weights without changing their bf16 planes"""
    return 2.0 ** -math.floor(math.log2(max(n, 1)) / 2)


def _planes(x):
    hi = x.bfloat16().float()
    lo = (x - hi).bfloat16().float()
    return hi.double(), lo.double()


def _split_oracle(a, b, precision):
    """S and T of a @ b^T (a [M, K], b [N, K], fp32) over the bf16 planes, in fp64"""
    a0, a1 = _planes(a)
    b0, b1 = _planes(b)
    if precision == "bf16":
        return a0 @ b0.T, a0.abs() @ b0.abs().T
    s = a0 @ b0.T + a1 @ b0.T + a0 @ b1.T
    t = a0.abs() @ b0.abs().T + a1.abs() @ b0.abs().T + a0.abs() @ b1.abs().T
    return s, t


def _softplus64(z):
    return torch.nn.functional.softplus(z, beta=100, threshold=20)


def _act64(z, epi):
    return _softplus64(z) if epi == 1 else torch.relu(z) if epi == 2 else z


def _act_bound(ez, h, epi):
    return ez + (2.0**-20 * h.abs() + 2.0**-24 if epi == 1 else 0.0)


# ---------------------------------------------------------------------------------------------------------------
# nt / nn
# ---------------------------------------------------------------------------------------------------------------
def _run_linear(kind, precision, P, N, K, xv, wv, bias=None, epi=0, ldx_extra=32, ldy_extra=8, ldw_extra=3):
    """Y = epi(X W^T + b) (nt: X [P, K], W [N, K]) or Y = X W (nn: X [P, N], W [N, K]) through the C ABI, with NaN read canaries and
    sentinel write canaries.  Returns (Y buffer, its width)."""
    L = _lib()
    lib = L.load()
    xin = K if kind == "nt" else N
    yout = N if kind == "nt" else K
    X = Buf(P, xin, pad16(xin) + ldx_extra, float("nan"))
    X.v.copy_(xv)
    W = Buf(N, K, K + ldw_extra, float("nan"))
    W.v.copy_(wv)
    Y = Buf(P, pad16(yout), pad16(yout) + ldy_extra, SENT)
    ws = _ws()
    n0 = L.launch_count()
    if kind == "nt":
        B = None
        if bias is not None:
            B = torch.full((pad16(N) + 6,), float("nan"), device="cuda")   # pointer 8 bytes in; NaN past pad16(N)
            B[2:2 + pad16(N)] = bias
        rc = lib.sdfb200_gemm_nt(L.PRECISION[precision], X.p, X.ld, W.p, W.ld, N, K, None if B is None else B[2:].data_ptr(), epi, Y.p, Y.ld, P,
                                 ws.data_ptr(), ws.numel(), L.stream_ptr())
    else:
        rc = lib.sdfb200_gemm_nn(L.PRECISION[precision], X.p, X.ld, W.p, W.ld, N, K, Y.p, Y.ld, P, ws.data_ptr(), ws.numel(), L.stream_ptr())
    assert rc == 0, lib.sdfb200_last_error_string()
    chunks = math.ceil(pad16(yout) / CHUNK) * math.ceil(pad16(xin) / CHUNK)
    assert L.launch_count() - n0 == (2 * chunks if P > 0 else 0)           # one tc_pack + one k_tc_linear per (N, K) chunk
    torch.cuda.synchronize()
    assert (Y.outside() == SENT).all(), "write outside [P, pad16] of Y"
    return Y, yout


def _check_linear(kind, precision, P, N, K, pattern, epi, with_bias, g):
    xin = K if kind == "nt" else N
    xv = _values(pattern, P, xin, g)
    wv = _values(pattern if pattern != "scaled" else "randn", N, K, g) * _pow2_rsqrt(K if kind == "nt" else N)
    bias = None
    if with_bias:
        bias = torch.randn(pad16(N), generator=g).cuda() * 0.05
        bias[::4] = 0.0                                                     # exact zeros (ReLU at z = 0 where the row is 0)
    Y, yout = _run_linear(kind, precision, P, N, K, xv, wv, bias, epi)
    y = Y.v.double()
    if P == 0:
        return
    wk = wv if kind == "nt" else wv.T.contiguous()                          # nn is nt with W^T
    s, t = _split_oracle(xv, wk, precision)
    chunks = math.ceil(pad16(xin) / CHUNK)
    e = (TERMS[precision] * min(xin, CHUNK) * UT + (chunks - 1) * U) * 1.01 * t
    b = torch.zeros(yout, dtype=torch.float64, device="cuda") if bias is None else bias[:yout].double()
    if bias is not None:
        e = e + U * (t + b.abs())
    ref = _act64(s + b, epi)
    _record(f"{kind}/{precision}/split", (y[:, :yout] - ref).abs(), _act_bound(e, ref, epi))
    if precision == "bf16x3":
        xt = xv.double() @ wk.double().T
        tt = xv.double().abs() @ wk.double().abs().T
        ref_t = _act64(xt + b, epi)
        _record(f"{kind}/{precision}/fp64", (y[:, :yout] - ref_t).abs(), _act_bound(e + SPLIT * tt, ref_t, epi))
    # padding columns: zero for epilogue 0 without bias, epilogue(bias pad) otherwise (the weight rows there are zero)
    pad = y[:, yout:]
    if pad.shape[1]:
        if bias is None:
            assert (pad == 0).all()
        else:
            bp = bias[yout:].double()
            ref_p = _act64(bp, epi).expand_as(pad)
            _record(f"{kind}/{precision}/pad", (pad - ref_p).abs(), _act_bound(torch.zeros_like(pad), ref_p, epi))


DIMS = [1, 3, 15, 16, 17, 31, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512, 513, 600]
P_LINEAR = [0, 1, 31, 32, 33, 127, 128, 129, 4095, 4097]
# every N and every K once (7 is prime to 20), P cycling through P_LINEAR; then the layer shapes: angelo / bakedsdf 71 and 167 -> 256,
# 256 -> 257 (skip), 217, 3, the NeRF field's 63 + 256 skip and its 128-wide head, the generic engine's 320
LINEAR_CASES = [(P_LINEAR[i % len(P_LINEAR)], n, DIMS[(7 * i + 5) % len(DIMS)]) for i, n in enumerate(DIMS)]
LINEAR_CASES += [(4097, 256, 71), (2049, 256, 167), (4097, 257, 256), (1000, 217, 256), (4097, 3, 256), (4097, 256, 319), (999, 128, 283),
                 (4097, 320, 320)]
assert sorted({k for _, _, k in LINEAR_CASES[:20]}) == sorted(DIMS)
assert any(k > 2 * CHUNK and n > 2 * CHUNK for _, n, k in LINEAR_CASES)        # three K chunks and three N chunks in one call
EPIS = [(0, False), (0, True), (1, True), (2, True)]


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("P,N,K", LINEAR_CASES)
def test_nt_table(P, N, K, precision):
    g = torch.Generator().manual_seed(P * 7 + N * 131 + K)
    for i, pattern in enumerate(PATTERNS):
        epi, wb = EPIS[(i + N + K) % len(EPIS)]
        if pattern == "lo1" or K > 2 * CHUNK:
            epi, wb = 1 if pattern != "lo1" else 0, pattern != "lo1"             # lo1 unmasked by an activation; bias over 3 K chunks
        _check_linear("nt", precision, P, N, K, pattern, epi, wb, g)


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("P,N,K", LINEAR_CASES)
def test_nn_table(P, N, K, precision):
    g = torch.Generator().manual_seed(P * 5 + N * 17 + K)
    for pattern in PATTERNS:
        _check_linear("nn", precision, P, K, N, pattern, 0, False, g)      # nn over the same table with N and K swapped: X [P, K] W [K, N]


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_epilogue_edges(precision):
    """softplus(beta = 100) around its 0.2 threshold, in its log branch, where e underflows (z < -0.87) and at 0; ReLU at exact zeros
    and signed zeros.  K = 1, W = 1: z is the split sum of x, exactly."""
    z = torch.tensor([0.2, 0.19999, 0.20001, 0.2 - 2**-20, 0.2 + 2**-20, 0.1999999, 0.2000001, 0.15, 0.05, 0.01, 1e-3, 0.0, -0.0, -1e-3, -0.01,
                      -0.1, -0.5, -0.86, -0.88, -0.9, -0.95, -2.0, -50.0, 1.0, 30.0, 1e-30, -1e-30])
    P = z.numel()
    xv = z.view(P, 1).cuda()
    wv = torch.ones(3, 1, device="cuda")
    for epi in (1, 2):
        bias = torch.tensor([0.0, 0.0, 0.0, 0.25]).cuda()                   # pad16(3) = 16 is padded below
        bias = torch.nn.functional.pad(bias, (0, 12), value=0.125)
        Y, _ = _run_linear("nt", precision, P, 3, 1, xv, wv, bias, epi)
        y = Y.v.double()
        s, _ = _split_oracle(xv, wv, precision)
        ref = _act64(s, epi)
        _record(f"nt/{precision}/epilogue", (y[:, :3] - ref).abs(), _act_bound(U * s.abs(), ref, epi))
        if epi == 2:
            zero = (s[:, 0] <= 0)
            assert (y[zero, :3] == 0).all() and not torch.isnan(y).any()
        pad_ref = _act64(bias[3:].double(), epi).expand(P, -1)
        _record(f"nt/{precision}/epilogue", (y[:, 3:] - pad_ref).abs(), _act_bound(torch.zeros_like(pad_ref), pad_ref, epi))


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("aux_cols", [200, 256, 300])
def test_dsoftplus_epilogue_across_n_chunks(aux_cols, precision):
    """epilogue 3 (Y *= softplus'(aux), columns < aux_cols) through the debug hook, with aux_cols before, at and inside the second
    256-wide N chunk and K over three chunks; the factor is held to an absolute 2^-21."""
    L = _lib()
    lib = L.load_debug()
    g = torch.Generator().manual_seed(aux_cols)
    M, Np, Kp = 1000, 512, 528
    xv = _values("randn", M, Kp, g)
    X = Buf(M, Kp, Kp + 32, float("nan"))
    X.v.copy_(xv)
    wv = torch.randn(Np, Kp, generator=g).cuda() / Kp**0.5
    aux = (torch.rand(M, Np, generator=g) * 0.02).cuda()
    aux[:, ::9] = 0.0
    aux[::7, 1::9] = 1e-12
    aux[::5, 2::9] = 1e-9
    aux[:, 3::9] = 0.5
    Y = Buf(M, Np, Np + 4, SENT)
    ws = _ws()
    lib.sdfb200_launch_count.restype = ctypes.c_int64                       # the debug library counts its own launches
    n0 = lib.sdfb200_launch_count()
    rc = lib.sdfb200_debug_tc_linear(2 if precision == "bf16x3" else 1, 3, X.p, X.ld, wv.data_ptr(), None, Y.p, Y.ld, M, Np, Kp, aux.data_ptr(), Np, aux_cols,
                                     ws.data_ptr(), L.stream_ptr())
    assert rc == 0, lib.sdfb200_last_error_string()
    assert lib.sdfb200_launch_count() - n0 == 2 * 2 * 3
    torch.cuda.synchronize()
    assert (Y.outside() == SENT).all()
    s, t = _split_oracle(xv, wv, precision)
    d = torch.ones_like(s)
    d[:, :aux_cols] = -torch.expm1(-100.0 * aux[:, :aux_cols].double())
    e = (TERMS[precision] * CHUNK * UT + 2 * U) * 1.01 * t
    bound = e + t * 2.0**-21 * (torch.arange(Np, device="cuda") < aux_cols) + U * t      # |d| <= 1
    _record(f"dsoftplus/{precision}/split", (Y.v.double() - s * d).abs(), bound)


# ---------------------------------------------------------------------------------------------------------------
# tn
# ---------------------------------------------------------------------------------------------------------------
def _run_tn(precision, P, N, K, av, bv, lda_extra=5, ldb_extra=7, ldc_extra=3, expect_launches=True):
    L = _lib()
    lib = L.load()
    A = Buf(P, N, N + lda_extra, float("nan"))
    A.v.copy_(av)
    B = Buf(P, K, K + ldb_extra, float("nan"))
    B.v.copy_(bv)
    C = Buf(N, K, K + ldc_extra, SENT)
    ws = _ws()
    n0 = L.launch_count()
    rc = lib.sdfb200_gemm_tn(L.PRECISION[precision], A.p, A.ld, B.p, B.ld, C.p, C.ld, P, N, K, ws.data_ptr(), ws.numel(), L.stream_ptr())
    assert rc == 0, lib.sdfb200_last_error_string()
    chunks = math.ceil(N / WG_ROWS_A) * math.ceil(K / WG_ROWS_B)
    assert L.launch_count() - n0 == 2 * chunks                               # one k_tc_wgrad + one k_wgrad_reduce per (N, K) chunk
    torch.cuda.synchronize()
    assert (C.outside() == SENT).all(), "write outside [N, K] of C"
    return C


def _tn_bound(precision, P, t):
    ctas = _ctas()
    stages = math.ceil(P / WG_PTS)
    grid = min(ctas, max(stages, 1))
    spills = math.ceil(math.ceil(stages / grid) / WG_SLICE) if stages else 1
    return (TERMS[precision] * min(P, WG_PTS * WG_SLICE) * UT + (spills + grid) * U) * 1.01 * t


def _tn_cases():
    c = _ctas()
    S = WG_PTS * WG_SLICE * c                                                 # points at which a CTA's first slice is full
    shapes = [(65, 257), (129, 33), (17, 600), (128, 256), (600, 129), (64, 64), (1, 1), (257, 513), (63, 3), (127, 15), (3, 511),
              (256, 16), (31, 65), (33, 127)]
    ps = [0, 1, 31, 33, 4097, WG_PTS * (c - 1), WG_PTS * c, WG_PTS * c + 1, S - WG_PTS, S - 1, S, S + 1, S + WG_PTS, 2 * S + 1]
    return [(p, *shapes[i % len(shapes)]) for i, p in enumerate(ps)]


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("case", range(14))
def test_tn_table(case, precision):
    P, N, K = _tn_cases()[case]
    g = torch.Generator().manual_seed(case * 31 + N)
    pats = PATTERNS if P <= 4097 else ["randn", "nonneg", "lo1"]
    for pattern in pats:
        av = _values(pattern, P, N, g, rowscale=False)
        bv = _values(pattern if pattern != "scaled" else "randn", P, K, g, rowscale=False)
        C = _run_tn(precision, P, N, K, av, bv)
        c = C.v.double()
        if P == 0:
            assert (C.v == 0).all() and not torch.signbit(C.v).any()
            continue
        s, t = _split_oracle(av.T.contiguous(), bv.T.contiguous(), precision)
        e = _tn_bound(precision, P, t)
        _record(f"tn/{precision}/split", (c - s).abs(), e)
        if precision == "bf16x3":
            tt = av.double().abs().T @ bv.double().abs()
            _record(f"tn/{precision}/fp64", (c - av.double().T @ bv.double()).abs(), e + SPLIT * tt)
        if pattern == "randn":                                                # rerun: the same bits (fixed-order reduction)
            assert torch.equal(_run_tn(precision, P, N, K, av, bv).v, C.v)


# ---------------------------------------------------------------------------------------------------------------
# placement, non-finite values, past 2^31 elements
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("kind", ["nt", "nn"])
def test_rows_are_independent_of_their_placement(kind, precision):
    """gemm(X[a:b]) == rows a:b of gemm(X), bit for bit, with a not a multiple of the 128-row tile (two N chunks, three K chunks)"""
    g = torch.Generator().manual_seed(11)
    P, N, K, a, b = 1000, 300, 600, 77, 901
    xin = K if kind == "nt" else N
    xv = _values("randn", P, xin, g)
    wv = torch.randn(N, K, generator=g).cuda() * 0.05
    bias = (torch.randn(pad16(N), generator=g) * 0.1).cuda() if kind == "nt" else None
    full, _ = _run_linear(kind, precision, P, N, K, xv, wv, bias, 1 if kind == "nt" else 0)
    part, _ = _run_linear(kind, precision, b - a, N, K, xv[a:b], wv, bias, 1 if kind == "nt" else 0)
    assert torch.equal(part.v, full.v[a:b])


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_non_finite_values_stay_in_their_row_or_column(precision):
    """A NaN in X row r reaches only Y row r; a NaN in A[m, n] of tn only C row n, in B[m, k] only C column k; everything else is
    finite and bit-identical to the clean run.  +-Inf: under bf16x3 the split makes it NaN (lo = inf - inf), pinned as it is."""
    g = torch.Generator().manual_seed(5)
    P, N, K = 300, 130, 270
    xv = _values("randn", P, K, g)
    wv = torch.randn(N, K, generator=g).cuda() / K**0.5
    for kind in ("nt", "nn"):
        xin = K if kind == "nt" else N
        x = xv[:, :xin].contiguous()
        clean, yout = _run_linear(kind, precision, P, N, K, x, wv)
        for r, c, v in ((5, 3, float("nan")), (200, xin - 1, float("inf")), (129, 0, float("-inf"))):
            xb = x.clone()
            xb[r, c] = v
            y, _ = _run_linear(kind, precision, P, N, K, xb, wv)
            other = torch.ones(P, dtype=torch.bool, device="cuda")
            other[r] = False
            assert torch.equal(y.v[other], clean.v[other]) and torch.isfinite(y.v[other]).all()
            row = y.v[r, :yout]
            if v != v or precision == "bf16x3":
                assert torch.isnan(row).all(), (kind, r, v)
            else:
                assert not torch.isfinite(row).any(), (kind, r, v)
    A = _values("randn", P, N, g)
    B = _values("randn", P, K, g)
    clean = _run_tn(precision, P, N, K, A, B).v.clone()
    for which, (m, j) in (("A", (7, 129)), ("B", (250, 257))):
        a2, b2 = A.clone(), B.clone()
        (a2 if which == "A" else b2)[m, j] = float("nan")
        c = _run_tn(precision, P, N, K, a2, b2).v
        hit = torch.zeros_like(c, dtype=torch.bool)
        if which == "A":
            hit[j] = True
        else:
            hit[:, j] = True
        assert torch.isnan(c[hit]).all() and torch.equal(c[~hit], clean[~hit])


@pytest.mark.parametrize("precision", ["bf16x3"])
@pytest.mark.parametrize("kind", ["nt", "nn", "tn"])
def test_past_2p31_elements(kind, precision):
    """One call with P = 2^23 + 129 rows of 256 (2^31 + 33024 elements per operand), checked on sampled rows (nt / nn: the first tile,
    the rows around element 2^31 and the tail; tn: all of C, against a chunked fp64 sum).  Needs about 17 GB of device memory."""
    L = _lib()
    lib = L.load()
    P, N, K = 2**23 + 129, 256, 256
    g = torch.Generator(device="cuda").manual_seed(3)
    ws = _ws()
    prec = L.PRECISION[precision]
    if kind in ("nt", "nn"):
        X = torch.randn(P, 256, device="cuda", generator=g)
        W = torch.randn(N, K, device="cuda", generator=g) / 16.0
        Y = torch.full((P + 1, 256), SENT, device="cuda")
        if kind == "nt":
            rc = lib.sdfb200_gemm_nt(prec, X.data_ptr(), 256, W.data_ptr(), K, N, K, None, 0, Y.data_ptr(), 256, P, ws.data_ptr(), ws.numel(), L.stream_ptr())
        else:
            rc = lib.sdfb200_gemm_nn(prec, X.data_ptr(), 256, W.data_ptr(), K, N, K, Y.data_ptr(), 256, P, ws.data_ptr(), ws.numel(), L.stream_ptr())
        assert rc == 0, lib.sdfb200_last_error_string()
        torch.cuda.synchronize()
        assert (Y[P] == SENT).all()
        rows = torch.cat([torch.arange(0, 128), torch.arange(2**23 - 300, 2**23 + 40), torch.arange(P - 200, P)]).cuda()
        wk = W if kind == "nt" else W.T.contiguous()
        s, t = _split_oracle(X[rows], wk, precision)
        e = (TERMS[precision] * CHUNK * UT) * 1.01 * t
        _record(f"{kind}/{precision}/split", (Y[rows].double() - s).abs(), e)
        del X, Y
    else:
        A = torch.rand(P, N, device="cuda", generator=g)
        B = torch.rand(P, K, device="cuda", generator=g)
        C = torch.full((N + 1, K), SENT, device="cuda")
        rc = lib.sdfb200_gemm_tn(prec, A.data_ptr(), N, B.data_ptr(), K, C.data_ptr(), K, P, N, K, ws.data_ptr(), ws.numel(), L.stream_ptr())
        assert rc == 0, lib.sdfb200_last_error_string()
        torch.cuda.synchronize()
        assert (C[N] == SENT).all()
        s = torch.zeros(N, K, dtype=torch.float64, device="cuda")
        t = torch.zeros_like(s)
        for c0 in range(0, P, 1 << 20):
            ds, dt = _split_oracle(A[c0:c0 + (1 << 20)].T.contiguous(), B[c0:c0 + (1 << 20)].T.contiguous(), precision)
            s += ds
            t += dt
        _record(f"tn/{precision}/split", (C[:N].double() - s).abs(), _tn_bound(precision, P, t))
        del A, B
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------
# autograd closure (linear_ops), bf16x3 against fp64 autograd of plain matmuls
# ---------------------------------------------------------------------------------------------------------------
# Every derivative below is a sum of products of the inputs and seeds (matmuls and transposes only), so the same graph evaluated in fp64
# on |inputs| gives the magnitude M of each output's terms.  A bf16x3 GEMM errs by at most (3.1 * 2^-16 + n 2^-23) of its terms'
# magnitude (n <= 3 * 300 here: < 1.6e-4 per GEMM); a chain of up to four of them, each rounded to fp32, stays below 2^-10 M.
EG = 2.0**-10


def _ref_nt(x, W):
    K, N = W.shape[1], W.shape[0]
    return torch.nn.functional.pad(x[:, :K] @ W.T, (0, pad16(N) - N))


def _ref_nn(g, W):
    N, K = W.shape
    return torch.nn.functional.pad(g[:, :N] @ W, (0, pad16(K) - K))


def _ref_tn(a, b, N, K):
    return a[:, :N].T @ b[:, :K]


def _leaves(ts, dtype, absval):
    out = []
    for t in ts:
        t = t.detach().to(dtype)
        out.append((t.abs() if absval else t).requires_grad_(True))
    return out


def _check_grads(tag, fn, ref_fn, inputs, order):
    """derivatives of `order` 1..3 of <fn(inputs), seed> (each further order contracts the previous gradients with fresh seeds),
    on the kernels vs fp64 autograd of the plain-matmul restatement"""
    g = torch.Generator().manual_seed(len(tag))
    outs = []
    for f, dtype, absval in ((fn, torch.float32, False), (ref_fn, torch.float64, False), (ref_fn, torch.float64, True)):
        torch.manual_seed(0)
        xs = _leaves(inputs, dtype, absval)
        y = f(*xs)
        gs = torch.Generator().manual_seed(1)
        seed = torch.randn(y.shape, generator=gs).to(y.device, dtype)
        loss = (y * (seed.abs() if absval else seed)).sum()
        res = []
        for k in range(order):
            grads = torch.autograd.grad(loss, xs, create_graph=k + 1 < order, allow_unused=True)
            grads = [torch.zeros_like(x) if gr is None else gr for x, gr in zip(xs, grads)]
            res.append(grads)
            if k + 1 < order:
                loss = 0
                for gr in grads:
                    sd = torch.randn(gr.shape, generator=gs).to(gr.device, dtype)
                    loss = loss + (gr * (sd.abs() if absval else sd)).sum()
        outs.append(res)
    for k in range(order):
        for i, (a, r, m) in enumerate(zip(outs[0][k], outs[1][k], outs[2][k])):
            _record(f"autograd/{tag}", (a.double() - r).abs(), EG * m + 1e-30)
    return outs[0]


def test_autograd_first_and_second_derivatives():
    from sdfstudio_b200 import linear_ops as lo

    g = torch.Generator().manual_seed(2)
    P, N, K = 300, 37, 53
    x = torch.nn.functional.pad(torch.randn(P, K, generator=g), (0, pad16(K) - K)).cuda()
    gy = torch.nn.functional.pad(torch.randn(P, N, generator=g), (0, pad16(N) - N)).cuda()
    W = (torch.randn(N, K, generator=g) / K**0.5).cuda()
    for order in (1, 2):
        gx = _check_grads(f"nt{order}", lambda x, W: lo.gemm_nt(x, W), _ref_nt, [x, W], order)[0][0]
        assert (gx[:, K:] == 0).all()                                         # input gradient on padding columns
        _check_grads(f"nn{order}", lambda g_, W: lo.gemm_nn(g_, W), _ref_nn, [gy, W], order)
        ga, gb = _check_grads(f"tn{order}", lambda a, b: lo.gemm_tn(a, b, N, K), lambda a, b: _ref_tn(a, b, N, K), [gy, x], order)[0]
        assert (ga[:, N:] == 0).all() and (gb[:, K:] == 0).all()               # _TN.backward: d/da and d/db


def test_autograd_third_order_chain():
    """nt -> nn -> tn -> nt, differentiated three times"""
    from sdfstudio_b200 import linear_ops as lo

    g = torch.Generator().manual_seed(3)
    P, N1, K1, K2, P2 = 200, 45, 29, 21, 70
    x = torch.nn.functional.pad(torch.randn(P, K1, generator=g), (0, pad16(K1) - K1)).cuda()
    W1 = (torch.randn(N1, K1, generator=g) / K1**0.5).cuda()
    W2 = (torch.randn(N1, K2, generator=g) / N1**0.5).cuda()
    x2 = torch.nn.functional.pad(torch.randn(P2, K1, generator=g), (0, pad16(K1) - K1)).cuda()

    def chain(nt, nn, tn):
        def f(x, W1, W2, x2):
            y = nt(x, W1)                         # [P, pad16(N1)]
            z = nn(y, W2)                         # [P, pad16(K2)]
            c = tn(z, x, K2, K1)                  # [K2, K1]
            return nt(x2, c)                      # [P2, pad16(K2)]
        return f

    _check_grads("chain3", chain(lo.gemm_nt, lo.gemm_nn, lo.gemm_tn), chain(_ref_nt, _ref_nn, _ref_tn), [x, W1, W2, x2], 3)


@pytest.mark.parametrize("act", [0, 1, 2])
def test_linear_with_activation_against_fp64_autograd(act):
    """linear_ops.linear at N % 16 != 0 and K % 16 != 0: forward, d/dx, d/dW, d/db.  The activation's derivative is taken from the
    kernel's own output, so its error adds |gy| * 100 * |dy| for softplus; ReLU elements within the forward bound of the kink are left
    out of the gradient check (either side is right there).  Input-gradient padding columns are exactly 0, and NaN in the padding
    columns of the output gradient changes nothing."""
    from sdfstudio_b200 import linear_ops as lo

    g = torch.Generator().manual_seed(act)
    P, N, K = 500, 45, 71
    xv = torch.randn(P, K, generator=g) * 0.3
    Wv = torch.randn(N, K, generator=g) / K**0.5 * 0.3
    bv = torch.randn(N, generator=g) * 0.05
    gyv = torch.randn(P, N, generator=g)
    x = torch.nn.functional.pad(xv, (0, pad16(K) - K)).cuda().requires_grad_(True)
    W, b = Wv.cuda().requires_grad_(True), bv.cuda().requires_grad_(True)
    y = lo.linear(x, W, b, act)
    gy = torch.nn.functional.pad(gyv, (0, pad16(N) - N), value=float("nan")).cuda()
    gx, gW, gb = torch.autograd.grad(y, (x, W, b), gy)
    assert (gx[:, K:] == 0).all() and torch.isfinite(gW).all() and torch.isfinite(gb).all()
    gy0 = gy.nan_to_num(0.0)
    assert all(torch.equal(u, v) for u, v in zip((gx, gW, gb), torch.autograd.grad(lo.linear(x, W, b, act), (x, W, b), gy0)))
    x64, W64, b64 = xv.double().cuda(), Wv.double().cuda(), bv.double().cuda()
    z = x64 @ W64.T + b64
    m = x64.abs() @ W64.abs().T + b64.abs()
    yr = _act64(z, act)
    ez = EG * m
    ey = _act_bound(ez, yr, act)
    _record(f"linear/act{act}", (y.detach()[:, :N].double() - yr).abs(), ey)
    g64 = gyv.double().cuda()
    dact = torch.sigmoid(100 * z) if act == 1 else (z > 0).double() if act == 2 else torch.ones_like(z)
    gz = g64 * dact
    egz = g64.abs() * 100 * ey if act == 1 else torch.zeros_like(z)
    keep = (z.abs() > ez) if act == 2 else torch.ones_like(z, dtype=torch.bool)
    gz_k, gza, egz = gz * keep, (gz.abs() + egz) * keep, egz * keep
    if act == 2:
        gx_k, gW_k, gb_k = torch.autograd.grad(lo.linear(x, W, b, act), (x, W, b), torch.nn.functional.pad(gyv.cuda() * keep, (0, pad16(N) - N)))
    else:
        gx_k, gW_k, gb_k = gx, gW, gb
    _record(f"linear/act{act}/dx", (gx_k[:, :K].double() - gz_k @ W64).abs(), EG * gza @ W64.abs() + egz @ W64.abs())
    _record(f"linear/act{act}/dW", (gW_k.double() - gz_k.T @ x64).abs(), EG * gza.T @ x64.abs() + egz.T @ x64.abs())
    _record(f"linear/act{act}/db", (gb_k.double() - gz_k.sum(0)).abs(), P * U * gza.sum(0) + egz.sum(0))
