"""-m gpu: the hash-MLP field kernel k_hash_mlp_field<T, F, H, HC> (csrc/hash_mlp.cuh) against fp64, through both C entry points
(sdfb200_density_field_forward: the proposal density field, HC = 0; sdfb200_nerfacto_field_forward: the grid background field, HC > 0)
and through the two modules (HashMLPDensityField, TCNNNerfactoField).

Every one of the 42 instantiations runs (table fp32 / fp16 x F {1, 2, 4, 8} x H {16, 32, 64} for the density half, table x H x HC
{16, 32, 64} for the colour half, F = 2), and the last test checks that the file launched each of them.

Inputs of the oracle.  The grid is evaluated in fp64 (oracle/hashgrid.py) at the kernel's own fp32 normalised positions: under the aabb
and the L-inf contraction they are bit-identical to the fp32 restatement (oracle.nerfacto.normalize), and each level takes the kernel's
fp32 position (fp32_positions), so fp64 blends the same cell with the same offsets.  The SH input is the kernel's fp32
((d + 1) * 0.5) * 2 - 1, made of correctly rounded operations, which is exact in fp64.  An fp16 table is held as table.half().double().
Only the kernel's arithmetic is measured.

Bounds are element-wise, propagated in fp64 alongside the oracle, u = 2^-24, gamma_K = K u / (1 - K u):
  grid feature   FWD_K u sum_c |w_c| |t_c| (FWD_K = 14, `weight_mag`): the grid operator's forward bound (test_gpu_grid_operator.py);
                 encode_level is the same code
  ReLU layer     fan-in K, input h with error e_in: every accumulator is a chain of K fmaf, so |fl(W h^) - W h| <= gamma_K |W| |h^|
                 and e_out = |W| e_in + gamma_K |W| (|h| + e_in).  ReLU is 1-Lipschitz.  The output rows (pre-activation, geometry
                 feature, the three colour logits) take the same step.
  density        expf has at most 2 ulp error (<= 4u relative; build.py has no fast-math): e = density (e^e_pre - 1) + EXP_K u density
                 e^e_pre, EXP_K = 4
  SH term        SH_K = 8 u times the term's magnitude with |.| on every factor (`sh_magnitude`): the rounded constant, at most three
                 products and one sum or fused multiply-add
  rgb            1 / (1 + expf(-z)): the sigmoid is 1/4-Lipschitz, and its evaluation adds expf (4u), the sum (u) and the quotient (u):
                 e = e_z / 4 + SIG_K u min(1, rgb + e_z / 4), SIG_K = 8
"""
import math

import pytest
import torch

from oracle import hashgrid
from oracle import nerfacto as onf

from helpers import corner_factors, geometry, weight_mag

pytestmark = pytest.mark.gpu

U = 2.0**-24
FWD_K, EXP_K, SH_K, SIG_K = 14, 4, 8, 8
DEV = "cuda"
BASE_RES = 16
AABB = [[-2.0, -2.0, -2.0], [2.0, 2.0, 2.0]]

# the instantiation matrix: (table dtype, F, H, HC), HC = 0 the density half alone; the colour half is instantiated for F = 2 only
DTYPES, FEATURES, WIDTHS = ("fp32", "fp16"), (1, 2, 4, 8), (16, 32, 64)
DENSITY = [(dt, F, H, 0) for dt in DTYPES for F in FEATURES for H in WIDTHS]
COLOUR = [(dt, 2, H, HC) for dt in DTYPES for H in WIDTHS for HC in WIDTHS]
INSTANTIATIONS = DENSITY + COLOUR
LAUNCHED = set()      # (dt, F, H, HC) of every launch this file made
WORST = {}            # (dt, F, H, HC) -> largest err / bound over the file


@pytest.fixture(autouse=True)
def _keep_global_rng():
    """the modules built here draw their initial weights from torch's global generators: restore them afterwards, so that the tests
    after this file see the generator state they would see without it"""
    cpu, gpu = torch.get_rng_state(), torch.cuda.get_rng_state_all()
    yield
    torch.set_rng_state(cpu)
    torch.cuda.set_rng_state_all(gpu)


def iid(inst):
    dt, F, H, HC = inst
    return f"{dt}-F{F}-H{H}" + (f"-HC{HC}" if HC else "")


def _lib():
    import sdfstudio_b200 as sb

    return sb._lib


def gamma(K):
    return K * U / (1 - K * U)


class Net:
    """One descriptor of either entry point with flat weights in the tcnn layout (density_fields.fully_fused_weights): base [H, in_pad] |
    (n_base - 1) x [H, H] | [16, H], head [HC, head_pad] | (n_head - 1) x [HC, HC] | [16, HC].  hc = 0: the density entry point, whose
    output is row 0 alone.  `pad` fills every padding region: the padded input columns and the output rows nothing reads."""

    def __init__(self, F, L, H, n_base, hc=0, n_head=1, geo=0, app=0, log2T=12, max_res=256, norm="linf", seed=0, pad=0.0):
        from sdfstudio_b200.encoding import make_grid_desc

        self.F, self.L, self.H, self.n_base, self.hc, self.n_head, self.geo, self.app, self.norm = F, L, H, n_base, hc, n_head, geo, app, norm
        self.max_res, self.growth = max_res, hashgrid.growth_factor(L, BASE_RES, max_res)
        self.desc = make_grid_desc("tcnn", L, F, log2T, BASE_RES, self.growth, False)
        self.meta = hashgrid.tcnn_grid_meta(L, F, log2T, BASE_RES, self.growth)
        self.scales = torch.tensor([self.desc.scale[l] for l in range(L)], dtype=torch.float32)
        assert self.scales.tolist() == [float(s) for s in self.meta["scale"]]
        self.in_dim, self.in_pad = L * F, (L * F + 15) // 16 * 16
        self.n_out = 1 + geo if hc else 1
        self.head_in = 16 + geo + app
        self.head_pad = (self.head_in + 15) // 16 * 16
        g = torch.Generator().manual_seed(seed)
        self.table = torch.rand(self.desc._total_entries * F, generator=g) * 2 - 1
        self.base = self._mlp(g, self.in_dim, self.in_pad, H, n_base, self.n_out, pad)
        self.head = self._mlp(g, self.head_in, self.head_pad, hc, n_head, 3, pad) if hc else None
        self.app_rows = torch.randn(64, max(app, 1), generator=g)[:, :app] * 0.5

    @staticmethod
    def _mlp(g, in_dim, in_pad, H, n_hidden, n_out, pad):
        w0 = torch.full((H, in_pad), pad)
        w0[:, :in_dim] = torch.randn(H, in_dim, generator=g) * math.sqrt(2.0 / in_dim)
        ws = [w0.reshape(-1)] + [(torch.randn(H, H, generator=g) * math.sqrt(2.0 / H)).reshape(-1) for _ in range(n_hidden - 1)]
        wo = torch.full((16, H), pad)
        wo[:n_out] = torch.randn(n_out, H, generator=g) * (1.5 / math.sqrt(H))
        return torch.cat(ws + [wo.reshape(-1)])

    def level_rows(self, active):
        """[rows of the table] True for the rows of levels >= active"""
        lvl = torch.zeros(self.desc._total_entries, dtype=torch.bool)
        for l in range(active, self.L):
            lvl[self.desc.offset[l]: self.desc.offset[l] + self.desc.size[l]] = True
        return lvl.repeat_interleave(self.F)

    def nerfacto_desc(self, S):
        d = _lib().NerfactoDesc()
        d.hidden_dim, d.n_hidden_layers, d.hidden_dim_color, d.n_hidden_layers_color = self.H, self.n_base, self.hc, self.n_head
        d.geo_feat_dim, d.appearance_dim, d.n_samples = self.geo, self.app, S
        d.contraction = {"aabb": _lib().CONTRACT_NONE, "linf": _lib().CONTRACT_LINF, "l2": _lib().CONTRACT_L2}[self.norm]
        return d

    def smem_bytes(self, rgb=True):
        """the kernel's dynamic shared memory (launch_hash_mlp): base weights (with the 16-row output block when there is a colour half),
        then the head's weights up to its three live output rows"""
        H, hc = self.H, self.hc
        base = H * self.in_pad + (self.n_base - 1) * H * H + (16 if hc else 1) * H
        head = hc * self.head_pad + (self.n_head - 1) * hc * hc + 3 * hc if hc and rgb else 0
        return 4 * (base + head)


def _grid_desc(net, dt, active=None):
    L = _lib()
    d = L.GridDesc.from_buffer_copy(net.desc)
    d.table_dtype = L.DT_F16 if dt == "fp16" else L.DT_F32
    d.active_levels = net.L if active is None else active
    return d


def _table(net, dt, table=None):
    t = net.table if table is None else table
    return (t.half() if dt == "fp16" else t).to(DEV).contiguous()


def run_density(net, pos, dt="fp32", active=None, table=None, base=None):
    """sdfb200_density_field_forward in point mode: {density, pre}"""
    L = _lib()
    n = pos.shape[0]
    t, w = _table(net, dt, table), (net.base if base is None else base).to(DEV).contiguous()
    out = {"density": torch.full((n,), float("nan"), device=DEV), "pre": torch.full((n,), float("nan"), device=DEV)}
    aabb = torch.tensor(AABB, device=DEV) if net.norm == "aabb" else None
    code = {"aabb": L.CONTRACT_NONE, "linf": L.CONTRACT_LINF, "l2": L.CONTRACT_L2}[net.norm]
    p = pos.to(DEV).contiguous()
    L.check(L.load().sdfb200_density_field_forward(_grid_desc(net, dt, active), t.data_ptr(), w.data_ptr(), net.H, net.n_base, code, L.ptr(aabb),
                                                   p.data_ptr(), n, out["density"].data_ptr(), out["pre"].data_ptr(), None), "density")
    torch.cuda.synchronize()
    if n:
        LAUNCHED.add((dt, net.F, net.H, 0))
    return out


def run_colour(net, origins, directions, bins=None, app=None, stride=None, dt="fp32", active=None, table=None, base=None, head=None, n_rows=None,
               want_rgb=True):
    """sdfb200_nerfacto_field_forward, point mode when bins is None: {density, pre, geo, rgb}.  `app` is a CUDA tensor whose data pointer
    is row 0 (a column slice is passed as is, with its row stride)."""
    L = _lib()
    S = 0 if bins is None else bins.shape[1] - 1
    R = origins.shape[0] if n_rows is None else n_rows
    n = R * S if S else R
    t = _table(net, dt, table)
    bw = (net.base if base is None else base).to(DEV).contiguous()
    hw = (net.head if head is None else head).to(DEV).contiguous()
    out = {k: torch.full(s, float("nan"), device=DEV) for k, s in (("density", (n,)), ("pre", (n,)), ("geo", (n, net.geo)), ("rgb", (n, 3)))}
    aabb = torch.tensor(AABB, device=DEV) if net.norm == "aabb" else None
    stride = net.app if stride is None else stride
    rc = L.load().sdfb200_nerfacto_field_forward(_grid_desc(net, dt, active), net.nerfacto_desc(S), t.data_ptr(), bw.data_ptr(), hw.data_ptr(), L.ptr(aabb),
                                                 origins.data_ptr(), None if directions is None else directions.data_ptr(),
                                                 None if bins is None else bins.data_ptr(), R, None if app is None else app.data_ptr(), stride,
                                                 out["density"].data_ptr(), out["rgb"].data_ptr() if want_rgb else None, out["pre"].data_ptr(),
                                                 out["geo"].data_ptr() if net.geo else None, None)
    L.check(rc, "nerfacto")
    torch.cuda.synchronize()
    if n:
        LAUNCHED.add((dt, net.F, net.H, net.hc))
    return out


# ------------------------------------------------------------------------------------------------------------------ the oracle and its bound
def x01_of(net, pos):
    """the kernel's fp32 normalised positions (oracle.nerfacto.normalize in fp32)"""
    pos = pos.detach().float().cpu()
    return onf.normalize(pos, torch.tensor(AABB), None) if net.norm == "aabb" else onf.normalize(pos, None, net.norm)


def sh_input(dirs):
    """the kernel's fp32 SH input ((d + 1) * 0.5) * 2 - 1, each operation correctly rounded"""
    d = dirs.detach().float().cpu()
    return ((d + 1.0) * 0.5) * 2.0 - 1.0


def sh_magnitude(x):
    """per SH term, its magnitude with |.| on every factor and summand (the terms of csrc/hash_mlp.cuh sh4)"""
    a, b, c = x.abs().unbind(-1)
    xx, yy, zz = a * a, b * b, c * c
    return torch.stack([
        torch.full_like(a, 0.28209479177387814), 0.48860251190291987 * b, 0.48860251190291987 * c, 0.48860251190291987 * a,
        1.0925484305920792 * a * b, 1.0925484305920792 * b * c, 0.94617469575755997 * zz + 0.31539156525251999, 1.0925484305920792 * a * c,
        0.54627421529603959 * (xx + yy), 0.59004358992664352 * b * (3 * xx + yy), 2.8906114426405538 * a * b * c,
        0.45704579946446572 * b * (1 + 5 * zz), 0.3731763325901154 * c * (5 * zz + 3), 0.45704579946446572 * a * (1 + 5 * zz),
        1.4453057213202769 * c * (xx + yy), 0.59004358992664352 * a * (xx + 3 * yy),
    ], -1)  # fmt: skip


def _layers(w, x, e, in_dim, in_pad, H, n_hidden, n_out):
    """the FullyFusedMLP walk of oracle.nerfacto.mlp with the error bound beside it: (out [N, n_out], its bound)"""
    def lin(W, h, eh):
        A = W.abs()
        return h @ W.t(), eh @ A.t() + gamma(W.shape[1]) * ((h.abs() + eh) @ A.t())

    o = H * in_pad
    z, ez = lin(w[:o].view(H, in_pad)[:, :in_dim], x, e)
    h = torch.relu(z)
    for _ in range(n_hidden - 1):
        z, ez = lin(w[o: o + H * H].view(H, H), h, ez)
        h, o = torch.relu(z), o + H * H
    out, eo = lin(w[o: o + 16 * H].view(16, H)[:n_out], h, ez)
    assert torch.allclose(out, onf.mlp(x, w, in_dim, H, n_hidden, n_out), rtol=1e-12, atol=1e-12)
    return out, eo


def reference(net, x01, dirs=None, app=None, dt="fp32", table=None):
    """fp64 outputs {density, pre, geo, rgb} at the kernel's fp32 normalised positions x01 [N, 3], and their element-wise bounds"""
    t = net.table if table is None else table
    t64 = (t.half() if dt == "fp16" else t).double().to(DEV).view(-1, net.F)
    x32 = x01.float().to(DEV)
    feat, rows = hashgrid.encode_tcnn_layout(x32.double(), t64, net.meta, net.F, False, return_indices=True, fp32_positions=True)
    w, _, _ = geometry(x32, net.scales, "tcnn", False)
    fmag = (weight_mag(corner_factors(w))[..., None] * t64.abs()[rows]).sum(2).reshape(x32.shape[0], -1)
    base = net.base.double().to(DEV).nan_to_num(0.0)
    out, eo = _layers(base, feat, FWD_K * U * fmag, net.in_dim, net.in_pad, net.H, net.n_base, net.n_out)
    pre, e_pre = out[:, 0], eo[:, 0]
    dens = torch.exp(pre)
    r = {"pre": pre, "density": dens, "geo": out[:, 1:]}
    b = {"pre": e_pre, "density": dens * torch.expm1(e_pre) + EXP_K * U * dens * torch.exp(e_pre), "geo": eo[:, 1:]}
    if dirs is not None:
        xs = sh_input(dirs).double().to(DEV)
        sh = onf.sh4_tcnn(xs)
        a64 = app.double().to(DEV)
        v = torch.cat([sh, r["geo"], a64], -1)
        ev = torch.cat([SH_K * U * sh_magnitude(xs), b["geo"], torch.zeros_like(a64)], -1)
        z, ez = _layers(net.head.double().to(DEV).nan_to_num(0.0), v, ev, net.head_in, net.head_pad, net.hc, net.n_head, 3)
        r["rgb"] = torch.sigmoid(z)
        b["rgb"] = ez / 4 + SIG_K * U * (r["rgb"] + ez / 4).clamp(max=1.0)
        # the oracle module's own composition on the same inputs (xs is exact in fp64 as the direction it stands for)
        assert torch.allclose(r["rgb"], onf.rgb(xs, r["geo"], a64, net.head.double().to(DEV).nan_to_num(0.0), _spec(net)), rtol=1e-12, atol=1e-12)
    return r, b


def _spec(net):
    return onf.NerfactoSpec(num_levels=net.L, max_res=net.max_res, log2_hashmap_size=net.desc.log2_hashmap_size,
                            hidden_dim=net.H, num_layers=net.n_base + 1, geo_feat_dim=net.geo, hidden_dim_color=net.hc, num_layers_color=net.n_head + 1,
                            appearance_embedding_dim=net.app)


def check(what, got, ref, bound, inst=None, rows=None):
    """every element finite and within its bound; records the largest err / bound of the instantiation"""
    for k in ref:
        if k not in got or (k == "geo" and ref[k].shape[1] == 0):
            continue
        g = got[k].detach().double().to(DEV)
        g = g if rows is None else g[rows]
        g = g.reshape(ref[k].shape)
        assert bool(torch.isfinite(g).all()), f"{what} {k}: {int((~torch.isfinite(g)).sum())} non-finite outputs"
        err, bnd = (g - ref[k]).abs(), bound[k]
        bad = ~(err <= bnd)
        if bool(bad.any()):
            i = int(torch.nonzero(bad.reshape(-1))[0])
            raise AssertionError(f"{what} {k}: {int(bad.sum())} of {bad.numel()} out of bound; first at {i}: got {float(g.reshape(-1)[i])!r} "
                                 f"ref {float(ref[k].reshape(-1)[i])!r} err {float(err.reshape(-1)[i]):.3e} bound {float(bnd.reshape(-1)[i]):.3e}")
        if inst is not None:
            WORST[inst] = max(WORST.get(inst, 0.0), float((err / bnd.clamp_min(1e-300)).max()))


# ------------------------------------------------------------------------------------------------------------------ inputs
def points(n, norm, seed):
    g = torch.Generator().manual_seed(seed)
    if norm == "aabb":
        return (torch.rand(n, 3, generator=g) * 2 - 1) * 1.95
    return torch.randn(n, 3, generator=g) * 2.5      # about half outside the unit cube: contracted


def directions(n, seed):
    return torch.nn.functional.normalize(torch.randn(n, 3, generator=torch.Generator().manual_seed(seed)), dim=-1)


def rays(R, S, norm, seed):
    """origins, directions [R, 3], sorted euclidean bins [R, S + 1]; under the aabb every midpoint stays inside it"""
    g = torch.Generator().manual_seed(seed)
    d = directions(R, seed + 1)
    if norm == "aabb":
        o, lo, hi = (torch.rand(R, 3, generator=g) - 0.5), 0.05, 1.4
    else:
        o = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1) * (2.0 + 0.8 * torch.rand(R, 1, generator=g))
        lo, hi = 0.2, 8.0
    bins = torch.sort(lo + (hi - lo) * torch.rand(R, S + 1, generator=g), -1).values
    return o, d, bins


def midpoints(o, d, bins):
    """Frustums.get_positions in fp32 (the kernel's ray_midpoint, rounding for rounding) and the per-sample directions"""
    R, S = bins.shape[0], bins.shape[1] - 1
    pos = onf.midpoints(o[:, None], d[:, None], bins[:, :-1, None], bins[:, 1:, None])
    return pos.reshape(-1, 3), d[:, None].expand(R, S, 3).reshape(-1, 3)


def cuda(*ts):
    return [None if t is None else t.to(DEV).contiguous() for t in ts]


def check_density(net, pos, inst, what, dt="fp32", table=None, **kw):
    got = run_density(net, pos, dt, table=table, **kw)
    r, b = reference(net, x01_of(net, pos), dt=dt, table=table)
    check(what, got, r, b, inst)
    return got


def check_colour(net, pos, dirs, app_rows, got, inst, what, dt="fp32", table=None, rows=None):
    r, b = reference(net, x01_of(net, pos), dirs, app_rows, dt=dt, table=table)
    check(what, got, r, b, inst, rows)


# ------------------------------------------------------------------------------------------------------------------ every instantiation
DENSITY_LEVELS = {1: 12, 2: 11, 4: 7, 8: 5}           # in_dim 12, 22, 28, 40: every layer 0 has padded columns
GEO_APP = [(15, 32), (3, 7), (0, 0), (15, 0), (8, 20), (0, 40)]


@pytest.mark.parametrize("inst", INSTANTIATIONS, ids=iid)
def test_instantiation_matches_fp64(inst):
    """one descriptor per instantiation, hidden layers, normalisation and mode varied across the matrix; an fp16 table is bit-equal to
    the fp32-table call on the quantised table; two identical calls give identical bits; ray mode equals point mode on its midpoints"""
    dt, F, H, HC = inst
    i = INSTANTIATIONS.index(inst)
    if HC == 0:
        net = Net(F, DENSITY_LEVELS[F], H, n_base=1 + i % 4, norm=("aabb", "linf")[(i // 4) % 2], seed=i)
        pos = points(2000, net.norm, seed=i)
        q = net.table.half().float()
        got = check_density(net, pos, inst, iid(inst), dt)
        if dt == "fp16":
            got32 = run_density(net, pos, "fp32", table=q)
            assert torch.equal(got["density"], got32["density"]) and torch.equal(got["pre"], got32["pre"])
        again = run_density(net, pos, dt)
        assert all(torch.equal(got[k], again[k]) for k in got)
        return
    j = i - len(DENSITY)
    geo, app = GEO_APP[j % len(GEO_APP)]
    net = Net(F, (16, 11, 8)[j % 3], H, n_base=1 + j % 3, hc=HC, n_head=1 + (j // 3) % 3, geo=geo, app=app, norm=("aabb", "linf")[j % 2], seed=i)
    ray_mode = (j // 2) % 2 == 1
    if ray_mode:
        R, S = 40, 49                                      # 1960 samples: not a multiple of the 256-thread block
        o, d, bins = rays(R, S, net.norm, seed=i)
        cam = torch.randint(0, 64, (R,), generator=torch.Generator().manual_seed(i))
        app_r = net.app_rows[cam]
        args = dict(origins=cuda(o)[0], directions=cuda(d)[0], bins=cuda(bins)[0], app=cuda(app_r)[0] if app else None)
        pos, dirs = midpoints(o, d, bins)
        app_s = app_r[:, None].expand(R, S, app).reshape(R * S, app)
    else:
        pos, dirs = points(2000, net.norm, seed=i), directions(2000, seed=i + 1)
        cam = torch.randint(0, 64, (2000,), generator=torch.Generator().manual_seed(i))
        app_s = net.app_rows[cam]
        args = dict(origins=cuda(pos)[0], directions=cuda(dirs)[0], app=cuda(app_s)[0] if app else None)
    got = run_colour(net, dt=dt, **args)
    check_colour(net, pos, dirs, app_s, got, inst, iid(inst), dt)
    if dt == "fp16":
        got32 = run_colour(net, dt="fp32", table=net.table.half().float(), **args)
        assert all(torch.equal(got[k], got32[k]) for k in got), "fp16 table != fp32 table on the quantised values"
    again = run_colour(net, dt=dt, **args)
    assert all(torch.equal(got[k], again[k]) for k in got), "two identical calls differ"
    if ray_mode:
        pt = run_colour(net, *cuda(pos, dirs), app=cuda(app_s)[0] if app else None, dt=dt)
        assert all(torch.equal(got[k], pt[k]) for k in got), "ray mode != point mode on the same midpoints"


# ------------------------------------------------------------------------------------------------------------------ edges
@pytest.mark.parametrize("F,L", [(2, 8), (1, 17), (2, 15), (2, 17), (8, 6), (8, 32)])
def test_in_pad_edges(F, L):
    """n_levels * F = 16 (the reference's default proportion of HashMLPDensityField), 17, 30, 34, 48 and 256 (the most levels, F = 8)"""
    net = Net(F, L, 32, n_base=2, norm="linf", seed=L)
    pos = points(1500, "linf", seed=L)
    check_density(net, pos, ("fp32", F, 32, 0), f"density in_dim {L * F}")
    if F == 2:
        net = Net(F, L, 16, n_base=2, hc=32, n_head=2, geo=15, app=32, norm="aabb", seed=L)
        pos, dirs = points(1500, "aabb", seed=L), directions(1500, seed=L)
        app = net.app_rows[torch.arange(1500) % 64]
        got = run_colour(net, *cuda(pos, dirs), app=cuda(app)[0])
        check_colour(net, pos, dirs, app, got, ("fp32", 2, 16, 32), f"colour in_dim {L * F}")


@pytest.mark.parametrize("geo,app", [(0, 0), (0, 1), (15, 0), (15, 1), (15, 2), (0, 32), (7, 25), (0, 48), (15, 33)])
def test_head_pad_edges(geo, app):
    """16 + geo + app = 16, 17, 31, 32, 33, 48 and 64: the head's column offsets 16 + geo + k and the geo-dependent row loads"""
    net = Net(2, 10, 32, n_base=2, hc=16, n_head=2, geo=geo, app=app, norm="linf", seed=geo * 100 + app)
    R, S = 23, 31
    o, d, bins = rays(R, S, "linf", seed=geo + app)
    app_r = net.app_rows[torch.arange(R)]
    got = run_colour(net, *cuda(o, d), bins=cuda(bins)[0], app=cuda(app_r)[0] if app else None)
    pos, dirs = midpoints(o, d, bins)
    check_colour(net, pos, dirs, app_r[:, None].expand(R, S, app).reshape(R * S, app), got, ("fp32", 2, 32, 16), f"geo {geo} app {app}")


@pytest.mark.parametrize("abi", ["density", "nerfacto"])
def test_poisoned_padding_is_never_read(abi):
    """the same weights with every padding region zero and NaN: padded base input columns, base output rows 1 + geo..15 (1..15 for the
    density entry point), padded head input columns and head output rows 3..15.  The outputs are bit-identical."""
    kw = dict(F=2, L=5, H=16, n_base=2, seed=3)
    if abi == "density":
        clean, dirty = Net(**kw), Net(**kw, pad=float("nan"))
        pos = points(700, "linf", 5)
        a, b = run_density(clean, pos), run_density(dirty, pos)
    else:
        kw.update(hc=32, n_head=2, geo=5, app=7)                       # in_dim 10 (pad 16), head input 28 (pad 32)
        clean, dirty = Net(**kw), Net(**kw, pad=float("nan"))
        assert bool(torch.isnan(dirty.base).any()) and bool(torch.isnan(dirty.head).any())
        pos, dirs = points(700, "linf", 5), directions(700, 6)
        app = clean.app_rows[torch.arange(700) % 64]
        a, b = (run_colour(n, *cuda(pos, dirs), app=cuda(app)[0]) for n in (clean, dirty))
        check_colour(clean, pos, dirs, app, a, ("fp32", 2, 16, 32), "clean padding")
    assert torch.equal(clean.base.nan_to_num(0.0), dirty.base.nan_to_num(0.0))
    for k in a:
        assert bool(torch.isfinite(a[k]).all()) and torch.equal(a[k], b[k]), k


def test_shared_memory_above_48k():
    """the largest accepted descriptors, past the 48 KB default: colour 32 levels, H = HC = 64, 3 + 3 hidden layers (~103 KB); density
    F = 8, 32 levels, H = 64, 4 hidden layers (~115 KB)"""
    net = Net(2, 32, 64, n_base=3, hc=64, n_head=3, geo=15, app=33, norm="linf", seed=7)
    assert net.smem_bytes() > 100 * 1024
    pos, dirs = points(3000, "linf", 7), directions(3000, 8)
    app = net.app_rows[torch.arange(3000) % 64]
    got = run_colour(net, *cuda(pos, dirs), app=cuda(app)[0])
    check_colour(net, pos, dirs, app, got, ("fp32", 2, 64, 64), "colour 103 KB")
    net = Net(8, 32, 64, n_base=4, norm="aabb", seed=9)
    assert net.smem_bytes() > 112 * 1024
    check_density(net, points(3000, "aabb", 9), ("fp32", 8, 64, 0), "density 115 KB")
    check_density(net, points(1000, "aabb", 10), ("fp16", 8, 64, 0), "density 115 KB fp16", dt="fp16")


def test_stride_loop():
    """N = 2^19 + 37 points: more than any resident grid (2048 threads x 132 SMs = 270336), so every colour block strides.  A strided
    subset of rows and the last 300 rows against fp64."""
    net = Net(2, 16, 64, n_base=2, hc=64, n_head=2, geo=15, app=32, norm="linf", seed=11)
    N = (1 << 19) + 37
    pos, dirs = points(N, "linf", 11), directions(N, 12)
    app = net.app_rows[torch.arange(N) % 64]
    got = run_colour(net, *cuda(pos, dirs), app=cuda(app)[0])
    rows = torch.cat([torch.arange(0, N - 300, 1009), torch.arange(N - 300, N)])
    check_colour(net, pos[rows], dirs[rows], app[rows], got, ("fp32", 2, 64, 64), "stride loop", rows=rows.to(DEV))


@pytest.mark.parametrize("N", [1, 127, 129, 255, 257])
def test_sizes(N):
    dn = Net(4, 6, 32, n_base=2, norm="aabb", seed=N)
    check_density(dn, points(N, "aabb", N), ("fp32", 4, 32, 0), f"density N={N}")
    net = Net(2, 8, 32, n_base=1, hc=16, n_head=3, geo=4, app=9, norm="linf", seed=N)
    pos, dirs = points(N, "linf", N), directions(N, N + 1)
    app = net.app_rows[torch.arange(N) % 64]
    check_colour(net, pos, dirs, app, run_colour(net, *cuda(pos, dirs), app=cuda(app)[0]), ("fp32", 2, 32, 16), f"colour N={N}")


@pytest.mark.parametrize("R,S", [(300, 1), (37, 29), (1, 1)])
def test_ray_mode_shapes(R, S):
    """S = 1, and R * S not a multiple of the block"""
    net = Net(2, 8, 16, n_base=2, hc=64, n_head=1, geo=15, app=2, norm="aabb", seed=R + S)
    o, d, bins = rays(R, S, "aabb", seed=R)
    app_r = net.app_rows[torch.arange(R) % 64]
    got = run_colour(net, *cuda(o, d), bins=cuda(bins)[0], app=cuda(app_r)[0])
    pos, dirs = midpoints(o, d, bins)
    check_colour(net, pos, dirs, app_r[:, None].expand(R, S, 2).reshape(-1, 2), got, ("fp32", 2, 16, 64), f"R={R} S={S}")


def test_appearance_rows():
    """a per-ray row whose stride exceeds app_dim (a column slice of a wider tensor), stride 0 (one row for every sample), and NULL with
    app_dim > 0 (zeros)"""
    net = Net(2, 8, 32, n_base=2, hc=32, n_head=2, geo=6, app=11, norm="linf", seed=21)
    R, S = 29, 17
    o, d, bins = rays(R, S, "linf", seed=21)
    pos, dirs = midpoints(o, d, bins)
    wide = torch.randn(R, 40, generator=torch.Generator().manual_seed(3))
    cols = wide[:, 5:16]                                        # app_dim 11, row stride 40
    got = run_colour(net, *cuda(o, d), bins=cuda(bins)[0], app=wide.to(DEV)[:, 5:], stride=40)
    check_colour(net, pos, dirs, cols[:, None].expand(R, S, 11).reshape(-1, 11), got, ("fp32", 2, 32, 32), "sliced appearance")
    one = net.app_rows[3]
    got = run_colour(net, *cuda(o, d), bins=cuda(bins)[0], app=cuda(one)[0], stride=0)
    check_colour(net, pos, dirs, one.expand(R * S, 11), got, ("fp32", 2, 32, 32), "stride 0")
    got = run_colour(net, *cuda(o, d), bins=cuda(bins)[0], app=None)
    check_colour(net, pos, dirs, torch.zeros(R * S, 11), got, ("fp32", 2, 32, 32), "NULL appearance")


@pytest.mark.parametrize("abi", ["density", "nerfacto"])
def test_active_levels(abi):
    """levels >= active_levels contribute exactly zero: bit-equal to a run with every level active on a table whose rows for those levels
    are zero"""
    if abi == "density":
        net = Net(4, 7, 32, n_base=3, norm="linf", seed=31)
        pos = points(900, "linf", 31)
        run = lambda **kw: run_density(net, pos, **kw)  # noqa: E731
    else:
        net = Net(2, 9, 16, n_base=2, hc=16, n_head=2, geo=15, app=0, norm="aabb", seed=32)
        pos, dirs = cuda(points(900, "aabb", 32), directions(900, 33))
        run = lambda **kw: run_colour(net, pos, dirs, **kw)  # noqa: E731
    for active in (0, 1, net.L - 1):
        masked = run(active=active)
        zeroed = run(table=torch.where(net.level_rows(active), torch.zeros(()), net.table))
        for k in masked:
            assert bool(torch.isfinite(masked[k]).all()) and torch.equal(masked[k], zeroed[k]), (active, k)
    full = run()
    assert not torch.equal(full["pre"], run(active=net.L - 1)["pre"])


# ------------------------------------------------------------------------------------------------------------------ the modules
def _fill(params, g, mask_live, scale):
    with torch.no_grad():
        params.copy_(torch.where(mask_live, torch.randn(params.shape, generator=g) * scale, torch.zeros(())))


def _nerfacto_module(H, HC, geo, app, n_base, n_head, norm, seed):
    import sdfstudio_b200 as sb

    sd = None if norm == "aabb" else sb.SceneContraction(order=float("inf"))
    f = sb.TCNNNerfactoField(torch.tensor(AABB), num_images=6, num_layers=n_base + 1, hidden_dim=H, geo_feat_dim=geo, num_levels=8, max_res=256,
                             log2_hashmap_size=11, num_layers_color=n_head + 1, hidden_dim_color=HC, appearance_embedding_dim=app,
                             spatial_distortion=sd)
    g = torch.Generator().manual_seed(seed)
    nb, nh = f.mlp_base, f.mlp_head
    with torch.no_grad():   # the init's zero padding is kept; the live weights spread so that every output varies
        w = nb.params[: nb.n_net]
        w.copy_((w != 0).float() * torch.randn(w.shape, generator=g) * (2.0 / math.sqrt(H)))
        nb.params[nb.n_net:] = torch.rand(nb.n_grid, generator=g) * 2 - 1
        nh.params.copy_((nh.params != 0).float() * torch.randn(nh.params.shape, generator=g) * (1.5 / math.sqrt(HC)))
        f.embedding_appearance.embedding.weight.mul_(0.5)
    return f.to(DEV)


def _module_net(nb, hc, n_head, geo, app, norm, head_params=None, max_res=256):
    """a Net over a module's flat parameters (built with `max_res`)"""
    net = Net.__new__(Net)
    d = nb.desc
    net.F, net.L, net.H, net.n_base = d.n_features, d.n_levels, nb.hidden_dim, nb.n_hidden_layers
    net.hc, net.n_head, net.geo, net.app, net.norm = hc, n_head, geo, app, norm
    net.desc = d
    net.scales = torch.tensor([d.scale[l] for l in range(net.L)], dtype=torch.float32)
    net.max_res, net.growth = max_res, hashgrid.growth_factor(net.L, BASE_RES, max_res)
    net.meta = hashgrid.tcnn_grid_meta(net.L, net.F, d.log2_hashmap_size, BASE_RES, net.growth)
    assert net.scales.tolist() == [float(x) for x in net.meta["scale"]]
    net.in_dim, net.in_pad, net.n_out = nb.in_dim, nb.in_pad, nb.n_output_dims
    net.head_in = 16 + geo + app
    net.head_pad = (net.head_in + 15) // 16 * 16
    p = nb.params.detach().cpu()
    net.base, net.table = p[: nb.n_net], p[nb.n_net:]
    net.head = None if head_params is None else head_params.detach().cpu()
    return net


NERFACTO_SHAPES = [  # (H, HC, geo, app, n_base, n_head, norm)
    (16, 64, 15, 32, 1, 2, "linf"), (64, 16, 15, 32, 2, 1, "aabb"), (32, 32, 0, 0, 1, 1, "linf"), (32, 32, 0, 32, 3, 2, "aabb"),
    (32, 32, 15, 0, 1, 3, "linf"), (16, 16, 15, 33, 2, 2, "linf"),
]
DENSITY_SHAPES = [(4, 32, 1), (4, 64, 2), (8, 32, 3), (8, 64, 4)]   # (F, H, n_hidden)


def _relu_keep(net, x01, dirs=None, app=None, margin=1e-4):
    """False for samples with any ReLU input within `margin` of 0 (fp64): fp32 and fp64 may take different sides of that kink"""
    t64 = net.table.double().to(DEV).view(-1, net.F)
    feat = hashgrid.encode_tcnn_layout(x01.double().to(DEV), t64, net.meta, net.F, False, fp32_positions=True)

    def walk(x, w, in_dim, in_pad, H, n_hidden):
        z = x @ w[: H * in_pad].view(H, in_pad)[:, :in_dim].t()
        m, o = z.abs().amin(1), H * in_pad
        for _ in range(n_hidden - 1):
            z = torch.relu(z) @ w[o: o + H * H].view(H, H).t()
            m, o = torch.minimum(m, z.abs().amin(1)), o + H * H
        return m, torch.relu(z) @ w[o: o + 16 * H].view(16, H).t()

    m, out = walk(feat, net.base.double().to(DEV), net.in_dim, net.in_pad, net.H, net.n_base)
    if dirs is not None:
        v = torch.cat([onf.sh4_tcnn(sh_input(dirs).double().to(DEV)), out[:, 1: 1 + net.geo], app.double().to(DEV)], -1)
        m = torch.minimum(m, walk(v, net.head.double().to(DEV), net.head_in, net.head_pad, net.hc, net.n_head)[0])
    return m > margin


@pytest.mark.parametrize("shape", NERFACTO_SHAPES, ids=lambda s: "H{}-HC{}-geo{}-app{}-{}".format(s[0], s[1], s[2], s[3], s[6]))
def test_nerfacto_module_kernel_composition_and_gradients(shape):
    """TCNNNerfactoField: the eval kernel and the training composition both within the fp64 bound on the same samples; the training
    gradients of mlp_base.params, mlp_head.params and the embedding match fp64 autograd (samples near a ReLU kink masked); the padding
    of both networks gets exactly zero gradient"""
    import sdfstudio_b200 as sb
    from sdfstudio_b200.rays import make_ray_samples

    H, HC, geo, app, n_base, n_head, norm = shape
    f = _nerfacto_module(H, HC, geo, app, n_base, n_head, norm, seed=H + HC + geo + app)
    R, S = 40, 24
    o, d, bins = rays(R, S, norm, seed=geo + app + 1)
    cam = torch.randint(0, 6, (R,), generator=torch.Generator().manual_seed(2))
    rb = sb.RayBundle(origins=o.to(DEV), directions=d.to(DEV), pixel_area=torch.ones(R, 1, device=DEV), camera_indices=cam.view(R, 1).to(DEV))
    b = bins.to(DEV).contiguous()
    rs = make_ray_samples(rb, b, b, None)
    f.train()
    with torch.no_grad():
        k = f(rs)                                   # train mode under no_grad: the kernel with the per-camera rows
        pre_k = f._density_before_activation.clone()
    n0 = sb._lib.launch_count()
    out = f(rs)                                     # the differentiable composition
    assert out[sb.FieldHeadNames.RGB].requires_grad and sb._lib.launch_count() > n0
    x01_c = f._sample_locations.detach().reshape(-1, 3).cpu()
    pos, dirs = midpoints(o, d, bins)
    emb = f.embedding_appearance.embedding.weight.detach().cpu()
    app_s = emb[cam][:, None].expand(R, S, app).reshape(R * S, app)
    net = _module_net(f.mlp_base, HC, n_head, geo, app, norm, f.mlp_head.params)
    tag = f"module {shape}"
    inst = ("fp32", 2, H, HC)
    r, bnd = reference(net, x01_of(net, pos), dirs, app_s)
    got = {"density": k[sb.FieldHeadNames.DENSITY], "rgb": k[sb.FieldHeadNames.RGB], "pre": pre_k}
    check(tag + " kernel", got, r, bnd, inst)
    r, bnd = reference(net, x01_c, dirs, app_s)
    check(tag + " composition", {"density": out[sb.FieldHeadNames.DENSITY], "rgb": out[sb.FieldHeadNames.RGB]}, r, bnd)

    g = torch.Generator().manual_seed(5)
    keep = _relu_keep(net, x01_c, dirs, app_s).view(R, S, 1).cpu()
    assert float(keep.float().mean()) > 0.9
    c_rgb, c_d = torch.randn(R, S, 3, generator=g) * keep, torch.randn(R, S, 1, generator=g) * keep
    loss = (out[sb.FieldHeadNames.RGB] * c_rgb.to(DEV)).sum() + (torch.log1p(out[sb.FieldHeadNames.DENSITY]) * c_d.to(DEV)).sum()
    params = [f.mlp_base.params, f.mlp_head.params, f.embedding_appearance.embedding.weight]
    grads = torch.autograd.grad(loss, params, allow_unused=True)
    p64 = [p.detach().double().cpu().requires_grad_(True) for p in params]
    spec = _spec(net)
    dens64, _, geo64 = onf.density(x01_c.double(), p64[0], spec)
    rgb64 = onf.rgb(dirs.double(), geo64, p64[2][cam][:, None].expand(R, S, app).reshape(R * S, app), p64[1], spec)
    loss64 = (rgb64.view(R, S, 3) * c_rgb.double()).sum() + (torch.log1p(dens64.view(R, S, 1)) * c_d.double()).sum()
    g64 = torch.autograd.grad(loss64, p64, allow_unused=True)
    for name, a, e in zip(("mlp_base.params", "mlp_head.params", "embedding"), grads, g64):
        if e is None or e.numel() == 0:
            continue
        a = torch.zeros_like(e) if a is None else a.double().cpu()
        rel = float((a - e).abs().max() / e.abs().max().clamp_min(1e-30))
        assert rel < 2e-3, (name, rel)
    nb, nh = f.mlp_base, f.mlp_head
    w0 = grads[0][: nb.hidden_dim * nb.in_pad].view(nb.hidden_dim, nb.in_pad)
    assert int(torch.count_nonzero(w0[:, nb.in_dim:])) == 0
    h0 = grads[1][: nh.hidden_dim * nh.in_pad].view(nh.hidden_dim, nh.in_pad)
    assert int(torch.count_nonzero(h0[:, nh.in_dim:])) == 0
    for gr, width, live in ((grads[0][: nb.n_net], nb.hidden_dim, nb.n_output_dims), (grads[1], nh.hidden_dim, 3)):
        assert int(torch.count_nonzero(gr[-16 * width:].view(16, width)[live:])) == 0   # the output rows nothing reads


@pytest.mark.parametrize("F,H,n_hidden", DENSITY_SHAPES)
def test_density_module_kernel_composition_and_gradients(F, H, n_hidden):
    """HashMLPDensityField at F = 4 and 8, H = 32 and 64: the eval kernel and the training composition within the fp64 bound, and the
    parameter gradient against fp64 autograd"""
    import sdfstudio_b200 as sb
    from sdfstudio_b200.density_fields import normalized_positions

    f = sb.HashMLPDensityField(torch.tensor(AABB), num_layers=n_hidden + 1, hidden_dim=H, spatial_distortion=sb.SceneContraction(order=float("inf")),
                               num_levels=6, max_res=256, log2_hashmap_size=11, features_per_level=F).to(DEV)
    nb = f.mlp_base
    g = torch.Generator().manual_seed(F * H)
    with torch.no_grad():
        w = nb.params[: nb.n_net]
        w.copy_(((w != 0).float().cpu() * torch.randn(w.shape, generator=g) * (2.0 / math.sqrt(H))).to(DEV))
        nb.params[nb.n_net:] = (torch.rand(nb.n_grid, generator=g) * 2 - 1).to(DEV)
    pos = points(1500, "linf", F + H)
    net = _module_net(nb, 0, 1, 0, 0, "linf")
    f.eval()
    dens, pre = f.density_from_positions(pos.to(DEV), return_pre_activation=True)
    r, bnd = reference(net, x01_of(net, pos))
    check(f"density module F={F} H={H}", {"density": dens, "pre": pre}, r, bnd, ("fp32", F, H, 0))
    f.train()
    dens_c, pre_c = f.density_from_positions(pos.to(DEV), return_pre_activation=True)
    x01 = normalized_positions(pos.to(DEV), f.aabb, f.spatial_distortion).cpu()
    r, bnd = reference(net, x01)
    check(f"density composition F={F} H={H}", {"density": dens_c, "pre": pre_c}, r, bnd)
    keep = _relu_keep(net, x01).cpu()
    assert float(keep.float().mean()) > 0.9
    c = torch.randn(1500, 1, generator=g) * keep[:, None]
    (grad,) = torch.autograd.grad((dens_c * c.to(DEV)).sum(), nb.params)
    p64 = nb.params.detach().double().cpu().requires_grad_(True)
    t64 = p64[nb.n_net:].view(-1, F)
    feat = hashgrid.encode_tcnn_layout(x01.double(), t64, net.meta, F, False, fp32_positions=True)
    pre64 = onf.mlp(feat, p64[: nb.n_net], nb.in_dim, H, n_hidden, 1)
    (g64,) = torch.autograd.grad((torch.exp(pre64) * c.double()).sum(), p64)
    rel = float((grad.double().cpu() - g64).abs().max() / g64.abs().max())
    assert rel < 2e-3, rel
    w0 = grad[: H * nb.in_pad].view(H, nb.in_pad)
    assert int(torch.count_nonzero(w0[:, nb.in_dim:])) == 0
    assert int(torch.count_nonzero(grad[nb.n_net - 16 * H: nb.n_net].view(16, H)[1:])) == 0


@pytest.mark.parametrize("which", ["geo_feat_dim", "appearance_embedding_dim"])
def test_nerfacto_field_without_geo_feature_or_appearance_trains_and_evaluates(which):
    """geo_feat_dim = 0 or appearance_embedding_dim = 0: the training composition (an empty geometry feature or appearance row) and the
    eval kernel both run, and agree"""
    import sdfstudio_b200 as sb
    from sdfstudio_b200.rays import make_ray_samples

    f = sb.TCNNNerfactoField(torch.tensor(AABB), num_images=3, hidden_dim=16, hidden_dim_color=16, num_levels=4, max_res=64, log2_hashmap_size=10,
                             **{which: 0}).to(DEV).train()
    R, S = 8, 5
    o, d, bins = rays(R, S, "aabb", seed=1)
    rb = sb.RayBundle(origins=o.to(DEV), directions=d.to(DEV), pixel_area=torch.ones(R, 1, device=DEV), camera_indices=torch.zeros(R, 1, dtype=torch.long,
                                                                                                                                       device=DEV))
    rs = make_ray_samples(rb, bins.to(DEV).contiguous(), bins.to(DEV).contiguous(), None)
    out = f(rs)
    (out[sb.FieldHeadNames.RGB].sum() + out[sb.FieldHeadNames.DENSITY].sum()).backward()
    assert f.mlp_base.params.grad is not None and bool(torch.isfinite(f.mlp_head.params.grad).all())
    with torch.no_grad():
        k = f(rs)
    for key in (sb.FieldHeadNames.RGB, sb.FieldHeadNames.DENSITY):
        assert float((k[key] - out[key]).abs().max()) < 1e-5, key


def test_constructors_refuse_what_the_kernel_refuses():
    """a descriptor the kernel refuses raises NotImplementedError at construction, and one it accepts constructs and runs"""
    import sdfstudio_b200 as sb

    L = _lib()
    lib = L.load()
    pos = torch.rand(4, 3, device=DEV)
    out = torch.empty(4, 3, device=DEV)
    for num_layers in range(0, 8):
        for H in (8, 16, 32, 48, 64, 128):
            for F in (1, 2, 3, 4, 8):
                kw = dict(num_layers=num_layers, hidden_dim=H, num_levels=3, max_res=32, log2_hashmap_size=8, features_per_level=F)
                try:
                    f = sb.HashMLPDensityField(torch.tensor(AABB), **kw).to(DEV)
                except NotImplementedError:
                    f = None
                # the kernel's answer, on a descriptor of the same shape
                dn = Net(F if F != 3 else 2, 3, 16, n_base=1)
                gd = _grid_desc(dn, "fp32")
                gd.n_features = F
                w = torch.zeros(64 * 64 * 8, device=DEV)
                t = _table(dn, "fp32")
                rc = lib.sdfb200_density_field_forward(gd, t.data_ptr(), w.data_ptr(), H, num_layers - 1, L.CONTRACT_LINF, None, pos.data_ptr(), 4,
                                                       out.data_ptr(), None, None)
                assert (rc == 0) == (f is not None), (kw, rc)
                if f is not None:
                    f.eval()
                    assert bool(torch.isfinite(f.density_fn(pos)).all())
    torch.cuda.synchronize()
    base = dict(hidden_dim=16, hidden_dim_color=16, num_layers=2, num_layers_color=2, geo_feat_dim=15, appearance_embedding_dim=32)
    changes = [dict(hidden_dim=v) for v in (8, 16, 32, 64, 128)] + [dict(hidden_dim_color=v) for v in (8, 32, 48, 128)]
    changes += [dict(num_layers=v) for v in (1, 2, 4, 5)] + [dict(num_layers_color=v) for v in (1, 3, 4, 5)]
    changes += [dict(geo_feat_dim=v) for v in (-1, 0, 15, 16)] + [dict(appearance_embedding_dim=v) for v in (-1, 0, 33, 34)]
    changes += [dict(geo_feat_dim=0, appearance_embedding_dim=48), dict(geo_feat_dim=0, appearance_embedding_dim=49)]
    for change in changes:
        kw = dict(base, **change)
        try:
            f = sb.TCNNNerfactoField(torch.tensor(AABB), num_images=2, num_levels=3, max_res=32, log2_hashmap_size=8, **kw).to(DEV)
        except NotImplementedError:
            f = None
        d = L.NerfactoDesc()
        d.hidden_dim, d.n_hidden_layers = kw["hidden_dim"], kw["num_layers"] - 1
        d.hidden_dim_color, d.n_hidden_layers_color = kw["hidden_dim_color"], kw["num_layers_color"] - 1
        d.geo_feat_dim, d.appearance_dim, d.contraction, d.n_samples = kw["geo_feat_dim"], kw["appearance_embedding_dim"], L.CONTRACT_LINF, 0
        dn = Net(2, 3, 16, n_base=1)
        big = torch.zeros(1 << 16, device=DEV)
        t = _table(dn, "fp32")
        rc = lib.sdfb200_nerfacto_field_forward(_grid_desc(dn, "fp32"), d, t.data_ptr(), big.data_ptr(), big.data_ptr(), None, pos.data_ptr(),
                                                pos.data_ptr(), None, 4, None, 0, out.data_ptr(), out.data_ptr(), None, None, None)
        assert (rc == 0) == (f is not None), (change, rc)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------ coverage: keep last
def test_every_instantiation_ran(request):
    """the set of (table, F, H, HC) this file launched is the whole family; under -s, the largest err / bound per instantiation"""
    matrix = [it for it in request.session.items if it.originalname == "test_instantiation_matches_fp64" and it.module is request.module]
    if len(matrix) < len(INSTANTIATIONS):
        pytest.skip("the instantiation matrix was deselected")
    assert len(INSTANTIATIONS) == 42 and len(set(INSTANTIATIONS)) == 42
    assert LAUNCHED == set(INSTANTIATIONS), sorted(set(INSTANTIATIONS) ^ LAUNCHED)
    print("\nlargest err / bound per instantiation:")
    for inst in INSTANTIATIONS:
        print(f"  {iid(inst):22s} {WORST.get(inst, float('nan')):.3f}")
