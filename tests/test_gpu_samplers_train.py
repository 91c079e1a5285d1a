"""-m gpu: the ray samplers in TRAINING mode against the oracle fed the product's own jitter, and the sampler kernels at the shapes and
edges the eval-mode tests never reach.

Training mode draws the stratified jitter with torch.rand inside ray_samplers.py.  The ``recorder`` fixture passes every draw through and
keeps a CPU copy, so the fp32 / fp64 oracle (oracle/samplers.py) runs on exactly the jitter the kernels saw.  The ``injector`` fixture makes
torch.rand return chosen values (the ends of the jitter range).  The composite samplers run on a shared sdf / density function: the oracle's,
evaluated on CPU copies of the product's own sample positions, so only the sampler arithmetic differs."""
import pytest
import torch

from oracle import cases, samplers

from helpers import assert_within_noise, cdf_consistency, load_train_golden, make_bundle, oracle64, train_case_inputs

pytestmark = pytest.mark.gpu
TOP = 1.0 - 2.0**-24          # the largest value torch.rand returns
SPACINGS = ["uniform", "lindisp", "sqrt", "log", "piecewise"]


@pytest.fixture
def recorder(monkeypatch):
    """A list that receives (fn, CPU copy, dtype) for every torch.rand / torch.randint call, in call order."""
    log = []
    rand, randint = torch.rand, torch.randint

    def rec_rand(*a, **k):
        t = rand(*a, **k)
        log.append(("rand", t.detach().cpu().clone(), t.dtype))
        return t

    def rec_randint(*a, **k):
        t = randint(*a, **k)
        log.append(("randint", t.detach().cpu().clone(), t.dtype))
        return t

    monkeypatch.setattr(torch, "rand", rec_rand)
    monkeypatch.setattr(torch, "randint", rec_randint)
    return log


@pytest.fixture
def injector(monkeypatch):
    """``inject(fn)``: from then on torch.rand returns fn(shape) (on the requested device and dtype); ``inject(None)`` restores it.
    Request it before ``recorder`` so that the recorder sees the injected values."""
    rand = torch.rand
    state = {"fn": None}

    def inj_rand(*a, **k):
        t = rand(*a, **k)
        return t if state["fn"] is None else state["fn"](tuple(t.shape)).to(device=t.device, dtype=t.dtype).contiguous()

    monkeypatch.setattr(torch, "rand", inj_rand)
    return lambda fn: state.__setitem__("fn", fn)


def draws_of(log, fn="rand"):
    return [t for f, t, _ in log if f == fn]


def ulp(x):
    return (torch.nextafter(x.abs(), torch.tensor(float("inf"))) - x.abs())


def ray_set(R, seed):
    """R rays with per-ray near / far planes (positive, as lindisp and log need)."""
    g = torch.Generator().manual_seed(seed)
    o, d, cam = cases.synthetic_rays(R, seed)
    nears = 0.05 + torch.rand(R, 1, generator=g)
    fars = nears + 0.5 + 4.5 * torch.rand(R, 1, generator=g)
    return o, d, cam, nears, fars


def shared_sdf(oracle, o, d):
    import sdfstudio_b200 as sb

    def fn(rs):                                   # the ORACLE's fp32 sdf at the product's sample starts
        starts = sb.rays.bins_of(rs)[:, :-1].cpu()
        return oracle.get_sdf(o, d, starts).cuda()[..., None]
    return fn


class Beta0Density:
    """density_fn of the ErrorBoundedSampler: only get_beta() is read by the product (the kernels evaluate the Laplace density)."""

    def __init__(self, beta0):
        self.beta0 = float(beta0)

    def get_beta(self):
        return torch.tensor([self.beta0], device="cuda")


def shared_density(level):
    return lambda pos: cases.proposal_density(pos.detach().cpu(), level).cuda()


# ----------------------------------------------------------------------------------------------------------------
# 1. draw order: the product draws what the reference draws, in the same order
# ----------------------------------------------------------------------------------------------------------------
def _run_composite(which, rb, oracle, o, d, anneal=1.0, beta0=cases.TRAIN_SAMPLER_BETA0):
    import sdfstudio_b200 as sb

    sdf = shared_sdf(oracle, o, d)
    if which == "neus":
        return sb.NeuSSampler().train()(rb, sdf_fn=sdf)
    if which == "error_bounded":
        return sb.ErrorBoundedSampler(num_samples=64, num_samples_eval=128, num_samples_extra=32).train()(
            rb, density_fn=Beta0Density(beta0), sdf_fn=sdf, return_eikonal_points=True)
    if which == "unisurf":
        occ = lambda s: torch.sigmoid(-10.0 * s.cpu()).cuda()  # noqa: E731  (the reference's get_occupancy, on CPU like the oracle)
        return sb.UniSurfSampler().train()(rb, occupancy_fn=occ, sdf_fn=sdf, return_surface_points=True)
    ps = sb.ProposalNetworkSampler(num_proposal_samples_per_ray=(256, 96), num_nerf_samples_per_ray=48, num_proposal_network_iterations=2).train()
    ps.set_anneal(anneal)
    return ps(rb, density_fns=[shared_density(0), shared_density(1)])


@pytest.mark.parametrize("which", ["neus", "error_bounded", "unisurf", "proposal_anneal1", "proposal_anneal0.5"])
def test_draw_order_matches_reference(recorder, which):
    G, meta = load_train_golden()
    spec, kw, o, d, cam, nears, fars, oracle = train_case_inputs()
    anneal = 0.5 if which.endswith("0.5") else 1.0
    recorder.clear()
    _run_composite(which.split("_anneal")[0] if which.startswith("proposal") else which, make_bundle(o, d, cam, nears, fars), oracle, o, d, anneal)
    got = [(f, list(t.shape), str(dt).replace("torch.", "")) for f, t, dt in recorder]
    want = [(x["fn"], x["shape"], x["dtype"]) for x in meta["draws"][which]]
    assert got == want


# ----------------------------------------------------------------------------------------------------------------
# 2. spaced bins in training mode
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [1, 2, 31, 32, 33, 256])
@pytest.mark.parametrize("single", [True, False], ids=["single", "perbin"])
@pytest.mark.parametrize("kind", SPACINGS)
def test_spaced_bins_train(injector, recorder, kind, single, S):
    import sdfstudio_b200 as sb

    R = 1001
    o, d, cam, nears, fars = ray_set(R, 31 + S)
    rb = make_bundle(o, d, cam, nears, fars)
    sampler = sb.SpacedSampler(kind, None, num_samples=S, single_jitter=single).train()
    base = torch.linspace(0.0, 1.0, S + 1)
    lower = torch.cat([base[:1], (base[1:] + base[:-1]) / 2.0])
    upper = torch.cat([(base[1:] + base[:-1]) / 2.0, base[-1:]])
    for inject in (None, 0.0, TOP):
        injector(None if inject is None else (lambda shape, v=inject: torch.full(shape, v)))
        recorder.clear()
        rs = sampler(rb)
        (t_rand,) = draws_of(recorder)
        assert t_rand.shape == (R, 1 if single else S + 1)
        ob = samplers.spaced_sampler(nears, fars, S, kind, t_rand)
        sp, eu = sb.rays.spacing_bins_of(rs).cpu(), sb.rays.bins_of(rs).cpu()
        assert torch.equal(sp, ob.spacing), f"{kind} jitter={inject}: spacing bins differ"
        if kind == "uniform":
            assert torch.equal(eu, ob.euclid)
        else:
            # the exact map of the same spacing bins, in fp64; the fp32 oracle's own distance from it sets the bound
            exact = samplers.make_to_euclid(kind, nears.double(), fars.double())(sp.double())
            n_ulp = float(((eu.double() - exact).abs() / ulp(ob.euclid).double()).max())
            n_ulp_oracle = float(((ob.euclid.double() - exact).abs() / ulp(ob.euclid).double()).max())
            assert n_ulp <= max(4.0, 2.0 * n_ulp_oracle), f"{kind} jitter={inject}: {n_ulp:.1f} ulp from exact (fp32 oracle: {n_ulp_oracle:.1f})"
        if inject == 0.0:
            assert torch.equal(sp, lower.expand(R, -1))          # every bin at its lower end
        elif inject == TOP:
            assert float((upper - sp).abs().max()) <= 2.0**-23                           # every bin at its upper end


# ----------------------------------------------------------------------------------------------------------------
# 3. PDF sampling in training mode
# ----------------------------------------------------------------------------------------------------------------
def _pdf_weights(R, s_in, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(R, s_in, generator=g) ** 6
    w[:3] = 0.0                                          # all-zero rows
    w[3:6] = 0.0
    w[3:6, s_in // 2] = 1.0                              # single spike: flat cdf on both sides, cdf ties at 1.0 after it
    w[6:9] = torch.logspace(-30, 0, s_in)[torch.randperm(s_in, generator=g)] if s_in > 1 else 1e-30   # 30 decades, no NaN
    return w


def _searchsorted_fp64(w, u_rand, s_out, pad, eps=1e-5):
    """The PDF sampler's searchsorted(cdf, u, side="right") with the cdf built in fp64 from the same weights and the same fp32 u."""
    nb = s_out + 1
    wd = w.double() + pad
    ws = wd.sum(-1, keepdim=True)
    padding = torch.relu(eps - ws)
    wd = wd + padding / wd.shape[-1]
    cdf = torch.cumsum(wd / (ws + padding), -1).clamp(max=1.0)
    cdf = torch.cat([torch.zeros_like(cdf[:, :1]), cdf], -1)
    u = (torch.linspace(0.0, 1.0 - 1.0 / nb, nb).expand(w.shape[0], nb) + u_rand / nb).contiguous()
    return torch.searchsorted(cdf, u.double(), side="right")


@pytest.mark.parametrize("s_in,s_out", [(1, 1), (64, 16), (128, 64), (1024, 96)])
@pytest.mark.parametrize("single", [True, False], ids=["single", "perbin"])
def test_pdf_sample_train(injector, recorder, s_in, s_out, single):
    import sdfstudio_b200 as sb

    R, pad = 1001, 1e-5
    nb = s_out + 1
    o, d, cam, nears, fars = ray_set(R, 7 + s_in)
    rb = make_bundle(o, d, cam, nears, fars)
    rs = sb.UniformSampler(num_samples=s_in).eval()(rb)
    ob = samplers.spaced_sampler(nears, fars, s_in, "uniform")
    w = _pdf_weights(R, s_in, s_in + s_out)
    wc = w.cuda()[..., None]
    pdf = sb.PDFSampler(include_original=False, single_jitter=single, histogram_padding=pad).train()
    recorder.clear()
    new, inds = pdf(rb, rs, wc, num_samples=s_out, return_indices=True)
    (u_rand,) = draws_of(recorder)
    assert u_rand.shape == (R, 1 if single else nb)
    onew, oinds = samplers.pdf_sampler(ob, w, s_out, histogram_padding=pad, u_rand=u_rand, return_indices=True)
    # the weights' sum is accumulated in a different order than torch.sum: where u falls within rounding of a cdf entry the index may move
    # to the neighbouring bin.  Against the same search in an fp64 cdf, the kernel may flip no more indices than the fp32 oracle does (or
    # the eval-mode test's 1e-5 of the indices, whichever is larger)
    d_ind = (inds.cpu() - oinds).abs()
    assert int(d_ind.max()) <= 1
    exact = _searchsorted_fp64(w, u_rand, s_out, pad)
    flips, own = int((inds.cpu() != exact).sum()), int((oinds != exact).sum())
    assert flips <= max(int(1e-5 * exact.numel()), own), f"{flips} indices differ from the fp64 search (fp32 oracle: {own})"
    nbins = sb.rays.spacing_bins_of(new).cpu()
    assert (nbins == onew.spacing).float().mean() > 0.5
    u = torch.linspace(0.0, 1.0 - 1.0 / nb, nb).expand(R, nb) + u_rand / nb
    # |cdf(bin) - u| in fp64: 2e-6, or twice the fp32 oracle's own value on the same inputs (the 30-decade rows reach 3.9e-6 at s_in >= 128)
    c_own = cdf_consistency(ob.spacing, w, onew.spacing, u, pad)
    c = cdf_consistency(ob.spacing, w, nbins, u, pad)
    assert c < max(2e-6, 2.0 * c_own), f"cdf consistency {c:.2e} (fp32 oracle: {c_own:.2e})"

    # include_original on the same jitter: the sorted merge of the original bins with the bins drawn above
    injector(lambda shape: u_rand.clone())
    new2 = sb.PDFSampler(include_original=True, single_jitter=single, histogram_padding=pad).train()(rb, rs, wc, num_samples=s_out)
    want = torch.sort(torch.cat([ob.spacing, nbins], -1), -1)[0]
    assert torch.equal(sb.rays.spacing_bins_of(new2).cpu(), want)

    # the top jitter: u = linspace[-1] + (1 - 2^-24) / nb rounds to exactly 1.0f -> searchsorted runs past the cdf
    top = u_rand.clone()
    top[::7] = TOP
    injector(lambda shape: top.clone())
    new3, inds3 = pdf(rb, rs, wc, num_samples=s_out, return_indices=True)
    onew3, oinds3 = samplers.pdf_sampler(ob, w, s_out, histogram_padding=pad, u_rand=top, return_indices=True)
    u3 = torch.linspace(0.0, 1.0 - 1.0 / nb, nb).expand(R, nb) + top / nb
    at_one = u3[:, -1] == 1.0
    assert bool(at_one[::7].all())
    assert bool((oinds3[at_one, -1] == s_in + 1).all()) and bool((inds3.cpu()[at_one, -1] == s_in + 1).all())
    assert torch.equal(sb.rays.spacing_bins_of(new3).cpu()[at_one, -1], onew3.spacing[at_one, -1])
    assert torch.equal(onew3.spacing[at_one, -1], ob.spacing[at_one, -1])


# ----------------------------------------------------------------------------------------------------------------
# 4. composite samplers in training mode on a shared sdf / density function
# ----------------------------------------------------------------------------------------------------------------
def _case(name):
    from oracle.field import OracleField, init_params

    spec, kw, o, d, cam, nears, fars = cases.case_inputs(name)
    params = init_params(spec, **cases.init_kwargs(kw))
    return spec, kw, o, d, cam, nears, fars, OracleField(spec, params), params


SDF_CASES = ["neusfacto_c1", cases.TRAIN_SAMPLER_CASE]


@pytest.mark.parametrize("name", SDF_CASES)
def test_neus_sampler_train_on_shared_sdf(recorder, name):
    import sdfstudio_b200 as sb

    spec, kw, o, d, cam, nears, fars, oracle, params = _case(name)
    recorder.clear()
    rs = _run_composite("neus", make_bundle(o, d, cam, nears, fars), oracle, o, d)
    t_rand, *u_rands = draws_of(recorder)
    assert t_rand.shape == (o.shape[0], 1) and len(u_rands) == 4          # single jitter by default
    on = samplers.neus_sampler(nears, fars, lambda s: oracle.get_sdf(o, d, s), t_rand=t_rand, u_rands=u_rands)
    pn = sb.rays.spacing_bins_of(rs).cpu()
    if name == "neusfacto_c1":                              # the eval-mode test's case and bounds
        err = float((pn - on.spacing).abs().max())
        assert err < 2e-6, err
        assert float((pn == on.spacing).float().mean()) > 0.5
        assert torch.equal(torch.argsort(pn[:, :-1], dim=-1, stable=True), torch.argsort(on.spacing[:, :-1], dim=-1, stable=True))
    else:
        # the clean sphere concentrates the weights at inv_s up to 512: the inverse CDF is ill-conditioned (2.8e-4 measured), so the bound
        # is the fp32 oracle's own distance from the fp64 oracle on the same jitter, as in the golden test of the eval sampler
        o64 = oracle64(spec, params, kw)
        on64 = samplers.neus_sampler(nears.double(), fars.double(), lambda s: o64.get_sdf(o.double(), d.double(), s), t_rand=t_rand.double(),
                                     u_rands=[u.double() for u in u_rands])
        assert_within_noise(pn, on.spacing, on64.spacing, "NeuSSampler spacing bins", factor=6.0, floor=4e-6)


@pytest.mark.parametrize("name", SDF_CASES)
def test_error_bounded_sampler_train_on_shared_sdf(recorder, name):
    import sdfstudio_b200 as sb

    spec, kw, o, d, cam, nears, fars, oracle, params = _case(name)
    beta0 = float(oracle.get_beta()) if name == "neusfacto_c1" else cases.TRAIN_SAMPLER_BETA0
    recorder.clear()
    rs, points = _run_composite("error_bounded", make_bundle(o, d, cam, nears, fars), oracle, o, d, beta0=beta0)
    fns = [f for f, _, _ in recorder]
    k = fns.index("randint")
    draws = [t for _, t, _ in recorder]
    t_rand, u_rands, idx, t_extra = draws[0], draws[1:k], draws[k], draws[k + 1]
    oe, opts = samplers.error_bounded_sampler(nears, fars, lambda s: oracle.get_sdf(o, d, s), torch.tensor([beta0]), t_rand=t_rand, u_rands=u_rands,
                                              t_rand_extra=t_extra, eikonal_idx=idx, origins=o, directions=d)
    pe = sb.rays.spacing_bins_of(rs).cpu()
    assert pe.shape == oe.spacing.shape
    assert idx.shape == (o.shape[0] * 10,) and points.shape == (o.shape[0] * 10, 3)
    if name == "neusfacto_c1":                              # the eval-mode test's case and bounds (one iteration: beta0 converges)
        assert float((pe - oe.spacing).abs().max()) < 1e-4, float((pe - oe.spacing).abs().max())
        assert float((sb.rays.bins_of(rs).cpu() - oe.euclid).abs().max()) < 4e-4
        # eikonal points: the frustum centres of the final (pre-extra) samples at the recorded randint indices
        assert float((points.cpu() - opts).abs().max()) < 4e-4
    else:
        # five iterations at beta0 = 0.005 on a clean sphere: 1e-2 measured, against the fp32 oracle's own distance from the fp64 oracle
        o64 = oracle64(spec, params, kw)
        dbl = lambda t: t.double()  # noqa: E731
        oe64, opts64 = samplers.error_bounded_sampler(dbl(nears), dbl(fars), lambda s: o64.get_sdf(dbl(o), dbl(d), s), torch.tensor([beta0], dtype=torch.float64),
                                                      t_rand=dbl(t_rand), u_rands=[dbl(u) for u in u_rands], t_rand_extra=dbl(t_extra), eikonal_idx=idx,
                                                      origins=dbl(o), directions=dbl(d))
        assert_within_noise(pe, oe.spacing, oe64.spacing, "ErrorBoundedSampler spacing bins", factor=6.0, floor=2e-5)
        assert_within_noise(points, opts, opts64, "ErrorBoundedSampler eikonal points", factor=6.0, floor=1e-4)


@pytest.mark.parametrize("name", SDF_CASES)
def test_unisurf_sampler_train_on_shared_sdf(recorder, name):
    import sdfstudio_b200 as sb

    spec, kw, o, d, cam, nears, fars, oracle, params = _case(name)
    recorder.clear()
    rs, surf = _run_composite("unisurf", make_bundle(o, d, cam, nears, fars), oracle, o, d)
    draws = draws_of(recorder)
    if len(draws) == 5:                                   # no ray hit the surface: 1024 random surface points between outside and interval
        assert draws[3].shape == (1024, 3)
        draws = draws[:3] + draws[4:]
    t_march, u_imp, t_out, t_int = draws
    jit = dict(t_rand_march=t_march, u_rand_importance=u_imp, t_rand_outside=t_out, t_rand_interval=t_int)
    u32, s32, m32 = samplers.unisurf_sampler(o, d, nears, fars, lambda s: oracle.get_sdf(o, d, s), **jit)
    o64 = oracle64(spec, params, kw)
    jit64 = {k: v.double() for k, v in jit.items()}
    u64, _, _ = samplers.unisurf_sampler(o.double(), d.double(), nears.double(), fars.double(), lambda s: o64.get_sdf(o.double(), d.double(), s), **jit64)
    assert_within_noise(sb.rays.bins_of(rs), u32.euclid, u64.euclid, "UniSurfSampler euclid bins", factor=6.0, floor=1e-5)
    if bool(m32.any()):
        assert surf.shape == s32.shape
        torch.testing.assert_close(surf.cpu(), s32, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("anneal", [1.0, 0.5])
def test_proposal_sampler_train_on_shared_density(recorder, anneal):
    """The bench workload's sampler: piecewise initial spacing, (256, 96) proposal samples, 48 final samples, per-bin jitter."""
    import sdfstudio_b200 as sb

    R = 1000
    o, d, cam = cases.synthetic_rays(R, 77)
    nears, fars = torch.full((R, 1), 0.5), torch.full((R, 1), 4.5)
    recorder.clear()
    rs, weights_list, rs_list = _run_composite("proposal", make_bundle(o, d, cam, nears, fars), None, o, d, anneal=anneal)
    t_rand, *u_rands = draws_of(recorder)
    assert t_rand.shape == (R, 257) and [u.shape for u in u_rands] == [(R, 97), (R, 49)]
    dens = [lambda p, i=i: cases.proposal_density(p, i)[..., 0] for i in range(2)]
    ob, owl, obl = samplers.proposal_sampler(o, d, nears, fars, dens, (256, 96), 48, anneal=anneal, t_rand=t_rand, u_rands=u_rands)
    assert torch.equal(sb.rays.spacing_bins_of(rs_list[0]).cpu(), obl[0].spacing)
    torch.testing.assert_close(weights_list[0][..., 0].cpu(), owl[0], rtol=2e-4, atol=1e-6)
    # level 1 sits on PDF-drawn positions in a shell of width 0.02 with peak density 50: its weights move with the bins (1.8e-5 measured),
    # so they are held to the fp32 oracle's own distance from the fp64 oracle on the same jitter
    dbl = lambda t: t.double()  # noqa: E731
    dens64 = [lambda p, i=i: cases.proposal_density(p, i)[..., 0] for i in range(2)]
    _, owl64, _ = samplers.proposal_sampler(dbl(o), dbl(d), dbl(nears), dbl(fars), dens64, (256, 96), 48, anneal=anneal, t_rand=dbl(t_rand),
                                            u_rands=[dbl(u) for u in u_rands])
    assert_within_noise(weights_list[1][..., 0], owl[1], owl64[1], "proposal level-1 weights", factor=6.0, floor=1e-6)
    torch.testing.assert_close(sb.rays.bins_of(rs_list[1]).cpu(), obl[1].euclid, rtol=0, atol=5e-3)
    torch.testing.assert_close(sb.rays.bins_of(rs).cpu(), ob.euclid, rtol=0, atol=2e-2)
    assert (sb.rays.bins_of(rs)[:, 1:] >= sb.rays.bins_of(rs)[:, :-1]).all()


# ----------------------------------------------------------------------------------------------------------------
# 5. kernel edges (eval mode, direct library calls)
# ----------------------------------------------------------------------------------------------------------------
def _volsdf_inputs(R, S, dtype=torch.float32, seed=0):
    """Jittered bins on [0.5, 4.5] and an sdf with one crossing per ray (rays 3 mod 4 stay outside); ray 1 has a NaN sample."""
    g = torch.Generator().manual_seed(seed + S)
    nears, fars = torch.full((R, 1), 0.5), torch.full((R, 1), 4.5)
    eu = samplers.spaced_sampler(nears, fars, S, "uniform", torch.rand(R, S + 1, generator=g)).euclid
    surf = 1.0 + 3.0 * torch.rand(R, 1, generator=g)
    surf[3::4] = 9.0
    slope = 0.5 + torch.rand(R, 1, generator=g)
    sdf = (surf - eu[:, :-1]) * slope + 0.01 * torch.randn(R, S, generator=g)
    if R > 1:
        sdf[1, S // 2] = float("nan")                    # a blown-up field sample: the error bound is NaN, beta stays as it is
    return eu, sdf


def _volsdf_reference(eu, sdf, beta0, beta_init, eps, beta_iters):
    deltas = eu[:, 1:] - eu[:, :-1]
    d_star = samplers.volsdf_dstar(sdf, deltas)
    beta = samplers.volsdf_updated_beta(beta0, beta_init.clone(), sdf, d_star, deltas, eps, beta_iters)
    w, T = samplers.weights_from_density(deltas, samplers.laplace_density(sdf, beta[:, None]))
    b = beta[:, None]
    err_int = torch.cumsum(torch.exp(-d_star / b) * deltas**2 / (4 * b**2), -1)
    err_w = (torch.clamp(torch.exp(err_int), max=1.0e6) - 1.0) * T
    return beta, w, err_w


@pytest.mark.parametrize("beta_iters", [0, 10])
@pytest.mark.parametrize("R", [1, 5, 4099])
@pytest.mark.parametrize("S", [33, 100, 1000])
def test_volsdf_step_shapes_and_nan_rows(S, R, beta_iters):
    import sdfstudio_b200 as sb

    lib = sb._lib.load()
    eps = 0.1
    eu, sdf = _volsdf_inputs(R, S)
    beta0 = torch.tensor([0.02])
    deltas = eu[:, 1:] - eu[:, :-1]
    beta_init = torch.sqrt((1.0 / (4.0 * torch.log(torch.tensor(eps + 1.0)))) * (deltas**2.0).sum(-1))
    beta = beta_init.cuda()
    w = torch.empty(R, S, device="cuda")
    ew = torch.empty(R, S, device="cuda")
    euc, sdfc, b0c = eu.cuda().contiguous(), sdf.cuda().contiguous(), beta0.cuda()
    sb._lib.check(lib.sdfb200_volsdf_step(euc.data_ptr(), sdfc.data_ptr(), b0c.data_ptr(), beta.data_ptr(), R, S, eps, beta_iters, w.data_ptr(),
                                          ew.data_ptr(), 0), "sdfb200_volsdf_step")
    beta, w, ew = beta.cpu(), w.cpu(), ew.cpu()
    b32, w32, e32 = _volsdf_reference(eu, sdf, beta0, beta_init, eps, beta_iters)
    b64, w64, e64 = _volsdf_reference(eu.double(), sdf.double(), beta0.double(), beta_init.double(), eps, beta_iters)
    ok = ~torch.isnan(sdf).any(-1)
    if R > 1:
        assert not bool(ok[1])
        assert torch.equal(beta[~ok], beta_init[~ok]) and torch.equal(b32[~ok], beta_init[~ok])     # NaN bound: beta untouched
        nan_at = S // 2
        assert torch.equal(torch.isnan(w[1]), torch.isnan(w32[1]))                              # NaN from the NaN sample on
        assert not bool(torch.isnan(ew[1, :nan_at]).any())
    # weights and err weights are at most ~1 and ~eps; the fp32 oracle's own error on them is 3e-8 .. 8e-8, so the floor sits just above it
    assert_within_noise(beta[ok], b32[ok], b64[ok], f"volsdf beta S={S} R={R}", floor=1e-7)
    assert_within_noise(w[ok], w32[ok], w64[ok], f"volsdf weights S={S} R={R}", floor=1e-7)
    assert_within_noise(ew[ok], e32[ok], e64[ok], f"volsdf err weights S={S} R={R}", floor=1e-7)
    assert float(e64[ok].max()) > 1e-3                  # the err weights compared are not all ~0
    if beta_iters == 10:
        assert bool((beta[ok] <= beta_init[ok]).all()) and bool((beta[ok] >= 0.02).all())


def test_volsdf_step_refuses_more_than_1000_samples():
    import sdfstudio_b200 as sb

    lib = sb._lib.load()
    R, S = 1, 1001
    eu, sdf = _volsdf_inputs(R, S)
    euc, sdfc = eu.cuda().contiguous(), sdf.cuda().contiguous()
    b0, beta = torch.tensor([0.02], device="cuda"), torch.ones(R, device="cuda")
    w, ew = torch.empty(R, S, device="cuda"), torch.empty(R, S, device="cuda")
    torch.cuda.synchronize()
    n0 = sb._lib.launch_count()
    rc = lib.sdfb200_volsdf_step(euc.data_ptr(), sdfc.data_ptr(), b0.data_ptr(), beta.data_ptr(), R, S, 0.1, 10, w.data_ptr(), ew.data_ptr(), 0)
    assert rc != 0
    assert "1000" in lib.sdfb200_last_error_string().decode()
    assert sb._lib.launch_count() == n0


@pytest.mark.parametrize("S", [2, 33])
def test_neus_upsample_weights_small_and_rising(S):
    import sdfstudio_b200 as sb

    lib = sb._lib.load()
    R = 517
    g = torch.Generator().manual_seed(S)
    nears, fars = torch.full((R, 1), 0.5), torch.full((R, 1), 4.5)
    ob = samplers.spaced_sampler(nears, fars, S, "uniform", torch.rand(R, S + 1, generator=g))
    sdf = (2.0 - ob.starts) * (torch.rand(R, 1, generator=g) - 0.3)     # falling on some rays, rising (cos clamped to 0) on others
    sdf[::3] = ob.starts[::3] - 2.0                                        # every third ray: rising everywhere
    wk = torch.empty(R, S, device="cuda")
    euc, sdfc = ob.euclid.cuda().contiguous(), sdf.cuda().contiguous()
    sb._lib.check(lib.sdfb200_neus_upsample_weights(euc.data_ptr(), sdfc.data_ptr(), R, S, 64.0, wk.data_ptr(), 0), "sdfb200_neus_upsample_weights")
    al = samplers.neus_fixed_inv_s_alpha(ob.deltas, sdf, 64.0)
    ow, _ = samplers.weights_from_alphas(al)
    torch.testing.assert_close(wk.cpu()[:, :-1], ow, rtol=2e-5, atol=5e-7)
    assert float(wk[:, -1].abs().max()) == 0.0


def test_unisurf_interval_edges():
    import sdfstudio_b200 as sb

    lib = sb._lib.load()
    R, S, delta = 300, 64, 0.25
    g = torch.Generator().manual_seed(5)
    nears = 0.3 + torch.rand(R, 1, generator=g)
    fars = nears + 3.0
    ob = samplers.spaced_sampler(nears, fars, S, "uniform", torch.rand(R, S + 1, generator=g))
    t = ob.starts
    sdf = (1.0 + 2.0 * torch.rand(R, 1, generator=g) - t) * (0.5 + torch.rand(R, 1, generator=g))   # one positive-to-negative crossing
    sdf[0] = 0.5 + t[0]                                   # no crossing
    sdf[1] = t[1] - 2.0                                   # negative-to-positive first crossing (inside -> outside): no hit
    sdf[2] = -sdf[2]                                      # same, on a random ray
    sdf[3] = torch.linspace(1.0, -1.0, S)                 # a sample of exactly 0 at no crossing ...
    sdf[3, S // 2] = 0.0
    sdf[3, S // 2 + 1:] = sdf[3, S // 2 + 1:].abs()       # ... and positive after it: no sign change at all
    sdf[4] = 1.0 - 2.0 * t[4] / float(t[4, -1])           # exactly 0 next to a later crossing
    sdf[4, 10] = 0.0
    sdf[5] = 1.0                                          # crossing in the last pair
    sdf[5, -1] = -0.5
    sdf[6] = -1.0                                         # all negative
    sdf[7, :] = 0.0                                       # all zero
    sdf[8, 20] = 0.0                                      # an exact zero right before the crossing of a random ray
    euc, sdfc = ob.euclid.cuda().contiguous(), sdf.cuda().contiguous()
    nc, fc = nears.cuda().contiguous(), fars.cuda().contiguous()
    z = torch.empty(R, device="cuda")
    hit = torch.empty(R, device="cuda", dtype=torch.uint8)
    n2, f2 = torch.empty_like(z), torch.empty_like(z)
    sb._lib.check(lib.sdfb200_unisurf_interval(euc.data_ptr(), sdfc.data_ptr(), nc.data_ptr(), fc.data_ptr(), R, S, delta, z.data_ptr(), hit.data_ptr(),
                                               n2.data_ptr(), f2.data_ptr(), 0), "sdfb200_unisurf_interval")
    oz, mask, on2, of2 = samplers.unisurf_interval(t, sdf, nears, fars, delta)
    assert torch.equal(hit.cpu().bool(), mask)
    assert [bool(mask[i]) for i in range(8)] == [False, False, False, False, True, True, False, False]
    assert torch.equal(z.cpu()[mask], oz)
    assert bool(torch.isnan(z.cpu()[~mask]).all())
    assert torch.equal(n2.cpu(), on2[:, 0]) and torch.equal(f2.cpu(), of2[:, 0])
