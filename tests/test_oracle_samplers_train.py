"""Pins the oracle's TRAINING-mode samplers (oracle/samplers.py with explicit jitter) against the unmodified reference run in
.train() (oracle/make_golden_samplers_train.py): the reference's recorded torch.rand / torch.randint draws are fed to the oracle,
which must then reproduce the reference's bins.  CPU-only; runs everywhere."""
import pytest
import torch

from oracle import cases, samplers

from helpers import load_train_golden, train_case_inputs, train_draws

SPACINGS = ["uniform", "lindisp", "sqrt", "log", "piecewise"]


@pytest.fixture(scope="module")
def golden():
    return load_train_golden()


@pytest.fixture(scope="module")
def case():
    return train_case_inputs()


def close(a, b, atol):
    torch.testing.assert_close(a, b, rtol=0, atol=atol)


@pytest.mark.parametrize("jitter", ["single", "perbin"])
@pytest.mark.parametrize("kind", SPACINGS)
def test_spaced_sampler_train_bit_exact(golden, case, kind, jitter):
    G, meta = golden
    spec, kw, o, d, cam, nears, fars, oracle = case
    run = f"spaced_{kind}_{jitter}"
    (t_rand,) = train_draws(G, meta, run)
    assert t_rand.shape == (nears.shape[0], 1 if jitter == "single" else kw["S"] + 1)
    b = samplers.spaced_sampler(nears, fars, kw["S"], kind, t_rand)
    assert torch.equal(b.spacing, G[f"{run}.spacing"])
    assert torch.equal(b.euclid, G[f"{run}.euclid"])


@pytest.mark.parametrize("run", ["pdf_noinc_single", "pdf_noinc_perbin", "pdf_inc_single", "pdf_inc_perbin", "pdf_top_jitter"])
def test_pdf_sampler_train_bit_exact(golden, case, run):
    G, meta = golden
    spec, kw, o, d, cam, nears, fars, oracle = case
    (u_rand,) = train_draws(G, meta, run)
    base = samplers.spaced_sampler(nears, fars, kw["S"], "uniform")
    new, inds = samplers.pdf_sampler(base, G["pdf_weights"], meta["pdf_num_samples"], histogram_padding=0.01, include_original="_inc_" in run,
                                     u_rand=u_rand, return_indices=True)
    assert torch.equal(inds, G[f"{run}.inds"][0])
    assert torch.equal(new.spacing, G[f"{run}.spacing"]) and torch.equal(new.euclid, G[f"{run}.euclid"])
    if run == "pdf_top_jitter":
        # u rounds to exactly 1.0f in the last bin: searchsorted runs past the cdf and the bin is the last edge
        nb = meta["pdf_num_samples"] + 1
        u = torch.linspace(0.0, 1.0 - 1.0 / nb, nb)[-1] + u_rand[:, -1] / nb
        assert bool((u == 1.0).all())
        assert bool((inds[:, -1] == kw["S"] + 1).all())
        assert torch.equal(new.spacing[:, -1], base.spacing[:, -1])


def test_neus_sampler_train(golden, case):
    G, meta = golden
    spec, kw, o, d, cam, nears, fars, oracle = case
    t_rand, *u_rands = train_draws(G, meta, "neus")
    trace = []
    nb = samplers.neus_sampler(nears, fars, lambda s: oracle.get_sdf(o, d, s), t_rand=t_rand, u_rands=u_rands, trace=trace)
    assert torch.equal(torch.stack([t["inds"] for t in trace]), G["neus.inds"])
    close(nb.spacing, G["neus.spacing"], 1e-6)
    close(nb.euclid, G["neus.euclid"], 4e-6)


def test_error_bounded_sampler_train(golden, case):
    G, meta = golden
    spec, kw, o, d, cam, nears, fars, oracle = case
    draws = train_draws(G, meta, "error_bounded")
    fns = [x["fn"] for x in meta["draws"]["error_bounded"]]
    k = fns.index("randint")
    t_rand, u_rands, idx, t_extra = draws[0], draws[1:k], draws[k], draws[k + 1]
    assert fns == ["rand"] * k + ["randint", "rand"] and len(u_rands) == 5       # the golden runs all max_total_iters iterations
    eb, pts = samplers.error_bounded_sampler(nears, fars, lambda s: oracle.get_sdf(o, d, s), torch.tensor([cases.TRAIN_SAMPLER_BETA0]),
                                             t_rand=t_rand, u_rands=u_rands, t_rand_extra=t_extra, eikonal_idx=idx, origins=o, directions=d)
    assert eb.spacing.shape == G["error_bounded.spacing"].shape
    close(eb.spacing, G["error_bounded.spacing"], 1e-6)
    close(eb.euclid, G["error_bounded.euclid"], 4e-6)
    close(pts, G["error_bounded.eikonal_points"], 4e-6)


def test_unisurf_sampler_train(golden, case):
    G, meta = golden
    spec, kw, o, d, cam, nears, fars, oracle = case
    draws = train_draws(G, meta, "unisurf")
    shapes = [tuple(x["shape"]) for x in meta["draws"]["unisurf"]]
    assert (1024, 3) not in shapes                      # the golden's rays do hit the surface: no random surface points
    t_march, u_imp, t_out, t_int = draws
    ub, surf, mask = samplers.unisurf_sampler(o, d, nears, fars, lambda s: oracle.get_sdf(o, d, s), t_rand_march=t_march, u_rand_importance=u_imp,
                                              t_rand_outside=t_out, t_rand_interval=t_int)
    assert bool(mask.any())
    close(ub.euclid, G["unisurf.euclid"], 4e-6)
    close(surf, G["unisurf.surface_points"], 1e-5)


@pytest.mark.parametrize("anneal", [1.0, 0.5])
def test_proposal_sampler_train(golden, case, anneal):
    G, meta = golden
    spec, kw, o, d, cam, nears, fars, oracle = case
    run = f"proposal_anneal{anneal:g}"
    t_rand, *u_rands = train_draws(G, meta, run)
    dens = [lambda p, i=i: cases.proposal_density(p, i)[..., 0] for i in range(2)]
    ob, owl, obl = samplers.proposal_sampler(o, d, nears, fars, dens, (256, 96), 48, anneal=anneal, t_rand=t_rand, u_rands=u_rands)
    for i in range(2):
        assert torch.equal(obl[i].spacing, G[f"{run}.level{i}.spacing"])
        assert torch.equal(owl[i], G[f"{run}.weights{i}"])
    assert torch.equal(ob.spacing, G[f"{run}.spacing"]) and torch.equal(ob.euclid, G[f"{run}.euclid"])



def test_volsdf_dstar_heron_branch_is_never_nan():
    """The d* of get_dstar (ray_samplers.py:704-726) in fp32, on near-degenerate triangles of every orientation and magnitude: the Heron
    branch is only taken when neither squared test fires and b + c - a > 0, and there the rounded area is never negative.  So a NaN d*
    needs a NaN input (samplers.cu relies on this: see the comment at kVolsdfMaxS)."""
    g = torch.Generator().manual_seed(0)
    n = 1 << 19
    nudge = lambda x, k: x + k * (torch.nextafter(x, torch.tensor(float("inf"))) - x)  # noqa: E731  (k ulps up)
    for scale in (1e-20, 1e-6, 1.0, 1e6, 1e18):
        a = scale * (0.01 + torch.rand(n, generator=g))                  # the section length
        p = a * torch.rand(n, generator=g) ** 3
        k = torch.randint(-4, 5, (n,), generator=g).float()
        for b, c in ((p, nudge(a - p, k)),                                # b + c ~ a: the flat triangle on the section
                     (p, nudge(a + p, k)),                                # c ~ a + b
                     (nudge(a + p, k), p),                                # b ~ a + c
                     (scale * torch.rand(n, generator=g) * 1e3, None)):   # |b - c| ~ a at large |sdf|
            if c is None:
                c = nudge(b + a * torch.rand(n, generator=g), k)
            sdf = torch.stack([b, c], -1)                                 # same sign: the mask keeps d*
            deltas = torch.stack([a, a], -1)
            d_star = samplers.volsdf_dstar(sdf, deltas)
            assert not bool(torch.isnan(d_star).any())
