"""-m gpu: the interlevel losses (sdfstudio_b200.losses, sdfb200_interlevel_loss) against the reference's goldens and the fp64 oracle
(oracle/losses.py): loss and gradient with respect to the proposal weights, for both forms, at the presets' shapes and at the edges.

Where a quantity is compared with fp64 the bound is the fp32 oracle's own distance from fp64 on the same inputs times a small factor
(helpers.assert_within_noise): both losses divide a clipped difference of prefix sums by a weight plus 1e-7 / 1e-5, so a fixed relative
bound would be unattainable by any fp32 implementation where the weights are small."""
import json
import os
import types

import numpy as np
import pytest
import torch

from oracle import cases, samplers
from oracle import density as odensity
from oracle import losses as olosses

from helpers import GOLDEN_DIR, assert_within_noise, load_golden, make_bundle

pytestmark = pytest.mark.gpu
RADII = olosses.ZIP_BLUR_RADII
FORMS = ["outer", "zip"]


@pytest.fixture(autouse=True)
def keep_global_rng():
    """The end-to-end tests seed torch's global generators and the samplers draw from them: put both back, so that the tests that run
    after this file see the random streams they see without it."""
    with torch.random.fork_rng(devices=[torch.cuda.current_device()]):
        yield


def golden_cases():
    with open(os.path.join(GOLDEN_DIR, "losses.json")) as f:
        return json.load(f)["cases"]


def as_samples(edges):
    """What the loss functions read of a RaySamples: spacing_starts / spacing_ends [R, S, 1] as slices of one edge buffer."""
    return types.SimpleNamespace(spacing_starts=edges[:, :-1, None], spacing_ends=edges[:, 1:, None])


def histogram(R, S, g, lo=0.0, hi=1.0, power=3.0):
    """Random strictly ascending edges on [lo, hi] and weights that sum to at most 1 (fp32, CPU)."""
    widths = torch.rand(R, S, generator=g) ** 2 + 0.02           # no bin of zero width: the Zip-NeRF form divides by the widths
    edges = torch.cat([torch.zeros(R, 1), torch.cumsum(widths, -1) / widths.sum(-1, keepdim=True)], -1) * (hi - lo) + lo
    w = torch.rand(R, S, generator=g) ** power
    return edges.contiguous(), (w / w.sum(-1, keepdim=True).clamp_min(1e-30) * torch.rand(R, 1, generator=g)).contiguous()


def product(levels, form):
    """sdfstudio_b200's loss over [(cp, wp), ..., (c, w)] (CPU tensors) -> (loss, [d loss / d wp per proposal level])."""
    import sdfstudio_b200 as sb

    leaves = [wp.cuda().requires_grad_(True) for _, wp in levels[:-1]]
    weights = [x[..., None] for x in leaves] + [levels[-1][1].cuda()[..., None]]
    fn = sb.interlevel_loss if form == "outer" else sb.interlevel_loss_zip
    loss = fn(weights, [as_samples(e.cuda()) for e, _ in levels])
    assert loss.shape == () and loss.is_cuda and loss.dtype == torch.float32
    return loss.detach(), list(torch.autograd.grad(loss, leaves, allow_unused=True))


def oracle(levels, form, dtype):
    leaves = [wp.to(dtype).requires_grad_(True) for _, wp in levels[:-1]]
    fn = olosses.interlevel_loss if form == "outer" else olosses.interlevel_loss_zip
    loss = fn([e.to(dtype) for e, _ in levels], leaves + [levels[-1][1].to(dtype)])
    return loss.detach(), list(torch.autograd.grad(loss, leaves))


def check_against_fp64(levels, form, what, ref32=None):
    """loss and gradients within 4x the fp32 oracle's (or the reference golden's) own error against fp64; the floor is 4e-6 of the
    largest exact value (a few fp32 roundings)."""
    loss, grads = product(levels, form)
    l32, g32 = ref32 if ref32 is not None else oracle(levels, form, torch.float32)
    l64, g64 = oracle(levels, form, torch.float64)
    assert_within_noise(loss, l32, l64, f"{what} {form} loss", floor=max(1e-12, 4e-6 * abs(float(l64))))
    for k, (g, a, b) in enumerate(zip(grads, g32, g64)):
        assert g.shape == b.shape
        assert_within_noise(g, a, b, f"{what} {form} d/dwp level {k}", floor=max(1e-12, 4e-6 * float(b.abs().max())))
    return loss, grads


# ----------------------------------------------------------------------------------------------------------------
# 1. the reference's goldens: sampler-made histograms (piecewise spacing, annealed sampling) and the hand-built edges
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("name", golden_cases())
def test_golden_parity(name, form):
    G = load_golden("losses")
    levels = [(G[f"{name}.cp0"], G[f"{name}.wp0"]), (G[f"{name}.cp1"], G[f"{name}.wp1"]), (G[f"{name}.c"], G[f"{name}.w"])]
    ref = (G[f"{name}.{form}"], [G[f"{name}.{form}_g0"], G[f"{name}.{form}_g1"]])
    loss, grads = check_against_fp64(levels, form, name, ref32=ref)
    if name == "zero_fine_weights":
        assert float(loss) == 0.0 and all(float(g.abs().max()) == 0.0 for g in grads)


# ----------------------------------------------------------------------------------------------------------------
# 2. shapes: the presets' (fine 48 / 128 / 96, proposals 256 / 96 / 64 / 128) and the ones they do not use
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("R", [0, 1, 37, 4096, 8192])
@pytest.mark.parametrize("sf,sp", [(48, 256), (48, 96), (128, 64), (96, 128), (33, 7), (1, 1), (1024, 1024)])
def test_shapes(sf, sp, R, form):
    g = torch.Generator().manual_seed(1000 * sf + sp + R)
    levels = [histogram(R, sp, g), histogram(R, sf, g)]
    if R == 0:
        import sdfstudio_b200 as sb

        n0 = sb._lib.launch_count()
        loss, (grad,) = product(levels, form)
        assert bool(torch.isnan(loss)) and grad.shape == (0, sp)                 # torch.mean over no elements, as in the reference
        assert sb._lib.launch_count() == n0
        return
    check_against_fp64(levels, form, f"Sf={sf} Sp={sp} R={R}")


def test_sizes_above_1024_are_refused():
    import sdfstudio_b200 as sb

    g = torch.Generator().manual_seed(3)
    n0 = sb._lib.launch_count()
    for sf, sp in ((1025, 8), (8, 1025)):
        for form in FORMS:
            with pytest.raises(sb._lib.Sdfb200Error, match="1024"):
                product([histogram(2, sp, g), histogram(2, sf, g)], form)
    assert sb._lib.launch_count() == n0


def test_third_proposal_level_is_not_visited_by_the_zip_form():
    g = torch.Generator().manual_seed(4)
    h = [histogram(9, s, g) for s in (64, 32, 16, 24)]
    loss3, grads3 = product(h, "zip")
    loss2, grads2 = product([h[0], h[1], h[3]], "zip")
    assert torch.equal(loss3, loss2) and torch.equal(grads3[0], grads2[0]) and torch.equal(grads3[1], grads2[1]) and grads3[2] is None
    # the outer form visits every level
    assert float(product(h, "outer")[0]) > float(product([h[0], h[1], h[3]], "outer")[0])
    # and one proposal level is blurred with the first radius only
    l1, _ = product([h[0], h[3]], "zip")
    want = olosses.interlevel_zip(h[3][0].double(), h[3][1].double(), h[0][0].double(), h[0][1].double(), RADII[0])
    assert abs(float(l1) - float(want)) < 1e-4 * float(want)


# ----------------------------------------------------------------------------------------------------------------
# 3. a fine bin of zero width
# ----------------------------------------------------------------------------------------------------------------
def test_zero_width_fine_bin():
    """The Zip-NeRF form divides the fine weights by the bin widths: a bin of zero width that carries weight makes that ray's density
    inf, its blurred histogram NaN, and the mean NaN, in the reference and here (the kernel neither faults nor loops: its searches are
    bounded by the sample counts).  The other rays' gradients stay finite.  The outer-measure form never divides by a width."""
    g = torch.Generator().manual_seed(5)
    R = 8
    (c, w), p0, p1 = histogram(R, 20, g), histogram(R, 32, g), histogram(R, 12, g)
    c[2, 7] = c[2, 8]
    w[2, 7] = 0.05
    levels = [p0, p1, (c, w)]
    check_against_fp64(levels, "outer", "zero-width fine bin")
    loss, grads = product(levels, "zip")
    l32, g32 = oracle(levels, "zip", torch.float32)
    assert not bool(torch.isfinite(loss)) and not bool(torch.isfinite(l32))
    others = [r for r in range(R) if r != 2]
    for gk, ok in zip(grads, g32):
        assert bool(torch.isfinite(gk[others]).all())
        torch.testing.assert_close(gk[others].cpu(), ok[others], rtol=1e-3, atol=1e-6 * float(ok[others].abs().max()))


# ----------------------------------------------------------------------------------------------------------------
# 4. determinism, launches, no host synchronisation
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", FORMS)
def test_same_inputs_same_bits(form):
    g = torch.Generator().manual_seed(6)
    levels = [histogram(4096, 256, g), histogram(4096, 96, g), histogram(4096, 48, g)]
    a, ga = product(levels, form)
    b, gb = product(levels, form)
    assert torch.equal(a, b) and all(torch.equal(x, y) for x, y in zip(ga, gb))


@pytest.mark.parametrize("form", FORMS)
def test_no_host_sync_and_two_launches_per_level(form):
    """Forward + backward of two proposal levels: 4 launches of this library (per level the loss kernel, which also writes the
    gradient, and the fixed-order mean; the backward is one ATen scale), and nothing that waits for the device."""
    import sdfstudio_b200 as sb

    g = torch.Generator().manual_seed(7)
    levels = [histogram(4096, 256, g), histogram(4096, 96, g), histogram(4096, 48, g)]
    leaves = [wp.cuda().requires_grad_(True) for _, wp in levels[:-1]]
    weights = [x[..., None] for x in leaves] + [levels[-1][1].cuda()[..., None]]
    rs = [as_samples(e.cuda()) for e, _ in levels]
    fn = sb.interlevel_loss if form == "outer" else sb.interlevel_loss_zip
    fn(weights, rs).backward()                                   # warm-up: module load, allocator
    torch.cuda.synchronize()
    n0 = sb._lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = fn(weights, rs)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert sb._lib.launch_count() - n0 == 4
    assert bool(torch.isfinite(loss)) and all(bool(torch.isfinite(x.grad).all()) for x in leaves)


# ----------------------------------------------------------------------------------------------------------------
# 5. end to end: the loss trains the proposal networks through the sampler
# ----------------------------------------------------------------------------------------------------------------
AABB = torch.tensor([[-1.0, -1, -1], [1, 1, 1]])
MAX_RES = (64, 256)
E2E_RAYS = 64


def proposal_setup(contraction):
    import sdfstudio_b200 as sb

    g = torch.Generator().manual_seed(9)
    nets = []
    for max_res in MAX_RES:
        sd = sb.SceneContraction(order=float("inf")) if contraction else None
        f = sb.HashMLPDensityField(AABB, num_layers=2, hidden_dim=16, spatial_distortion=sd, num_levels=5, max_res=max_res, log2_hashmap_size=17).cuda().train()
        with torch.no_grad():
            nb = f.mlp_base
            nb.params[nb.n_net:] = ((torch.rand(nb.n_grid, generator=g) * 2 - 1) * 0.5).cuda()
        nets.append(f)
    o, d, cam = cases.synthetic_rays(E2E_RAYS, 77)
    nears, fars = torch.full((E2E_RAYS, 1), 0.5), torch.full((E2E_RAYS, 1), 4.5)
    fine_w = torch.rand(E2E_RAYS, 48, generator=g) ** 3
    fine_w = fine_w / fine_w.sum(-1, keepdim=True) * 0.9
    sampler = sb.ProposalNetworkSampler(num_proposal_samples_per_ray=(256, 96), num_nerf_samples_per_ray=48, num_proposal_network_iterations=2).train()
    return nets, sampler, (o, d, cam, nears, fars), fine_w


def product_step(nets, sampler, rays, fine_w, form):
    import sdfstudio_b200 as sb

    rs, weights_list, rs_list = sampler(make_bundle(*rays), density_fns=[n.density_fn for n in nets])
    assert all(w.requires_grad for w in weights_list)
    fn = sb.interlevel_loss if form == "outer" else sb.interlevel_loss_zip
    return fn(weights_list + [fine_w.cuda()[..., None]], rs_list + [rs])


def oracle_chain(nets, rays, fine_w, form, contraction, jitter, dtype):
    """The same step in torch-CPU at `dtype`: oracle sampler on the recorded jitter (each level resampled from detached weights, as
    PDFSampler does), oracle density fields on parameter copies that require grad, oracle loss.  -> (loss, [d loss / d params])."""
    o, d, _, nears, fars = (t.to(dtype) if t.is_floating_point() else t for t in rays)
    t_rand, *u_rands = [j.to(dtype) for j in jitter]
    params = [n.mlp_base.params.detach().cpu().to(dtype).requires_grad_(True) for n in nets]
    bins_list, weights_list, cur, weights = [], [], None, None
    for i, ns in enumerate((256, 96, 48)):
        cur = samplers.spaced_sampler(nears, fars, ns, "piecewise", t_rand) if i == 0 else \
            samplers.pdf_sampler(cur, weights.detach(), ns, histogram_padding=0.01, u_rand=u_rands[i - 1])
        bins_list.append(cur.spacing)
        if i < 2:
            nb = nets[i].mlp_base
            gf = float(np.exp((np.log(MAX_RES[i]) - np.log(16)) / 4))
            dens, _ = odensity.density_field(samplers.frustum_centres(o, d, cur), params[i][: nb.n_net], params[i][nb.n_net:], 16, 1, 5, 2, 17, 16, gf,
                                             aabb=None if contraction else AABB.to(dtype), contraction="linf" if contraction else None)
            weights, _ = samplers.weights_from_density(cur.deltas, dens[..., 0])
            weights_list.append(weights)
    fn = olosses.interlevel_loss if form == "outer" else olosses.interlevel_loss_zip
    loss = fn(bins_list, weights_list + [fine_w.to(dtype)])
    return loss.detach(), torch.autograd.grad(loss, params)


@pytest.fixture
def rand_log(monkeypatch):
    log = []
    rand = torch.rand

    def rec(*a, **k):
        t = rand(*a, **k)
        log.append(t.detach().cpu().clone())
        return t

    monkeypatch.setattr(torch, "rand", rec)
    return log


@pytest.mark.parametrize("form,contraction", [("zip", False), ("outer", True)], ids=["neus-facto", "bakedsdf"])
def test_loss_trains_both_proposal_networks(rand_log, form, contraction):
    """interlevel_loss_zip on a neus-facto sampler, interlevel_loss on bakedsdf's (L-inf scene contraction): mlp_base.params.grad of BOTH
    networks is finite, non-zero in the MLP section and in the table section, and agrees with the oracle chain in fp64 on the same jitter,
    judged like the level weights in test_gpu_samplers_train.py (level 1 sits on PDF-drawn positions: factor 6 of the fp32 chain's own
    error; the floor is 1e-3 of the largest exact entry)."""
    nets, sampler, rays, fine_w = proposal_setup(contraction)
    rand_log.clear()
    torch.manual_seed(11)
    loss = product_step(nets, sampler, rays, fine_w, form)
    jitter = list(rand_log)
    assert [tuple(j.shape) for j in jitter] == [(E2E_RAYS, 257), (E2E_RAYS, 97), (E2E_RAYS, 49)]
    loss.backward()
    l32, g32 = oracle_chain(nets, rays, fine_w, form, contraction, jitter, torch.float32)
    l64, g64 = oracle_chain(nets, rays, fine_w, form, contraction, jitter, torch.float64)
    assert_within_noise(loss, l32, l64, f"{form} loss", factor=6.0, floor=1e-4 * float(l64))
    for k, net in enumerate(nets):
        nb = net.mlp_base
        grad = nb.params.grad
        assert grad is not None and bool(torch.isfinite(grad).all())
        for what, sl in (("MLP", slice(0, nb.n_net)), ("table", slice(nb.n_net, None))):
            assert float(grad[sl].abs().max()) > 0.0, f"network {k}: no gradient reached the {what} section"
            assert_within_noise(grad[sl], g32[k][sl], g64[k][sl], f"{form} network {k} {what} gradient", factor=6.0,
                                floor=1e-3 * float(g64[k][sl].abs().max()))


def test_ten_optimiser_steps_reduce_the_loss():
    nets, sampler, rays, fine_w = proposal_setup(False)
    opt = torch.optim.Adam([n.mlp_base.params for n in nets], lr=1e-3)
    history = []
    for _ in range(11):
        torch.manual_seed(11)                                     # the same jitter every step: one fixed objective
        loss = product_step(nets, sampler, rays, fine_w, "zip")
        history.append(float(loss))
        opt.zero_grad()
        loss.backward()
        opt.step()
    assert history[-1] < history[0], history
