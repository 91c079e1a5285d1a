"""CPU-only: oracle/losses.py (the restatement of the interlevel losses) against the reference's goldens and, where the reference tree
is present, against the reference itself; the argument checks of sdfstudio_b200.losses and of sdfb200_interlevel_loss, none of which
needs a GPU."""
import json
import os
import types

import pytest
import torch

from oracle import losses as olosses
from oracle.ref_import import reference_available

from helpers import GOLDEN_DIR, load_golden


def golden_cases():
    with open(os.path.join(GOLDEN_DIR, "losses.json")) as f:
        return json.load(f)["cases"]


def levels_of(G, name, dtype=torch.float32):
    """[(cp0, wp0), (cp1, wp1), (c, w)] of a golden case."""
    return [(G[f"{name}.{e}"].to(dtype), G[f"{name}.{w}"].to(dtype)) for e, w in (("cp0", "wp0"), ("cp1", "wp1"), ("c", "w"))]


def oracle_loss_and_grads(levels, form):
    leaves = [levels[0][1].clone().requires_grad_(True), levels[1][1].clone().requires_grad_(True)]
    fn = olosses.interlevel_loss if form == "outer" else olosses.interlevel_loss_zip
    loss = fn([levels[0][0], levels[1][0], levels[2][0]], leaves + [levels[2][1]])
    return (loss.detach(), *torch.autograd.grad(loss, leaves))


@pytest.mark.parametrize("form", ["outer", "zip"])
@pytest.mark.parametrize("name", golden_cases())
def test_oracle_reproduces_reference_golden(name, form):
    G = load_golden("losses")
    loss, g0, g1 = oracle_loss_and_grads(levels_of(G, name), form)
    # the same torch-CPU ops in the same order: equal to the last bits (one ulp of slack for the summation order of mean)
    torch.testing.assert_close(loss, G[f"{name}.{form}"], rtol=2e-7, atol=0)
    torch.testing.assert_close(g0, G[f"{name}.{form}_g0"], rtol=1e-6, atol=1e-12)
    torch.testing.assert_close(g1, G[f"{name}.{form}_g1"], rtol=1e-6, atol=1e-12)


def test_goldens_are_not_trivial():
    G = load_golden("losses")
    for name in ("sampler_anneal1", "sampler_anneal0.5", "proposal_edges_on_knots", "knots_past_the_ends"):
        for form in ("outer", "zip"):
            assert float(G[f"{name}.{form}"]) > 1e-4
            assert float(G[f"{name}.{form}_g0"].abs().max()) > 0 and float(G[f"{name}.{form}_g1"].abs().max()) > 0
    c = G["knots_past_the_ends.c"]
    assert float((c - 0.03).min()) < 0 and float((c + 0.03).max()) > 1


def _as_samples(edges):
    return types.SimpleNamespace(spacing_starts=edges[:, :-1, None], spacing_ends=edges[:, 1:, None])


@pytest.mark.skipif(not reference_available(), reason="needs the reference tree")
@pytest.mark.parametrize("sizes", [(48, 256, 96), (128, 64, 7), (1, 1, 1)])
def test_oracle_matches_reference_on_fresh_inputs(sizes):
    from oracle.make_golden_losses import _hist
    from oracle.ref_import import install_shims

    install_shims()
    from nerfstudio.model_components import losses as ref

    sf, s0, s1 = sizes
    g = torch.Generator().manual_seed(sum(sizes))
    R = 19
    (c, w), (cp0, wp0), (cp1, wp1) = _hist(R, sf, g), _hist(R, s0, g), _hist(R, s1, g)
    for form, rfn in (("outer", ref.interlevel_loss), ("zip", ref.interlevel_loss_zip)):
        leaves = [wp0.clone().requires_grad_(True), wp1.clone().requires_grad_(True)]
        rl = rfn([leaves[0][..., None], leaves[1][..., None], w[..., None]], [_as_samples(cp0), _as_samples(cp1), _as_samples(c)])
        rg = torch.autograd.grad(rl, leaves)
        ol, og0, og1 = oracle_loss_and_grads([(cp0, wp0), (cp1, wp1), (c, w)], form)
        torch.testing.assert_close(ol, rl.detach(), rtol=2e-7, atol=0)
        torch.testing.assert_close(og0, rg[0], rtol=1e-6, atol=1e-12)
        torch.testing.assert_close(og1, rg[1], rtol=1e-6, atol=1e-12)


def test_oracle_is_dtype_generic():
    G = load_golden("losses")
    l32, *_ = oracle_loss_and_grads(levels_of(G, "sampler_anneal1"), "zip")
    l64, g0, _ = oracle_loss_and_grads(levels_of(G, "sampler_anneal1", torch.float64), "zip")
    assert l64.dtype == torch.float64 and g0.dtype == torch.float64
    assert abs(float(l32) - float(l64)) < 1e-4 * float(l64)


# ---- sdfstudio_b200.losses: shape and device validation happens before any library call ---------------------------------------------
def _lists(R=(5, 5, 5), S=(8, 6, 4), bins_extra=(1, 1, 1)):
    weights = [torch.rand(r, s, 1) for r, s in zip(R, S)]
    samples = [_as_samples(torch.sort(torch.rand(r, s + e), -1)[0]) for r, s, e in zip(R, S, bins_extra)]
    return weights, samples


@pytest.mark.parametrize("fn", ["interlevel_loss", "interlevel_loss_zip"])
def test_losses_validate_shapes_and_device(fn):
    import sdfstudio_b200 as sb

    f = getattr(sb, fn)
    assert f is getattr(sb.losses, fn)
    with pytest.raises(ValueError, match="bin edges"):
        f(*_lists(bins_extra=(1, 2, 1)))                       # weights [R, 6, 1] against 8 edges
    with pytest.raises(ValueError, match="rays"):
        f(*_lists(R=(5, 4, 5)))
    with pytest.raises(ValueError, match="length"):
        w, s = _lists()
        f(w[:2], s)
    with pytest.raises(ValueError):
        w, s = _lists()
        f([x[..., 0] for x in w], s)                           # weights without the trailing axis
    with pytest.raises(RuntimeError, match="CUDA only"):
        f(*_lists())                                           # consistent shapes, CPU tensors: there is no CPU path


def test_ray_samples_to_sdist_reads_both_kinds_of_samples():
    import sdfstudio_b200 as sb

    edges = torch.sort(torch.rand(3, 9), -1)[0]
    assert torch.equal(sb.ray_samples_to_sdist(_as_samples(edges)), edges)


# ---- sdfb200_interlevel_loss: bad arguments come back as error codes before any launch ----------------------------------------------
@pytest.mark.skipif(torch.cuda.is_available(), reason="the calls get sentinel device pointers, which a call that is not rejected would launch on")
def test_interlevel_loss_entry_point_rejects_bad_arguments():
    from sdfstudio_b200 import _lib

    lib = _lib.load()
    P = dict(c=0x10000, w=0x20000, cp=0x30000, wp=0x40000, per_ray=0x50000, loss=0x60000, grad=0x70000)

    def call(sf=48, sp=96, R=16, form=_lib.INTERLEVEL_ZIP, r=0.03, **ptrs):
        p = {**P, **ptrs}
        return lib.sdfb200_interlevel_loss(p["c"], p["w"], sf, p["cp"], p["wp"], sp, R, form, r, p["per_ray"], p["loss"], p["grad"], None)

    n0 = _lib.launch_count()
    for required in ("c", "w", "cp", "wp", "per_ray"):
        assert call(**{required: None}) == -1, required
        assert b"NULL" in lib.sdfb200_last_error_string()
    for form in (_lib.INTERLEVEL_OUTER, _lib.INTERLEVEL_ZIP):
        assert call(sf=0, form=form) == -1 and call(sp=0, form=form) == -1
        assert call(sf=1025, form=form) == -1 and b"1024" in lib.sdfb200_last_error_string()
        assert call(sp=1025, form=form) == -1 and b"1024" in lib.sdfb200_last_error_string()
        assert call(R=-1, form=form) == -1
    assert call(form=2) == -1 and call(form=-1) == -1
    assert call(r=0.0) == -1 and call(r=-0.03) == -1 and b"blur_radius" in lib.sdfb200_last_error_string()
    assert call(r=float("nan")) == -1
    assert call(r=0.0, form=_lib.INTERLEVEL_OUTER, R=0) == 0                    # the outer form does not read the radius
    assert call(R=0, c=None, per_ray=None) == 0                                  # an empty batch returns before the pointer checks
    assert call(R=0, sf=2000) == -1                                              # but not before the size checks
    assert _lib.launch_count() == n0
