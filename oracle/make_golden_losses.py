"""TEST INFRASTRUCTURE -- mints tests/golden/losses.{npz,json}: the UNMODIFIED reference interlevel losses (interlevel_loss and
interlevel_loss_zip of nerfstudio/model_components/losses.py) and their autograd gradients with respect to the proposal weights.

Container-only (needs the reference, via oracle/ref_import.py).  Usage:  python -m oracle.make_golden_losses

Every case is two proposal levels and a final level, (edges [R,S+1], weights [R,S]) each, stored with the two losses and the four
gradients.  The `sampler_*` cases come from the reference's ProposalNetworkSampler((256, 96) -> 48) in training mode over the
analytic proposal densities of cases.proposal_density (piecewise initial spacing; `anneal0.5` anneals the weights the PDF sampler
draws from), with seeded final weights.  The rest are hand-built edges, see edge_cases()."""
import json
import os
import types

import numpy as np
import torch

from . import cases
from .make_golden import GOLDEN_DIR, make_bundle, npy
from .make_golden_samplers_train import train_inputs
from .ref_import import install_shims, ref_modules

SEED = 20261016
RADII = (0.03, 0.003)


def _hist(R, S, g, lo=0.0, hi=1.0, power=3.0):
    """Random ascending edges on [lo, hi] (both ends included) and weights that sum to at most 1."""
    inner = torch.sort(torch.rand(R, S - 1, generator=g), -1)[0] if S > 1 else torch.zeros(R, 0)
    edges = torch.cat([torch.zeros(R, 1), inner, torch.ones(R, 1)], -1) * (hi - lo) + lo
    w = torch.rand(R, S, generator=g) ** power
    return edges.contiguous(), (w / w.sum(-1, keepdim=True) * torch.rand(R, 1, generator=g)).contiguous()


def edge_cases():
    """name -> [(cp0, wp0), (cp1, wp1), (c, w)], fp32 CPU."""
    g = torch.Generator().manual_seed(SEED)
    R = 6
    out = {}
    c, w = _hist(R, 24, g)
    p0, p1 = _hist(R, 40, g), _hist(R, 17, g)
    # the proposal edges ARE the fine edges: every search hits a tie
    out["identical_edges"] = [(c.clone(), _hist(R, 24, g)[1]), (c.clone(), w.clone() * 0.5), (c, w)]
    # the whole fine histogram inside one proposal bin, and the whole proposal histogram inside one fine bin
    ci, wi = _hist(R, 16, g, 0.41, 0.57)
    wide = torch.tensor([0.0, 0.2, 0.4, 0.6, 0.8, 1.0]).expand(R, -1).contiguous()
    out["fine_inside_one_proposal_bin"] = [(wide, _hist(R, 5, g)[1]), (torch.tensor([0.0, 0.4, 0.6, 1.0]).expand(R, -1).contiguous(), _hist(R, 3, g)[1]), (ci, wi)]
    cw = torch.tensor([0.0, 0.3, 0.7, 1.0]).expand(R, -1).contiguous()
    out["proposal_inside_one_fine_bin"] = [_hist(R, 12, g, 0.35, 0.65), _hist(R, 7, g, 0.45, 0.46), (cw, _hist(R, 3, g)[1])]
    out["zero_proposal_weights"] = [(p0[0], torch.zeros_like(p0[1])), (p1[0], torch.zeros_like(p1[1])), (c, w)]
    out["zero_fine_weights"] = [p0, p1, (c, torch.zeros_like(w))]
    # fine edges within the blur radius of 0 and 1: knots below 0 and above 1, proposal edges between them
    ce = torch.tensor([0.0, 0.001, 0.002, 0.02, 0.029, 0.5, 0.971, 0.98, 0.998, 0.999, 1.0]).expand(R, -1).contiguous()
    out["knots_past_the_ends"] = [p0, p1, (ce, _hist(R, 10, g)[1])]
    # proposal edges exactly ON the blurred knots c -+ r of their level (the side="right" tie of the resampling search)
    levels = []
    for r in RADII:
        knots = torch.sort(torch.cat([c - r, c + r], -1), -1)[0]
        levels.append((knots.contiguous(), _hist(R, knots.shape[1] - 1, g)[1]))
    out["proposal_edges_on_knots"] = levels + [(c, w)]
    # one sample per level
    out["single_samples"] = [_hist(R, 1, g), _hist(R, 1, g, 0.2, 0.9), _hist(R, 1, g, 0.1, 0.8)]
    # weights annealed by pow, as the sampler anneals what it draws from
    out["annealed_weights"] = [(p0[0], p0[1] ** 0.5), (p1[0], p1[1] ** 0.25), (c, w ** 0.5)]
    return out


def _as_samples(edges):
    return types.SimpleNamespace(spacing_starts=edges[:, :-1, None], spacing_ends=edges[:, 1:, None])


def sampler_cases(R):
    RS = R.ray_samplers
    spec, kw, o, d, cam, nears, fars, _ = train_inputs()
    rb = make_bundle(R, o, d, cam, nears, fars)
    dens = [lambda p, i=i: cases.proposal_density(p, i) for i in range(2)]
    g = torch.Generator().manual_seed(SEED + 1)
    out = {}
    torch.manual_seed(SEED)
    for anneal in (1.0, 0.5):
        ps = RS.ProposalNetworkSampler(num_proposal_samples_per_ray=(256, 96), num_nerf_samples_per_ray=48, num_proposal_network_iterations=2).train()
        ps.set_anneal(anneal)
        rs, wl, rsl = ps(rb, density_fns=dens)
        sdist = lambda s: torch.cat([s.spacing_starts[..., 0], s.spacing_ends[:, -1:, 0]], -1).contiguous()   # noqa: E731
        w = torch.rand(o.shape[0], 48, generator=g) ** 3
        w = w / w.sum(-1, keepdim=True) * torch.rand(o.shape[0], 1, generator=g)
        out[f"sampler_anneal{anneal:g}"] = [(sdist(rsl[0]), wl[0][..., 0].contiguous()), (sdist(rsl[1]), wl[1][..., 0].contiguous()), (sdist(rs), w)]
    return out


def mint():
    R = ref_modules()
    install_shims()
    from nerfstudio.model_components import losses as ref_losses

    out, names = {}, []
    for name, levels in {**sampler_cases(R), **edge_cases()}.items():
        names.append(name)
        (cp0, wp0), (cp1, wp1), (c, w) = levels
        for k, v in dict(cp0=cp0, wp0=wp0, cp1=cp1, wp1=wp1, c=c, w=w).items():
            out[f"{name}.{k}"] = npy(v)
        for form, fn in (("outer", ref_losses.interlevel_loss), ("zip", ref_losses.interlevel_loss_zip)):
            leaves = [wp0.clone().requires_grad_(True), wp1.clone().requires_grad_(True)]
            loss = fn([leaves[0][..., None], leaves[1][..., None], w[..., None]], [_as_samples(cp0), _as_samples(cp1), _as_samples(c)])
            grads = torch.autograd.grad(loss, leaves)
            out[f"{name}.{form}"] = npy(loss.detach())
            out[f"{name}.{form}_g0"], out[f"{name}.{form}_g1"] = npy(grads[0]), npy(grads[1])
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    path = os.path.join(GOLDEN_DIR, "losses.npz")
    np.savez_compressed(path, **out)
    with open(os.path.join(GOLDEN_DIR, "losses.json"), "w") as f:
        json.dump({"seed": SEED, "radii": list(RADII), "cases": names}, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"wrote {path}: {os.path.getsize(path) / 1024:.0f} KiB, {len(names)} cases")


if __name__ == "__main__":
    torch.set_num_threads(8)
    mint()
