"""TEST INFRASTRUCTURE -- mints tests/golden/samplers_train.{npz,json}: the UNMODIFIED reference samplers in TRAINING mode.

Container-only (needs the reference, via oracle/ref_import.py).  Usage:  python -m oracle.make_golden_samplers_train

Training mode draws its stratified jitter with ``torch.rand`` (and VolSDF's eikonal points with ``torch.randint``).  While the
reference runs, both are wrapped to record every draw in order.  The fixture stores, per run, the drawn tensors, their
(function, shape, dtype) in draw order (json) and the reference's outputs, so the oracle can be fed the very same jitter.
Rays and field parameters are regenerated from the seed of ``cases.TRAIN_SAMPLER_CASE`` as in make_golden.py.
"""
import contextlib
import json
import os

import numpy as np
import torch

from . import cases
from .field import init_params
from .make_golden import GOLDEN_DIR, build_reference_field, make_bundle, npy
from .ref_import import ref_modules

SEED = 20261016
PDF_S_OUT = 24
TOP_JITTER = 1.0 - 2.0**-24   # the largest value torch.rand returns


@contextlib.contextmanager
def recording(log: list, inject=None):
    """Wraps torch.rand / torch.randint: every draw is appended to ``log`` as (fn, tensor).  ``inject(shape)``, if given,
    replaces the values torch.rand returns."""
    rand, randint = torch.rand, torch.randint

    def rec_rand(*a, **k):
        t = rand(*a, **k)
        if inject is not None:
            t = inject(t.shape).to(t.dtype)
        log.append(("rand", t.clone()))
        return t

    def rec_randint(*a, **k):
        t = randint(*a, **k)
        log.append(("randint", t.clone()))
        return t

    torch.rand, torch.randint = rec_rand, rec_randint
    try:
        yield log
    finally:
        torch.rand, torch.randint = rand, randint


@contextlib.contextmanager
def searchsorted_log(log: list):
    orig = torch.searchsorted

    def ss(*a, **k):
        r = orig(*a, **k)
        log.append(r.clone())
        return r

    torch.searchsorted = ss
    try:
        yield log
    finally:
        torch.searchsorted = orig


def bins_of(s):
    return (npy(torch.cat([s.spacing_starts[..., 0], s.spacing_ends[:, -1:, 0]], -1)),
            npy(torch.cat([s.frustums.starts[..., 0], s.frustums.ends[:, -1:, 0]], -1)))


def train_inputs():
    """(spec, kw, origins, directions, camera_indices, nears, fars) of the golden's rays, and the PDF test weights [n, S]."""
    spec, kw, o, d, cam, nears, fars = cases.case_inputs(cases.TRAIN_SAMPLER_CASE)
    n = cases.TRAIN_SAMPLER_RAYS
    o, d, cam, nears, fars = o[:n], d[:n], cam[:n], nears[:n], fars[:n]
    g = torch.Generator().manual_seed(kw["seed"] + 99)
    w = torch.rand(n, kw["S"], generator=g) ** 4
    w[0] = 0.0                                  # all-zero row: the eps padding path
    w[1] = 0.0
    w[1, kw["S"] // 2] = 1.0                    # one spike: a flat cdf with ties on both sides
    w[2] = torch.logspace(-30, 0, kw["S"])      # NaN-free, 30 decades of dynamic range
    return spec, kw, o, d, cam, nears, fars, w


def mint():
    R = ref_modules()
    RS = R.ray_samplers
    spec, kw, o, d, cam, nears, fars, pdf_w = train_inputs()
    params = init_params(spec, **cases.init_kwargs(kw))
    field = build_reference_field(R, spec, params, kw)
    rb = make_bundle(R, o, d, cam, nears, fars)
    S = kw["S"]
    out, runs = {}, {}
    torch.manual_seed(SEED)

    def run(name, fn, inject=None, log_inds=False):
        draws, inds = [], []
        with recording(draws, inject), (searchsorted_log(inds) if log_inds else contextlib.nullcontext()):
            res = fn()
        runs[name] = [{"fn": f, "shape": list(t.shape), "dtype": str(t.dtype).replace("torch.", "")} for f, t in draws]
        for k, (_, t) in enumerate(draws):
            out[f"{name}.draw{k}"] = npy(t)
        if log_inds:
            out[f"{name}.inds"] = np.stack([npy(i) for i in inds])
        return res

    def store(name, rs):
        out[f"{name}.spacing"], out[f"{name}.euclid"] = bins_of(rs)

    # ---- spaced samplers: every spacing, single and per-bin jitter -------------------------------------------------
    classes = {"uniform": RS.UniformSampler, "lindisp": RS.LinearDisparitySampler, "sqrt": RS.SqrtSampler, "log": RS.LogSampler,
               "piecewise": RS.UniformLinDispPiecewiseSampler}
    for kind, cls in classes.items():
        for single in (True, False):
            name = f"spaced_{kind}_{'single' if single else 'perbin'}"
            store(name, run(name, lambda: cls(num_samples=S, single_jitter=single).train()(rb)))

    # ---- PDFSampler on eval-mode uniform bins --------------------------------------------------------------------
    base = RS.UniformSampler(num_samples=S).eval()(rb)
    out["pdf_weights"] = npy(pdf_w)
    for inc in (False, True):
        for single in (True, False):
            name = f"pdf_{'inc' if inc else 'noinc'}_{'single' if single else 'perbin'}"
            smp = RS.PDFSampler(include_original=inc, single_jitter=single, histogram_padding=0.01).train()
            store(name, run(name, lambda: smp(rb, base, pdf_w[..., None], num_samples=PDF_S_OUT), log_inds=True))
    # the top jitter: u = linspace(...)[-1] + (1 - 2^-24) / nb rounds to exactly 1.0f
    smp = RS.PDFSampler(include_original=False, histogram_padding=0.01).train()
    name = "pdf_top_jitter"
    store(name, run(name, lambda: smp(rb, base, pdf_w[..., None], num_samples=PDF_S_OUT), inject=lambda shape: torch.full(shape, TOP_JITTER),
                    log_inds=True))

    # ---- composite samplers driven by the reference field -------------------------------------------------------
    store("neus", run("neus", lambda: RS.NeuSSampler().train()(rb, sdf_fn=field.get_sdf), log_inds=True))

    class Beta0Density:   # the field's LaplaceDensity with get_beta() pinned to TRAIN_SAMPLER_BETA0
        def get_beta(self):
            return torch.tensor([cases.TRAIN_SAMPLER_BETA0])

        def __call__(self, sdf, beta=None):
            return field.laplace_density(sdf, beta=beta)

    eb = RS.ErrorBoundedSampler(num_samples=64, num_samples_eval=128, num_samples_extra=32).train()
    rs_e, eik = run("error_bounded", lambda: eb(rb, density_fn=Beta0Density(), sdf_fn=field.get_sdf, return_eikonal_points=True))
    store("error_bounded", rs_e)
    out["error_bounded.eikonal_points"] = npy(eik)

    us = RS.UniSurfSampler().train()
    rs_u, surf = run("unisurf", lambda: us(make_bundle(R, o, d, cam, nears, fars), occupancy_fn=field.get_occupancy, sdf_fn=field.get_sdf,
                                           return_surface_points=True))
    store("unisurf", rs_u)
    out["unisurf.surface_points"] = npy(surf)

    dens = [lambda p, i=i: cases.proposal_density(p, i) for i in range(2)]
    for anneal in (1.0, 0.5):
        name = f"proposal_anneal{anneal:g}"
        ps = RS.ProposalNetworkSampler(num_proposal_samples_per_ray=(256, 96), num_nerf_samples_per_ray=48, num_proposal_network_iterations=2).train()
        ps.set_anneal(anneal)
        rs_p, wl, rsl = run(name, lambda: ps(rb, density_fns=dens))
        store(name, rs_p)
        for i, (w, r) in enumerate(zip(wl, rsl)):
            out[f"{name}.weights{i}"] = npy(w[..., 0])
            out[f"{name}.level{i}.spacing"] = bins_of(r)[0]

    os.makedirs(GOLDEN_DIR, exist_ok=True)
    path = os.path.join(GOLDEN_DIR, "samplers_train.npz")
    np.savez_compressed(path, **out)
    meta = {"case": cases.TRAIN_SAMPLER_CASE, "rays": cases.TRAIN_SAMPLER_RAYS, "seed": SEED, "pdf_num_samples": PDF_S_OUT, "draws": runs}
    with open(os.path.join(GOLDEN_DIR, "samplers_train.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"wrote {path}: {os.path.getsize(path) / 1024:.0f} KiB, {len(runs)} runs")


if __name__ == "__main__":
    torch.set_num_threads(8)
    mint()
