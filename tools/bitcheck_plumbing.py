"""Bit-identity check of the Python plumbing around the library calls: renders (dense, packed, from alphas, SDFField.render) under every
background form, with and without autograd, and the kernel forwards of the background and proposal fields in ray and point mode under
each contraction.  Every case runs after torch.manual_seed, so "random" backgrounds draw the same numbers on two trees.

  python tools/bitcheck_plumbing.py --out A.pt          # on one tree (needs a GPU)
  python tools/bitcheck_plumbing.py --compare A.pt B.pt # every tensor equal (torch.equal) and every launch count the same
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _cases():
    import sdfstudio_b200 as sb
    from sdfstudio_b200 import renderers
    from sdfstudio_b200.rays import make_ray_samples

    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(0)
    R, S = 300, 48
    o = torch.randn(R, 3, generator=g)
    o = o / o.norm(dim=-1, keepdim=True) * 2.5
    d = torch.nn.functional.normalize(-o + 0.6 * torch.randn(R, 3, generator=g), dim=-1)
    bins = torch.sort(0.2 + 7.8 * torch.rand(R, S + 1, generator=g), dim=-1).values
    cam = torch.randint(0, 8, (R,), generator=g)
    rb = sb.RayBundle(origins=o.to(dev), directions=d.to(dev), pixel_area=torch.ones(R, 1, device=dev), camera_indices=cam.view(R, 1).to(dev))
    b = bins.to(dev).contiguous()
    rs = make_ray_samples(rb, b, b, None)
    rs_pt = rb.get_ray_samples(b[:, :-1, None], b[:, 1:, None])          # no bin buffer: point mode
    w = torch.rand(R, S, 1, generator=g).to(dev) * 0.05
    alphas = torch.rand(R, S, 1, generator=g).to(dev) * 0.1
    rgb, nrm = torch.rand(R, S, 3, generator=g).to(dev), torch.rand(R, S, 3, generator=g).to(dev)
    backgrounds = {"color": torch.tensor([0.2, 0.5, 0.9]), "per_ray": torch.rand(R, 3, generator=g).to(dev), "last_sample": "last_sample",
                   "random": "random"}

    def grads(fn, *leaves):
        leaves = [t.clone().requires_grad_(True) for t in leaves]
        out = fn(*leaves)
        loss = sum((v.float() * (k + 1)).sum() for k, v in enumerate(out.values()) if v.requires_grad)
        loss.backward()
        return {**out, **{f"grad{i}": t.grad for i, t in enumerate(leaves)}}

    for bn, bg in backgrounds.items():
        for method in ("expected", "median"):
            kw = dict(bins=b, background=bg, depth_method=method, want_acc=True, want_normal=True)
            yield f"render/{bn}/{method}", lambda kw=kw: renderers._render(w, rgb=rgb, normals=nrm, **kw)
            yield f"render_grad/{bn}/{method}", lambda kw=kw: grads(lambda w_, c_, n_: renderers._render(w_, rgb=c_, normals=n_, **kw), w, rgb, nrm)
        yield f"from_alphas/{bn}", lambda bg=bg: sb.render_from_alphas(alphas, rgb, nrm, rs, bg)
        yield f"from_alphas_grad/{bn}", lambda bg=bg: grads(lambda a_, c_, n_: sb.render_from_alphas(a_, c_, n_, rs, bg, training=True), alphas, rgb, nrm)
    yield "render/no_rgb", lambda: renderers._render(w, bins=b, depth_method="expected", want_acc=True)
    dens = torch.rand(R, S, 1, generator=g).to(dev) * 2.0
    for tn, wt in (("", False), ("_T", True)):
        as_dict = lambda r: dict(zip(("weights", "transmittance"), r)) if isinstance(r, tuple) else {"weights": r}  # noqa: E731
        yield f"weights_alphas{tn}", lambda wt=wt: as_dict(sb.rays.weights_from_alphas(alphas, wt))
        yield f"weights_alphas_grad{tn}", lambda wt=wt: grads(lambda a_: as_dict(sb.rays.weights_from_alphas(a_, wt)), alphas)
        yield f"weights_density{tn}", lambda wt=wt: as_dict(sb.rays.weights_from_density(b, dens, wt))
        yield f"weights_density_grad{tn}", lambda wt=wt: grads(lambda d_: as_dict(sb.rays.weights_from_density(b, d_, wt)), dens)
    idx = torch.arange(R, device=dev).repeat_interleave(S)
    for bn in ("color", "per_ray", "random"):
        yield f"packed/{bn}", lambda bn=bn: renderers._render_packed(w.reshape(-1), idx, R, rgb=rgb.reshape(-1, 3), normals=nrm.reshape(-1, 3), ray_samples=rs_pt,
                                                                     background=backgrounds[bn], want_acc=True, want_normal=True, want_depth=True)

    torch.manual_seed(0)
    cfg = sb.SDFFieldConfig(use_grid_feature=True, num_layers=2, num_layers_color=2, hidden_dim=256, log2_hashmap_size=14, precision="bf16x3")
    sdf = sb.SDFField(cfg, torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), 8).to(dev).eval()
    rs_cam = make_ray_samples(rb, b, b, None)
    for bn, bg in backgrounds.items():
        yield f"sdf_render/{bn}", lambda bg=bg: sdf.render(rs_cam, bg, sample_outputs=("sdf",))
    for prec in ("bf16x3", "fp32"):    # the fused engine and the generic one: every per-sample head
        torch.manual_seed(0)
        cfg_p = sb.SDFFieldConfig(use_grid_feature=True, num_layers=2, num_layers_color=2, hidden_dim=256, log2_hashmap_size=14, precision=prec)
        f = sb.SDFField(cfg_p, torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), 8).to(dev).eval()
        yield f"sdf_outputs/{prec}", lambda f=f: {str(k): v for k, v in f.get_outputs(rs_cam, return_alphas=True, return_occupancy=True).items()}
    for norm in ("linf", "l2", "none"):
        sd = None if norm == "none" else sb.SceneContraction(order=float("inf") if norm == "linf" else None)
        torch.manual_seed(1)
        nerf = sb.NeRFField(position_encoding=sb.NeRFEncoding(3, 10, 0.0, 8.0, include_input=True),
                            direction_encoding=sb.NeRFEncoding(3, 4, 0.0, 4.0, include_input=True), spatial_distortion=sd).to(dev).eval()
        nfc = sb.TCNNNerfactoField(torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), num_images=8, log2_hashmap_size=12, max_res=512,
                                   spatial_distortion=sd).to(dev).eval()
        with torch.no_grad():
            nfc.mlp_base.params.normal_(0, 0.3, generator=None)
        prop = sb.HashMLPDensityField(torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), spatial_distortion=sd).to(dev).eval()
        for mode, samples in (("ray", rs), ("point", rs_pt)):
            yield f"nerf/{norm}/{mode}", lambda f=nerf, s=samples: dict(zip(("density", "rgb"), f._kernel_forward(s)))
            yield f"nerfacto/{norm}/{mode}", lambda f=nfc, s=samples: dict(zip(("density", "rgb"), f._kernel_forward(s)))
        yield f"proposal/{norm}", lambda f=prop: dict(zip(("density", "pre"), f.density_from_positions(rs.frustums.get_positions() * 0.7,
                                                                                                      return_pre_activation=True)))


def run(path):
    import sdfstudio_b200 as sb

    res = {}
    for name, fn in _cases():
        torch.manual_seed(1234)
        n0 = sb._lib.launch_count()
        out = fn()
        torch.cuda.synchronize()
        res[name] = ({k: v.detach().cpu() for k, v in out.items() if torch.is_tensor(v)}, sb._lib.launch_count() - n0)
    torch.save(res, path)
    print(f"{len(res)} cases -> {path}")


def compare(a_path, b_path):
    a, b = torch.load(a_path), torch.load(b_path)
    bad = [n for n in a if n not in b] + [n for n in b if n not in a]
    for n in a.keys() & b.keys():
        (ta, la), (tb, lb) = a[n], b[n]
        if la != lb or ta.keys() != tb.keys() or not all(torch.equal(ta[k], tb[k]) for k in ta):
            bad.append(n)
    print(f"{len(a)} cases, {sum(len(v[0]) for v in a.values())} tensors, {len(bad)} differ" + (f": {sorted(bad)}" if bad else ""))
    return 1 if bad else 0


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2)
    args = ap.parse_args()
    sys.exit(compare(*args.compare) if args.compare else run(args.out))
