"""neus-acc on the GPU: the occupancy march and prune (csrc/occupancy.cu), the packed weights / accumulation (csrc/render.cu,
render_backward.cu), SDFField on packed samples, and the composition of models/neus_acc.py:96-142 from this package, each against
oracle/occupancy.py and the fp64 field oracle.  The march, weights and accumulation are nerfacc arithmetic and are checked against the
restatement only (DESIGN §4)."""
import numpy as np
import pytest
import torch

from oracle import occupancy
from oracle.field import OracleField, scene_contraction

from helpers import build_case, load_golden, make_bundle

pytestmark = pytest.mark.gpu


def _maxrel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _sampler(lo, hi, res, grid=None, step=None):
    import sdfstudio_b200 as sb

    s = sb.NeuSAccSampler(aabb=torch.tensor([[lo] * 3, [hi] * 3]), resolution=res, steps_warpup=0, steps_per_grid_update=1).cuda()
    if grid is not None:
        s._binary.copy_(torch.as_tensor(grid))
    if step is not None:
        s.step_size = step
    return s


def _check_march(s, o, d, nears, fars):
    import sdfstudio_b200 as sb

    R = o.shape[0]
    rb = sb.RayBundle(origins=o.float().cuda(), directions=d.float().cuda(), pixel_area=torch.ones(R, 1, device="cuda"),
                      nears=nears.reshape(R, 1).float().cuda(), fars=fars.reshape(R, 1).float().cuda())
    ri, ts, te = s.march(rb)
    off = ri._packed_offsets.cpu().numpy()
    c_ref, ri_ref, ts_ref, te_ref = occupancy.march(o.numpy(), d.numpy(), nears.numpy(), fars.numpy(), s._roi_aabb, s._binary.cpu().numpy(),
                                                    s.step_size)
    assert np.array_equal(np.diff(off), c_ref)
    assert np.array_equal(ri.cpu().numpy(), ri_ref)
    assert np.array_equal(ts[:, 0].cpu().numpy().view(np.uint32), ts_ref.view(np.uint32))
    assert np.array_equal(te[:, 0].cpu().numpy().view(np.uint32), te_ref.view(np.uint32))
    return c_ref


def _shell(res, radius=0.5, width=0.1):
    c = (np.arange(res) + 0.5) / res * 2 - 1
    x, y, z = np.meshgrid(c, c, c, indexing="ij")
    return np.abs(np.sqrt(x * x + y * y + z * z) - radius) < width


def test_march_matches_oracle_bitwise():
    from sdfstudio_b200.synthetic import dtu_like_rays

    res = 64
    shell = _shell(res)
    o, d, _, nears, fars = dtu_like_rays(1024, 5)
    counts = _check_march(_sampler(-1.0, 1.0, res, shell, 0.004), o, d, nears[:, 0], fars[:, 0])
    assert counts.sum() > 0 and (counts == 0).any()

    # axis-aligned directions (0 * inf in the voxel skip), rays that miss the ROI, near > far, rays starting inside the box
    axes = torch.cat([torch.eye(3), -torch.eye(3)])
    o_ax = -2.0 * axes + torch.tensor([0.13, -0.21, 0.07])
    o_miss = torch.tensor([[0.0, 3.0, -3.0], [1.5, 1.5, 0.0], [0.0, 0.0, 2.0]])
    d_miss = torch.tensor([[0.0, 0.0, 1.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    g = torch.Generator().manual_seed(9)
    o_in = torch.rand(64, 3, generator=g) * 1.2 - 0.6
    d_in = torch.nn.functional.normalize(torch.randn(64, 3, generator=g), dim=-1)
    o_all = torch.cat([o_ax, o_miss, o_in, o_in[:4]])
    d_all = torch.cat([axes, d_miss, d_in, d_in[:4]])
    R = o_all.shape[0]
    nears_all = torch.cat([torch.full((R - 68,), 0.3), torch.zeros(64), torch.full((4,), 3.0)])
    fars_all = torch.cat([torch.full((R - 4,), 4.0), torch.full((4,), 1.0)])   # the last four: near > far
    for grid in (shell, np.zeros_like(shell), np.ones_like(shell)):
        counts = _check_march(_sampler(-1.0, 1.0, res, grid, 0.01), o_all, d_all, nears_all, fars_all)
        assert (counts[-4:] == 0).all() and (counts[6:9] == 0).all()
        if not grid.any():
            assert counts.sum() == 0

    # absorbing far: t stops increasing just past 2^15 with a 1e-3 step; the march must end there
    counts = _check_march(_sampler(-1e9, 1e9, 4, np.ones((4, 4, 4), bool), 1e-3), torch.zeros(1, 3), torch.tensor([[1.0, 0.0, 0.0]]),
                          torch.tensor([32767.5]), torch.tensor([1e8]))
    assert 100 < counts[0] < 1000


def test_prune_matches_reference_grid():
    g = load_golden("neus_acc")
    vs = g["voxel_size"][0]
    s = _sampler(-1.2, 1.2, 16, g["binary0"])
    near_threshold = 0
    for k, (before, sdf, after) in enumerate(((g["binary0"], g["sdf1"], g["binary1"]), (g["binary1"], g["sdf2"], g["binary2"]))):
        s._binary.copy_(before)
        s.step_size = float(g[f"step_size{k + 1}"][0])
        inv = g["inv_s"][k: k + 1]
        s.update_binary_grid(1, sdf_fn=lambda x, sdf=sdf: sdf[: x.shape[0]].cuda(), inv_s=lambda inv=inv: inv.cuda())
        alpha64 = occupancy.prune_alpha(sdf.double(), vs.double(), s.step_size, inv.double())
        near = ((alpha64 - s.alpha_thres).abs() <= 1e-6 * s.alpha_thres)
        near_threshold += int(near.sum())
        idx = torch.nonzero(before.reshape(-1)).reshape(-1)[~near]
        assert torch.equal(s._binary.cpu().reshape(-1)[idx], after.reshape(-1)[idx])
        assert not (s._binary.cpu() & ~before).any()
    print(f"prune: {near_threshold} voxels within 1e-6 of alpha_thres")
    assert int(s._update_counter) == 2


def _ragged(seed, n_rays=300, max_len=200):
    g = torch.Generator().manual_seed(seed)
    counts = torch.randint(0, max_len, (n_rays,), generator=g)
    counts[::17] = 0
    ri = torch.repeat_interleave(torch.arange(n_rays), counts)
    alphas = torch.rand(ri.numel(), generator=g) ** 3
    alphas[torch.randint(0, ri.numel(), (40,), generator=g)] = 1.0
    alphas[torch.randint(0, ri.numel(), (40,), generator=g)] = 0.0
    return ri, alphas, occupancy.offsets_of(counts.numpy())


def test_packed_weights_forward_backward():
    import sdfstudio_b200 as sb

    ri, alphas, off = _ragged(1)
    n = off.size - 1
    a = alphas.cuda()[:, None].requires_grad_(True)
    w = sb.packed.render_weight_from_alpha(a, ray_indices=ri.cuda(), n_rays=n)
    w2 = sb.packed.render_weight_from_alpha(a.detach(), ray_indices=ri.cuda(), n_rays=n)
    assert torch.equal(w.detach(), w2)
    a64 = alphas.double().requires_grad_(True)
    w64 = occupancy.packed_weights64(a64, off)
    assert float((w.detach().cpu()[:, 0].double() - w64.detach()).abs().max()) < 1e-6
    gw = torch.randn(ri.numel(), generator=torch.Generator().manual_seed(2))
    w.backward(gw.cuda()[:, None])
    w64.backward(gw.double())
    assert torch.isfinite(a.grad).all()
    assert _maxrel(a.grad[:, 0], a64.grad) < 1e-5
    # packed_info (start, count) form
    counts = torch.from_numpy(np.diff(off))
    pi = torch.stack([torch.from_numpy(off[:-1]), counts], -1).int().cuda()
    assert torch.equal(sb.packed.render_weight_from_alpha(a.detach(), packed_info=pi), w2)


@pytest.mark.parametrize("C", [None, 1, 3])
def test_packed_accumulate_forward_backward(C):
    import sdfstudio_b200 as sb

    ri, alphas, off = _ragged(3)
    n = off.size - 1
    g = torch.Generator().manual_seed(4)
    w = (alphas * 0.5)[:, None].cuda().requires_grad_(True)
    v = torch.randn(ri.numel(), C, generator=g).cuda().requires_grad_(True) if C else None
    out = sb.packed.accumulate_along_rays(w, ri.cuda(), values=v, n_rays=n)
    again = sb.packed.accumulate_along_rays(w.detach(), ri.cuda(), values=None if v is None else v.detach(), n_rays=n)
    assert torch.equal(out.detach(), again)
    w64 = w.detach().cpu().double().requires_grad_(True)
    v64 = v.detach().cpu().double().requires_grad_(True) if C else None
    ref = occupancy.accumulate64(w64, ri, v64, n)
    assert out.shape == ref.shape
    assert _maxrel(out, ref) < 1e-6
    go = torch.randn(ref.shape, generator=g)
    out.backward(go.cuda())
    ref.backward(go.double())
    assert _maxrel(w.grad, w64.grad) < 1e-6
    if C:
        assert _maxrel(v.grad, v64.grad) < 1e-6


def _flat(rs):
    """The samples of a dense RaySamples [R,S] as packed samples [N] (per-sample origins / directions, starts / ends [N,1])."""
    import sdfstudio_b200 as sb

    fr = rs.frustums
    R, S = fr.starts.shape[:2]
    f = sb.Frustums(origins=fr.origins.reshape(-1, 3).contiguous(), directions=fr.directions.reshape(-1, 3).contiguous(),
                    starts=fr.starts.reshape(-1, 1).contiguous(), ends=fr.ends.reshape(-1, 1).contiguous(), pixel_area=fr.pixel_area.reshape(-1, 1))
    return sb.RaySamples(frustums=f, camera_indices=rs.camera_indices.reshape(-1, 1).contiguous(), deltas=rs.deltas.reshape(-1, 1).contiguous())


@pytest.mark.parametrize("config", ["neus_generic_fp32", "neusfacto_fused_bf16x3"])
def test_field_on_packed_samples_equals_dense(config):
    import sdfstudio_b200 as sb
    from sdfstudio_b200.synthetic import dtu_like_rays, perturb_field_

    torch.manual_seed(0)
    if config == "neus_generic_fp32":
        cfg = sb.SDFFieldConfig(precision="fp32")
    else:
        cfg = sb.SDFFieldConfig(use_grid_feature=True, num_layers=2, num_layers_color=2, hidden_dim=256, bias=0.5, beta_init=0.3, inside_outside=False,
                                log2_hashmap_size=15, grid_layout="torch", precision="bf16x3")
    field = perturb_field_(sb.SDFField(cfg, torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), 49), 0).cuda().eval()
    R, S = 64, 48
    o, d, cam, nears, fars = dtu_like_rays(R, 11)
    with torch.no_grad():
        rs = sb.UniformSampler(num_samples=S, train_stratified=False).eval()(make_bundle(o, d, cam, nears, fars))
        flat = _flat(rs)
        dense, packed = field(rs, return_alphas=True), field(flat, return_alphas=True)
        for k in (sb.FieldHeadNames.RGB, sb.FieldHeadNames.SDF, sb.FieldHeadNames.NORMAL, sb.FieldHeadNames.GRADIENT, sb.FieldHeadNames.ALPHA):
            assert packed[k].shape == (R * S, dense[k].shape[-1])
            assert torch.equal(packed[k], dense[k].reshape(R * S, -1)), k
        assert torch.equal(field.get_sdf(flat), field.get_sdf(rs).reshape(R * S, 1))
        assert torch.equal(field.get_alpha(flat), field.get_alpha(rs).reshape(R * S, 1))


def test_neus_acc_composition_and_training_step():
    import sdfstudio_b200 as sb

    spec, kw, o, d, cam, nears, fars, oracle, field = build_case("neusfacto_c1")
    R = 48
    o, d, cam, nears, fars = o[:R], d[:R], cam[:R], nears[:R], fars[:R]
    s = _sampler(-1.0, 1.0, 32)
    # this field's sdf is >= 0.35 on the whole box: prune at a low inv_s so that the voxels nearest its zero level set stay occupied
    s.update_binary_grid(0, sdf_fn=lambda x: field.forward_geonetwork(x)[:, 0].contiguous(), inv_s=lambda: torch.tensor([2.0], device="cuda"))
    assert int(s._update_counter) == 1 and 0 < int(s._binary.sum()) < s._binary.numel()
    s.step_size = 0.01
    bundle = make_bundle(o, d, cam, nears, fars)
    rs, ri = s(bundle, sdf_fn=field.get_sdf, alpha_fn=field.get_alpha)
    N = ri.numel()
    assert N > 0 and rs.frustums.starts.shape == (N, 1)
    _check_march(s, o, d, nears[:, 0], fars[:, 0])

    def compose(fo, weights_fn, acc_fn):
        w = weights_fn(fo["alpha"])
        mid = (rs.frustums.starts + rs.frustums.ends) / 2
        return {"rgb": acc_fn(w, fo["rgb"]), "normal": acc_fn(w, fo["normal"]), "accumulation": acc_fn(w, None), "depth": acc_fn(w, mid)}

    # ---- eval: the package vs the oracle (fp32 march, fp64 / fp32 field and compositing on the same samples)
    with torch.no_grad():
        fo = field(rs, return_alphas=True)
        got = compose({"alpha": fo[sb.FieldHeadNames.ALPHA], "rgb": fo[sb.FieldHeadNames.RGB], "normal": fo[sb.FieldHeadNames.NORMAL]},
                      lambda a: sb.packed.render_weight_from_alpha(a, ray_indices=ri, n_rays=R),
                      lambda w, v: sb.packed.accumulate_along_rays(w, ri, values=v, n_rays=R))
    ric = ri.cpu()
    ts, de = rs.frustums.starts.cpu(), rs.deltas.cpu()
    off = ri._packed_offsets.cpu().numpy()
    refs = {}
    for dt, of in ((torch.float64, OracleField(spec, oracle.p, dtype=torch.float64)), (torch.float32, oracle)):
        oo = of.get_outputs(o[ric].to(dt), d[ric].to(dt), ts.to(dt), de.to(dt), cam[ric], return_alphas=True)
        w = occupancy.packed_weights64(oo["alphas"][:, 0, 0], off)
        mid = (ts + rs.frustums.ends.cpu()).double() / 2
        refs[dt] = {"rgb": occupancy.accumulate64(w, ric, oo["rgb"][:, 0], R), "normal": occupancy.accumulate64(w, ric, oo["normals"][:, 0], R),
                    "accumulation": occupancy.accumulate64(w, ric, None, R), "depth": occupancy.accumulate64(w, ric, mid, R)}
    for k, v in got.items():
        exact, noise = refs[torch.float64][k], (refs[torch.float32][k] - refs[torch.float64][k]).abs().max()
        err = (v.detach().double().cpu() - exact).abs().max()
        bound = max(1e-4 * float(exact.abs().max()), 4.0 * float(noise))
        assert float(err) <= bound, f"{k}: {float(err):.3e} > {bound:.3e}"

    # ---- one training step: rgb L1 + eikonal on eik_grad, gradients of every field parameter vs fp64 autograd
    if spec.contraction is not None:
        field.spatial_distortion = sb.SceneContraction(order=float("inf") if spec.contraction == "linf" else None)
    field.train()
    g = torch.Generator().manual_seed(3)
    target = torch.rand(R, 3, generator=g)
    fo = field(rs, return_alphas=True)
    w = sb.packed.render_weight_from_alpha(fo[sb.FieldHeadNames.ALPHA], ray_indices=ri, n_rays=R)
    rgb = sb.packed.accumulate_along_rays(w, ri, values=fo[sb.FieldHeadNames.RGB], n_rays=R)
    eik = ((fo[sb.FieldHeadNames.GRADIENT].norm(2, dim=-1) - 1) ** 2).mean()
    loss = (rgb - target.cuda()).abs().mean() + 0.1 * eik
    field.zero_grad()
    loss.backward()

    of = OracleField(spec, oracle.p, dtype=torch.float64)
    for v in of.p.values():
        if v.is_floating_point():
            v.requires_grad_(True)
    of.training = True
    pos = o[ric].double() + d[ric].double() * ts.double()
    x = scene_contraction(pos, spec.contraction).requires_grad_(True)
    h = of.forward_geonetwork(x)
    sdf, geo = h[:, :1], h[:, 1:]
    grads = torch.autograd.grad(sdf, x, torch.ones_like(sdf), create_graph=True)[0]
    rgb_s = of.get_colors(x, d[ric].double(), grads, geo, cam[ric].reshape(-1))
    alphas = of.get_alpha(d[ric].double(), de.double(), sdf, grads)
    w64 = occupancy.packed_weights64(alphas[:, 0], off)
    rgb64 = occupancy.accumulate64(w64, ric, rgb_s, R)
    loss64 = (rgb64 - target.double()).abs().mean() + 0.1 * ((grads.norm(2, dim=-1) - 1) ** 2).mean()
    loss64.backward()
    assert abs(float(loss) - float(loss64)) < 2e-4 * max(1.0, abs(float(loss64)))
    name_map = {"hash_table": "encoding.hash_table" if spec.grid_layout == "torch" else "encoding.params"}
    params = dict(field.named_parameters())
    errs = {}
    for k, v in of.p.items():
        if not v.is_floating_point() or v.grad is None or name_map.get(k, k) not in params or params[name_map.get(k, k)].grad is None:
            continue
        gc = params[name_map.get(k, k)].grad
        if float(v.grad.abs().max()) == 0.0:
            assert float(gc.abs().max()) < 1e-9, k
            continue
        errs[k] = _maxrel(gc.reshape(v.grad.shape), v.grad)
    assert len(errs) > 4
    bad = {k: f"{e:.2e}" for k, e in errs.items() if e >= 2e-3}
    assert not bad, f"grad max-rel errors: {bad}"

    # ---- the sampler's state dict round-trips
    s2 = _sampler(-1.0, 1.0, 32)
    s2.load_state_dict(s.state_dict())
    s2.step_size = s.step_size
    for k, v in s.state_dict().items():
        assert torch.equal(s2.state_dict()[k], v), k
    ri2, ts2, te2 = s2.march(bundle)
    assert torch.equal(ri2, ri) and torch.equal(ts2, rs.frustums.starts) and torch.equal(te2, rs.frustums.ends)
