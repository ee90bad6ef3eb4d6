"""Fused map-parameter step (rtg_map_adam_step / mapoptim.MapOptimizer) against the reference's eager flow: torch
activations + masked l2 attach loss + torch.optim.Adam over the six groups of GaussianPointCloud.parametrize
(SLAM/gaussian_pointcloud.py:245-284, SLAM/multiprocess/mapper.py:384-401,452-456)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import helpers
from rtg_slam_b200 import scene

pytestmark = pytest.mark.gpu

LRS = dict(xyz=1e-3, f_dc=5e-4, f_rest=5e-4 / 20.0, opacity=2e-4, scaling=4e-3, rotation=1e-3)  # configs/base.yaml:82-86 (+ a non-zero opacity lr)


def _raw_map(P, dev, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)
    raw = dict(xyz=r(P, 3), features_dc=r(P, 1, 3) * 0.5, features_rest=r(P, 15, 3) * 0.1, opacity=r(P, 1) * 2.0 + 1.0,
               scaling=r(P, 3) * 0.5 - 3.0, rotation=r(P, 4) * (0.5 + torch.rand(P, 1, generator=g)))
    return {k: v.to(dev) for k, v in raw.items()}


def _get_normal(scaling_raw, rotation_raw):
    """GaussianPointCloud.get_normal (gaussian_pointcloud.py:539-550) in eager torch."""
    q = F.normalize(rotation_raw)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], dim=-1).view(-1, 3, 3)
    idx = torch.argmin(torch.exp(scaling_raw), dim=1)
    n = torch.gather(R.transpose(1, 2), 1, idx[:, None, None].expand(-1, -1, 3))[:, 0, :]
    return n / (torch.norm(n, dim=-1, keepdim=True) + 1e-8)


# 300,007 and 1,000,003 rows: map_adam_kernel launches one wave of resident CTAs (at most 1056 x 8 warps on 132 SMs), so
# its grid-stride loop makes a second and later pass over the 32-row blocks, and the last block is partial
@pytest.mark.parametrize("P,with_attach,use_radii", [(5003, True, True), (4096, False, False), (37, True, False), (300_007, False, False),
                                                     (1_000_003, True, True)])
def test_map_step_matches_torch_activations_and_adam(cuda_device, P, with_attach, use_radii):
    from rtg_slam_b200.mapoptim import MapOptimizer
    dev = cuda_device
    raw = _raw_map(P, dev, seed=P)
    torch.manual_seed(P + 1)
    vis = torch.rand(P, device=dev) < 0.4  # rows that receive a rasterizer gradient
    W = {k: torch.randn_like(v) * vis.view(-1, *([1] * (v.dim() - 1))).float() for k, v in
         dict(xyz=raw["xyz"], shs=torch.cat([raw["features_dc"], raw["features_rest"]], 1), opacity=raw["opacity"],
              scales=raw["scaling"], rotations=raw["rotation"]).items()}
    # a few visible rows with an exactly zero colour gradient: their confidence must not move
    zero_dc = vis & (torch.rand(P, device=dev) < 0.2)
    W["shs"][zero_dc, 0, :] = 0
    init_stat = {"opacity": raw["opacity"].clone(), "scaling": raw["scaling"] + 0.05 * torch.randn_like(raw["scaling"]),
                 "xyz": raw["xyz"] + 0.01 * torch.randn_like(raw["xyz"]), "rotation_raw": raw["rotation"] + 0.02 * torch.randn_like(raw["rotation"])}
    iters = 10

    def image_loss(d):  # any smooth function of the activated tensors stands in for render + loss (reference_flow repeats it)
        return sum((W[k] * (d[k] ** 2 + d[k])).sum() for k in W)

    # ---- reference flow, in float32 (the reference's own precision) and in float64
    def reference_flow(dtype):
        p = {k: torch.nn.Parameter(v.to(dtype, copy=True)) for k, v in raw.items()}
        Wd, ist = {k: v.to(dtype) for k, v in W.items()}, {k: v.to(dtype) for k, v in init_stat.items()}
        groups = [{"params": [p["xyz"]], "lr": LRS["xyz"]}, {"params": [p["features_dc"]], "lr": LRS["f_dc"]},
                  {"params": [p["features_rest"]], "lr": LRS["f_rest"]}, {"params": [p["opacity"]], "lr": LRS["opacity"]},
                  {"params": [p["scaling"]], "lr": LRS["scaling"]}, {"params": [p["rotation"]], "lr": LRS["rotation"]}]
        ref_opt = torch.optim.Adam(groups, lr=0.0, eps=1e-15)
        conf_ref = torch.zeros(P, device=dev)
        for _ in range(iters):
            d = dict(xyz=p["xyz"], shs=torch.cat((p["features_dc"], p["features_rest"]), dim=1), opacity=torch.sigmoid(p["opacity"]),
                     scales=torch.exp(p["scaling"]), rotations=F.normalize(p["rotation"]))
            loss = sum((Wd[k] * (d[k] ** 2 + d[k])).sum() for k in Wd)
            if with_attach:
                m = (torch.sigmoid(ist["opacity"]) < 0.9).squeeze()
                l2 = lambda a, b: ((a - b) ** 2).mean()
                if m.sum() > 0:
                    loss = loss + 1000 * (l2(p["scaling"][m], ist["scaling"][m]) + l2(p["xyz"][m], ist["xyz"][m])
                                          + l2(p["rotation"][m], ist["rotation_raw"][m]))
            loss.backward()
            ref_opt.step()
            conf_ref[(p["features_dc"].grad.abs() != 0).any(dim=-1).squeeze(-1)] += 1
            ref_opt.zero_grad(set_to_none=True)
        return p, conf_ref
    p, conf_ref = reference_flow(torch.float32)
    p64, _ = reference_flow(torch.float64)
    # Rows on which float32 rounding alone moves the reference by more than a tenth of the bound: Adam with eps = 1e-15
    # turns a gradient component that cancels to rounding level into a full step of either sign. At a million rows a
    # rotation row or so does that (float32 torch 1e-3 from float64 there); the kernel is held to float64 on them instead.
    ill = torch.zeros(P, dtype=torch.bool, device=dev)
    for k in p:
        top = float(p64[k].detach().abs().max())
        ill |= (p[k].detach().double() - p64[k].detach()).abs().reshape(P, -1).amax(1) > 1e-6 * top
    print(f"P={P}: {int(ill.sum())} rows where float32 torch is more than 1e-6 from float64")
    assert int(ill.sum()) <= P // 100_000
    ok = ~ill

    # ---- fused flow
    conf = torch.zeros(P, device=dev)
    opt = MapOptimizer(raw["xyz"], raw["features_dc"], raw["features_rest"], raw["opacity"], raw["scaling"], raw["rotation"], LRS,
                       confidence=conf)
    assert torch.allclose(opt.normal, _get_normal(raw["scaling"], raw["rotation"]), atol=2e-6)
    if with_attach:
        opt.set_attach(init_stat)
    radii = vis.to(torch.int32) * 7 if use_radii else None
    for _ in range(iters):
        image_loss({k: opt.gaussian_data()[k] for k in W}).backward()
        if use_radii:  # what rtg_splat_backward_visible leaves behind: unspecified values in the culled rows
            for t in (opt.xyz, opt.shs, opt.opacity, opt.scales, opt.rotations):
                t.grad[~vis] = float("nan")
        opt.step(radii=radii)
        assert opt.xyz.grad is None

    def rel(a, b):
        return float((a[ok] - b[ok]).abs().max()) / (float(b.abs().max()) + 1e-12)
    got = dict(xyz=opt.xyz.detach(), features_dc=opt.features_dc, features_rest=opt.features_rest, opacity=opt.opacity_raw,
               scaling=opt.scaling_raw, rotation=opt.rotation_raw)
    for k in got:
        moved = float((p[k].detach() - raw[k]).abs().max())
        assert moved > 0, k
        e = rel(got[k], p[k].detach())
        assert e < 1e-5, (k, e, moved)
        # the ill-conditioned rows: no further from float64 than a few times float32 torch is
        want, ref = p64[k].detach()[ill], p[k].detach()[ill].double()
        top = float(p64[k].detach().abs().max())
        assert bool(((got[k][ill].double() - want).abs() <= 4 * (ref - want).abs() + 1e-5 * top).all()), k
    # activated tensors for the next render, and the normal
    assert rel(opt.scales.detach(), torch.exp(p["scaling"].detach())) < 1e-5
    assert rel(opt.rotations.detach(), F.normalize(p["rotation"].detach())) < 1e-5
    assert rel(opt.opacity.detach(), torch.sigmoid(p["opacity"].detach())) < 1e-5
    n_ref = _get_normal(p["scaling"].detach(), p["rotation"].detach())
    same_axis = torch.argmin(opt.scales.detach(), 1) == torch.argmin(torch.exp(p["scaling"].detach()), 1)
    assert float(same_axis.float().mean()) > 0.999
    assert float((opt.normal - n_ref)[same_axis & ok].abs().max()) < 1e-4
    assert torch.equal(conf, conf_ref) and float(conf.max()) == iters
    if with_attach:
        m = (torch.sigmoid(init_stat["opacity"]) < 0.9).squeeze()
        l2 = lambda a, b: ((a - b) ** 2).mean()
        want = 1000 * (l2(p["scaling"][m], init_stat["scaling"][m]) + l2(p["xyz"][m], init_stat["xyz"][m])
                       + l2(p["rotation"][m], init_stat["rotation_raw"][m]))
        assert abs(float(opt.attach_loss()) - float(want)) < 1e-4 * float(want)


def test_map_step_argument_errors(cuda_device):
    from rtg_slam_b200.mapoptim import MapOptimizer
    dev = cuda_device
    raw = _raw_map(64, dev, seed=1)
    with pytest.raises(ValueError):
        MapOptimizer(raw["xyz"], raw["features_dc"], raw["features_rest"][:, :8], raw["opacity"], raw["scaling"], raw["rotation"], LRS)
    with pytest.raises(TypeError):
        MapOptimizer(raw["xyz"].cpu(), raw["features_dc"], raw["features_rest"], raw["opacity"], raw["scaling"], raw["rotation"], LRS)
    opt = MapOptimizer(raw["xyz"], raw["features_dc"], raw["features_rest"], raw["opacity"], raw["scaling"], raw["rotation"], LRS)
    with pytest.raises(RuntimeError):
        opt.step()  # no gradients yet
    sum(v.sum() for k, v in opt.gaussian_data().items() if k != "normal").backward()
    with pytest.raises(TypeError):
        opt.step(radii=torch.ones(64, device=dev))  # not int32


def test_backward_visible_rows_only_leaves_culled_rows_untouched(cuda_device):
    """rtg_splat_backward_visible: identical gradients on the rows with radii > 0, no store to the others."""
    from rtg_slam_b200.rasterizer import GaussianRasterizer, grad_buffers, visible_rows_only
    dev = cuda_device
    cam = scene.make_camera("small")
    g = scene.surfel_room(6000, seed=3)
    rs = helpers.make_settings(cam, dev)
    t = helpers.to_torch(g, dev)
    gc, gd = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in scene.upstream_grads(cam, seed=2)[:2]]
    names = ("xyz", "shs", "opacity", "scales", "rotations")
    buf_names = dict(xyz="means3D", shs="shs", opacity="opacities", scales="scales", rotations="rotations")

    def run(sparse):
        p = {k: t[k].clone().requires_grad_(True) for k in names}
        bufs = {buf_names[k]: torch.full_like(p[k], float("nan")) for k in names}
        out = GaussianRasterizer(rs)(means3D=p["xyz"], opacities=p["opacity"], shs=p["shs"], scales=p["scales"], rotations=p["rotations"])
        with grad_buffers(bufs), visible_rows_only(sparse):
            torch.autograd.backward([out[0], out[1]], [gc.view_as(out[0]), gd.view_as(out[1])])
        return {k: p[k].grad.clone() for k in names}, out[7]

    dense, radii = run(False)
    sparse, radii2 = run(True)
    assert torch.equal(radii, radii2)
    vis = radii > 0
    assert 0 < int(vis.sum()) < vis.numel()
    for k in names:
        assert not torch.isnan(dense[k]).any()
        assert float(dense[k][~vis].abs().max()) == 0.0
        assert torch.isnan(sparse[k][~vis]).all(), k
        # same kernels, same accumulation order up to atomics
        assert float((sparse[k][vis] - dense[k][vis]).abs().max()) <= 1e-5 * float(dense[k].abs().max()) + 1e-12


def test_map_optimizer_loop_matches_eager_flow_through_the_rasterizer(cuda_device):
    """Ten iterations of render -> fused mapping loss -> backward -> step from raw parameters: MapOptimizer (with
    visible_rows_only and radii) against torch activations + attach loss + torch.optim.Adam around the same rasterizer."""
    from rtg_slam_b200.loss import l1_color_depth_loss
    from rtg_slam_b200.mapoptim import MapOptimizer
    from rtg_slam_b200.rasterizer import GaussianRasterizer, visible_rows_only
    dev = cuda_device
    cam = scene.make_camera("small")
    P = 8000
    g = scene.surfel_room(P, seed=11)
    rs = helpers.make_settings(cam, dev)
    t = helpers.to_torch(g, dev)
    with torch.no_grad():
        tgt = GaussianRasterizer(rs)(means3D=t["xyz"] + 0.002, opacities=t["opacity"], shs=t["shs"] * 0.9, scales=t["scales"],
                                     rotations=t["rotations"])
    gt_color, gt_depth = tgt[0].permute(1, 2, 0).contiguous(), tgt[1][0].contiguous()
    op = t["opacity"].clamp(1e-4, 1 - 1e-4)
    raw = dict(xyz=t["xyz"].clone(), features_dc=t["shs"][:, :1].clone(), features_rest=t["shs"][:, 1:].clone(),
               opacity=torch.log(op / (1 - op)), scaling=torch.log(t["scales"]), rotation=t["rotations"] * 1.7)
    lrs = dict(xyz=1e-4, f_dc=5e-4, f_rest=5e-4 / 20, opacity=0.0, scaling=1e-3, rotation=1e-3)
    init_stat = {"opacity": raw["opacity"].clone(), "scaling": raw["scaling"].clone(), "xyz": raw["xyz"].clone(),
                 "rotation_raw": raw["rotation"].clone()}
    init_stat["opacity"][::3] = -1.0  # a third of the rows is "attached"
    iters = 10

    def image_loss(out):
        return l1_color_depth_loss({"render": out[0], "depth": out[1], "depth_index_map": out[3]}, gt_color, gt_depth,
                                   color_weight=0.8, depth_weight=1.0, depth_error_max=0.1)[0]

    p = {k: torch.nn.Parameter(v.clone()) for k, v in raw.items()}
    ref_opt = torch.optim.Adam([{"params": [p["xyz"]], "lr": lrs["xyz"]}, {"params": [p["features_dc"]], "lr": lrs["f_dc"]},
                                {"params": [p["features_rest"]], "lr": lrs["f_rest"]}, {"params": [p["opacity"]], "lr": lrs["opacity"]},
                                {"params": [p["scaling"]], "lr": lrs["scaling"]}, {"params": [p["rotation"]], "lr": lrs["rotation"]}],
                               lr=0.0, eps=1e-15)
    m = (torch.sigmoid(init_stat["opacity"]) < 0.9).squeeze()
    l2 = lambda a, b: ((a - b) ** 2).mean()
    ref_losses = []
    for _ in range(iters):
        out = GaussianRasterizer(rs)(means3D=p["xyz"], opacities=torch.sigmoid(p["opacity"]),
                                     shs=torch.cat((p["features_dc"], p["features_rest"]), dim=1), scales=torch.exp(p["scaling"]),
                                     rotations=F.normalize(p["rotation"]))
        loss = image_loss(out)
        attach = 1000 * (l2(p["scaling"][m], init_stat["scaling"][m]) + l2(p["xyz"][m], init_stat["xyz"][m])
                         + l2(p["rotation"][m], init_stat["rotation_raw"][m]))
        (loss + attach).backward()
        ref_opt.step()
        ref_opt.zero_grad(set_to_none=True)
        ref_losses.append(float(loss.detach()))

    opt = MapOptimizer(raw["xyz"], raw["features_dc"], raw["features_rest"], raw["opacity"], raw["scaling"], raw["rotation"], lrs)
    opt.set_attach(init_stat)
    losses = []
    for _ in range(iters):
        d = opt.gaussian_data()
        out = GaussianRasterizer(rs)(means3D=d["xyz"], opacities=d["opacity"], shs=d["shs"], scales=d["scales"], rotations=d["rotations"])
        loss = image_loss(out)
        with visible_rows_only():
            loss.backward()
        opt.step(radii=out[7])
        losses.append(float(loss.detach()))
    assert ref_losses[-1] < ref_losses[0]
    for a, b in zip(losses, ref_losses):
        assert abs(a - b) < 2e-4 * abs(b), (losses, ref_losses)
    got = dict(xyz=opt.xyz.detach(), features_dc=opt.features_dc, features_rest=opt.features_rest, opacity=opt.opacity_raw,
               scaling=opt.scaling_raw, rotation=opt.rotation_raw)
    for k in got:
        # eps = 1e-15: an element whose gradient is numerically zero steps by sign(noise) * lr, so a few elements may differ
        # by up to 2 * lr * iterations (atomic order in the rasterizer backward); everything else must agree closely
        diff = (got[k] - p[k].detach()).abs()
        scale = float(p[k].detach().abs().max())
        off = float((diff > 1e-5 * scale).float().mean())
        assert off < 5e-3, (k, off)
        assert float(diff.max()) <= 2.0 * max(lrs.values()) * iters + 1e-6, k


# ----------------------------------------------------------------------------- Mapping.history_merge (mapper.py:212-250)
def _close_fp32(a, b, ulps=2):
    return np.all(np.abs(a.astype(np.float64) - b.astype(np.float64)) <= ulps * 1.2e-7 * np.maximum(1.0, np.abs(b)))


@pytest.mark.parametrize("name", sorted(helpers.HISTORY_MERGE_SIZES))
@pytest.mark.parametrize("max_weight", [0.5, 0.9])
def test_history_merge_matches_reference_golden(cuda_device, name, max_weight):
    """mapoptim.history_merge (one kernel, in place) against the golden outputs of the reference's own history_merge method with its
    unmodified slerp (tests/golden/history_merge.npz) and against the numpy oracle. The lerps are the same fp32 operations in
    the same order; the rotation is bounded per row by the conditioning of slerp (helpers.slerp_tolerance)."""
    import os
    from oracle import mapmerge_oracle as mm
    from rtg_slam_b200.mapoptim import history_merge
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "history_merge.npz"))
    hist, cur = helpers.history_merge_inputs(name)
    dev = cuda_device
    h = {k: torch.from_numpy(v).to(dev) for k, v in hist.items()}
    c = {k: torch.from_numpy(v.copy()).to(dev) for k, v in cur.items()}
    history_merge(h, c["confidence"], c["xyz"], c["features_dc"], c["features_rest"], c["scaling"], c["rotation_raw"], max_weight)
    want, dot = mm.history_merge(hist, cur, max_weight)
    for k, ck in (("xyz", "xyz"), ("features_dc", "features_dc"), ("features_rest", "features_rest"), ("scaling", "scaling")):
        got = c[ck].cpu().numpy()
        assert _close_fp32(got, gold[f"{name}_{max_weight}_{k}"]), k
        assert _close_fp32(got, want[k]), k
    got = c["rotation_raw"].cpu().numpy()
    tol = 2 * helpers.slerp_tolerance(dot)
    assert np.isfinite(got).all()
    assert np.all(np.abs(got - gold[f"{name}_{max_weight}_rotation"]).max(-1) <= tol)
    assert torch.equal(c["confidence"].cpu(), torch.from_numpy(cur["confidence"]))   # inputs other than the five are untouched
    # a non-positive weight leaves everything as it is (mapper.py:213-214)
    before = c["xyz"].clone()
    history_merge(h, c["confidence"], c["xyz"], c["features_dc"], c["features_rest"], c["scaling"], c["rotation_raw"], 0.0)
    assert torch.equal(before, c["xyz"])


def test_map_optimizer_history_merge_on_the_sh_block(cuda_device):
    """MapOptimizer.history_snapshot / history_merge: the same kernel on the optimiser's own layout (features_dc / features_rest
    are the two slices of one (P,16,3) block, row stride 48) and the activation forward afterwards."""
    from oracle import mapmerge_oracle as mm
    from rtg_slam_b200.mapoptim import MapOptimizer
    dev = cuda_device
    hist, cur = helpers.history_merge_inputs("window")
    P = hist["xyz"].shape[0]
    t = lambda a: torch.from_numpy(a.copy()).to(dev)
    opacity = torch.randn(P, 1, device=dev)
    conf = t(hist["confidence"]).view(-1).contiguous()
    # the optimiser starts from the history state ...
    raw_rot0 = t(hist["rotation"]) * 1.7          # raw quaternion whose normalisation is the history rotation
    raw_rot0[5:8] = 0                             # zero quaternions stay zero under F.normalize
    opt = MapOptimizer(t(hist["xyz"]), t(hist["features_dc"]), t(hist["features_rest"]), opacity, t(hist["scaling"]), raw_rot0,
                       [1e-3] * 6, confidence=conf)
    snap = opt.history_snapshot()
    assert set(snap) == {"opacity", "confidence", "xyz", "features_dc", "features_rest", "scaling", "rotation", "rotation_raw"}  # mapper.py:146-155
    assert snap["confidence"].shape == (P, 1) and snap["features_rest"].shape == (P, 15, 3) and snap["features_rest"].is_contiguous()
    # ... and "optimises" to the current state of the fixture
    with torch.no_grad():
        opt.xyz.copy_(t(cur["xyz"]))
        opt.shs[:, :1].copy_(t(cur["features_dc"]))
        opt.shs[:, 1:].copy_(t(cur["features_rest"]))
        opt.scaling_raw.copy_(t(cur["scaling"]))
        opt.rotation_raw.copy_(t(cur["rotation_raw"]))
        conf.copy_(t(cur["confidence"]).view(-1))
    opt.history_merge(snap, 0.5)
    hist_used = dict(hist)
    hist_used["rotation"] = snap["rotation"].cpu().numpy()    # normalize(1.7 q): equal to the fixture's up to rounding
    want, dot = mm.history_merge(hist_used, cur, 0.5)
    assert _close_fp32(opt.xyz.detach().cpu().numpy(), want["xyz"])
    assert _close_fp32(opt.features_dc.cpu().numpy(), want["features_dc"])
    assert _close_fp32(opt.features_rest.cpu().numpy(), want["features_rest"])
    assert _close_fp32(opt.scaling_raw.cpu().numpy(), want["scaling"])
    assert np.all(np.abs(opt.rotation_raw.cpu().numpy() - want["rotation"]).max(-1) <= 2 * helpers.slerp_tolerance(dot))
    assert torch.equal(opt.opacity_raw, opacity)                                      # _opacity is not merged
    # activated tensors follow the merged raw parameters
    d = opt.gaussian_data()
    assert torch.allclose(d["rotations"], F.normalize(opt.rotation_raw), atol=1e-6)
    assert torch.allclose(d["scales"], torch.exp(opt.scaling_raw), rtol=1e-6)
    with pytest.raises(RuntimeError):
        MapOptimizer(t(hist["xyz"]), t(hist["features_dc"]), t(hist["features_rest"]), opacity, t(hist["scaling"]), raw_rot0,
                     [1e-3] * 6).history_snapshot()


def test_map_optimizer_with_frozen_stable_rows(cuda_device):
    """`frozen=`: the reference renders `global_params = cat(unstable, stable.detach())` (mapper.py:1034-1108) and only the
    unstable cloud is optimised. Here the stable rows sit behind the optimised rows of the same buffers; the fused step must
    move exactly the first P rows like torch activations + torch.optim.Adam on the unstable parameters, leave the frozen
    rows bit-identical, and history_snapshot / history_merge / write_back must see P rows."""
    from rtg_slam_b200.mapoptim import MapOptimizer
    dev = cuda_device
    P, S, iters = 3001, 1777, 6
    raw = _raw_map(P, dev, seed=11)
    st = _raw_map(S, dev, seed=12)
    frozen = dict(xyz=st["xyz"], opacity=torch.sigmoid(st["opacity"]), scales=torch.exp(st["scaling"]), rotations=F.normalize(st["rotation"]),
                  shs=torch.cat([st["features_dc"], st["features_rest"]], 1).contiguous(), normal=_get_normal(st["scaling"], st["rotation"]))
    torch.manual_seed(5)
    vis = torch.rand(P + S, device=dev) < 0.5
    shapes = dict(xyz=(P + S, 3), shs=(P + S, 16, 3), opacity=(P + S, 1), scales=(P + S, 3), rotations=(P + S, 4))
    W = {k: torch.randn(s, device=dev) * vis.view(-1, *([1] * (len(s) - 1))).float() for k, s in shapes.items()}

    def image_loss(d):
        return sum((W[k] * (d[k] ** 2 + d[k])).sum() for k in W)

    # ---- reference flow: parameters of the unstable cloud only, the stable activations are concatenated every iteration
    p = {k: torch.nn.Parameter(v.clone()) for k, v in raw.items()}
    groups = [{"params": [p[k]], "lr": LRS[g]} for k, g in (("xyz", "xyz"), ("features_dc", "f_dc"), ("features_rest", "f_rest"),
                                                          ("opacity", "opacity"), ("scaling", "scaling"), ("rotation", "rotation"))]
    ref_opt = torch.optim.Adam(groups, lr=0.0, eps=1e-15)
    for _ in range(iters):
        un = dict(xyz=p["xyz"], shs=torch.cat((p["features_dc"], p["features_rest"]), dim=1), opacity=torch.sigmoid(p["opacity"]),
                  scales=torch.exp(p["scaling"]), rotations=F.normalize(p["rotation"]))
        image_loss({k: torch.cat([un[k], frozen[k].detach()]) for k in un}).backward()
        ref_opt.step()
        ref_opt.zero_grad(set_to_none=True)

    # ---- fused flow
    conf = torch.zeros(P, device=dev)
    opt = MapOptimizer(raw["xyz"], raw["features_dc"], raw["features_rest"], raw["opacity"], raw["scaling"], raw["rotation"], LRS,
                       confidence=conf, frozen=frozen)
    d0 = opt.gaussian_data()
    assert all(d0[k].shape[0] == P + S for k in ("xyz", "opacity", "scales", "rotations", "shs", "normal"))
    snap = opt.history_snapshot()
    assert snap["xyz"].shape == (P, 3) and snap["rotation"].shape == (P, 4) and snap["features_rest"].shape == (P, 15, 3)
    radii = vis.to(torch.int32) * 3
    for _ in range(iters):
        image_loss({k: opt.gaussian_data()[k] for k in W}).backward()
        for t in (opt.xyz, opt.shs, opt.opacity, opt.scales, opt.rotations):
            t.grad[~vis] = float("nan")        # what rtg_splat_backward_visible leaves in culled rows
        opt.step(radii=radii)

    def rel(a, b):
        return float((a - b).abs().max()) / (float(b.abs().max()) + 1e-12)
    d = opt.gaussian_data()
    assert rel(d["xyz"].detach()[:P], p["xyz"].detach()) < 1e-5 and rel(opt.features_rest, p["features_rest"].detach()) < 1e-5
    assert rel(opt.scaling_raw, p["scaling"].detach()) < 1e-5 and rel(opt.rotation_raw, p["rotation"].detach()) < 1e-5
    assert rel(d["scales"].detach()[:P], torch.exp(p["scaling"].detach())) < 1e-5
    assert float((p["xyz"].detach() - raw["xyz"]).abs().max()) > 0
    for k in ("xyz", "opacity", "scales", "rotations", "shs", "normal"):        # the frozen rows never move
        assert torch.equal(d[k].detach()[P:], frozen[k]), k
    assert float(conf.max()) == iters and conf.numel() == P
    # history merge and write-back act on the optimised rows only
    opt.history_merge(snap, 0.5)
    for k in ("xyz", "shs", "rotations"):
        assert torch.equal(opt.gaussian_data()[k].detach()[P:], frozen[k]), k
    pc = opt.write_back(type("PC", (), {})())
    assert pc._xyz.shape == (P, 3) and pc._features_dc.shape == (P, 1, 3) and pc._features_rest.shape == (P, 15, 3)
    assert pc._rotation.shape == (P, 4) and pc._opacity.shape == (P, 1)
    with pytest.raises(TypeError):
        MapOptimizer(raw["xyz"], raw["features_dc"], raw["features_rest"], raw["opacity"], raw["scaling"], raw["rotation"], LRS,
                     frozen=dict(frozen, shs=frozen["shs"][:, :4]))
