"""GPU tests of the feature map's weight gradient (rtg_splat_features_backward_geometry through
rasterize_features(weight_grad=True)): per Gaussian against the float64 statement (oracle/feature_weights_oracle.py) on the
rasterizer's test scenes, identities with the rasterizer's own colour and T_map backwards at 1 M Gaussians, the behaviour
of the option, and expected depth (F = (z_view, 1)) against the statement and as a pose-refinement loss.

The per-row metric is gradcheck.check_rows at the rasterizer backward's bounds (RTOL 1e-3, C 5e-6, widened only to 10 x
the call's own run-to-run spread); the camera gradient is held to test_camera_grad_gpu.py's tolerance (per block
max|g - ref| / max|ref| below max(1e-3, 10 x run-to-run)). Pixels within 1e-3 of a decision threshold get the upstream
gradient 0 (gradcheck.decision_mask). The compositing sums are float atomics in a varying order, so two runs of any
backward differ in the last bits: where the code paths are the same, "equal" below means within that spread."""
import numpy as np
import pytest
import torch

import gradcheck as gck
import helpers
from oracle.antialias_oracle import AntialiasedOracleRender
from oracle.feature_weights_oracle import weight_gradient
from oracle.features_oracle import features as feature_statement
from oracle.splat_oracle import OracleRender
from rtg_slam_b200 import features as features_mod
from rtg_slam_b200 import rasterizer, scene
from rtg_slam_b200.features import rasterize_features
from rtg_slam_b200.rasterizer import GaussianRasterizer, antialiased, visible_rows_only
from test_camera_grad_gpu import CAM, KW, inputs_for, pose_error, se3_exp
from test_raster_grad_rows_gpu import gpu_forward

pytestmark = pytest.mark.gpu

CHANNELS = (1, 3, 16, 33, 128)


@pytest.fixture(scope="module", autouse=True)
def own_capacity_checks(cuda_device):
    prev = rasterizer._state(cuda_device).mode
    rasterizer.set_capacity_checks("sync", cuda_device)
    yield
    rasterizer.set_capacity_checks(prev, cuda_device)


def tensors(inputs, dev, grad=False):
    return {KW[k]: torch.from_numpy(np.ascontiguousarray(v)).to(dev).requires_grad_(grad and k != "shs") for k, v in inputs.items()}


def mask_t(mask, dev):
    return None if mask is None else torch.from_numpy(np.ascontiguousarray(mask, dtype=np.int32)).to(dev)


def statement(cam, gg, kw, F, G, aa=False, camera=False):
    kw = dict(kw)
    kw.pop("colors_precomp", None)
    return weight_gradient(cam, gg, F, G, tile_mask=kw.pop("tile_mask", None), cov3D_precomp=kw.pop("cov3D_precomp", None),
                           antialiased=aa, camera=camera, **kw)


def run(rs, inputs, dev, F, G, mask=None, camera=False, aa=False):
    """Forward + backward of <G, feature map> with weight_grad: ({geometry gradients}, {camera gradients} or None)."""
    t = tensors(inputs, dev, grad=True)
    if camera:
        rs = rs._replace(**{k: getattr(rs, k).detach().clone().requires_grad_(True) for k in CAM})
    with antialiased(aa):
        _, fmap = rasterize_features(rs, **t, features=torch.from_numpy(F).to(dev), tile_mask=mask_t(mask, dev),
                                     weight_grad=True)
    (fmap * torch.from_numpy(G).to(dev)).sum().backward()
    geo = {k: v.grad.cpu().numpy() for k, v in t.items() if v.requires_grad}
    cams = {k: getattr(rs, k).grad.cpu().numpy() for k in CAM} if camera else None
    return geo, cams


def rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


CONFIGS = [("small", "sh"), ("ragged", "sh"), ("masked", "sh"), ("dense", "sh"), ("axis_room", "sh"),
           ("small", "cov3D_precomp"), ("small", "antialiased"), ("masked", "antialiased")]
CAMERA_CONFIGS = {("small", "sh"), ("masked", "sh"), ("small", "cov3D_precomp"), ("small", "antialiased")}


@pytest.mark.parametrize("name,mode", CONFIGS)
def test_rows_match_the_f64_statement(cuda_device, name, mode):
    dev = cuda_device
    aa = mode == "antialiased"
    cam, g, mask = gck.scene_case(name)
    inputs, over = inputs_for(g, "sh" if aa else mode)
    gg, kw = gck.oracle_args(inputs, mask, over)
    cls = AntialiasedOracleRender if aa else OracleRender
    o32, o64 = (cls(cam, gg, precision=p, tie_eps=1e-3, **kw) for p in ("f32", "f64"))
    P, H, W = len(g["xyz"]), cam.height, cam.width
    rs = helpers.make_settings(cam, dev, **over)
    with antialiased(aa):
        fwd = gpu_forward(cam, inputs, dev, mask, **over)
    dm = gck.decision_mask(cam, gg, kw, gpu_forward=fwd, oracles=(o32, o64))
    assert dm.mean() <= gck.MAX_MASKED_SHARE.get(name, 0.01), (name, int(dm.sum()), dm.size)
    rows, excluded = gck.comparable_rows(cam, gg, kw, o32, o64, gpu_radii=fwd["radii"])
    camera = (name, mode) in CAMERA_CONFIGS
    rng = np.random.default_rng(sum(map(ord, name + mode)))
    for c in CHANNELS:
        F = rng.standard_normal((P, c)).astype(np.float32)
        G = rng.uniform(0.0, 1.0, (c, H, W)).astype(np.float32) / (H * W)
        G[:, dm] = 0.0
        a, ca = run(rs, inputs, dev, F, G, mask, camera, aa)
        b, cb = run(rs, inputs, dev, F, G, mask, camera, aa)
        ref, rc = statement(cam, gg, kw, F, G, aa, camera)
        assert set(a) == set(ref), (set(a), set(ref))
        gck.check_rows(f"{name}/{mode} C={c}", a, ref, rows, o64, gg, again=b)
        for k, v in a.items():
            assert np.all(v[fwd["radii"] == 0] == 0), k
        if camera:
            for k in CAM:
                if k == "campos":   # the map reads no colour
                    assert np.all(ca[k] == 0) and np.all(rc[k] == 0)
                    continue
                err, jit = rel(ca[k], rc[k]), rel(cb[k], ca[k])
                print(f"  d{k}: rel err {err:.2e}, run-to-run {jit:.2e}")
                assert err < max(1e-3, 10 * jit), (k, err, jit)
    print(f"{name}/{mode}: {int(dm.sum())} pixels masked, {int(rows.sum())} rows compared, left out {excluded}")


# ------------------------------------------------------------------------------------------------ at the timed sizes
@pytest.fixture(scope="module")
def room_1m():
    g = scene.surfel_room(1_000_000, seed=2024)
    return g, inputs_for(g, "colors_precomp")[0]


def rasterizer_grads(rs, t, tm, loss_of):
    rs = rs._replace(**{k: getattr(rs, k).detach().clone().requires_grad_(True) for k in CAM})
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in t.items()}
    outs = GaussianRasterizer(rs)(**leaves, tile_mask=tm)
    loss_of(outs).backward()
    out = {k: v.grad for k, v in leaves.items() if k != "colors_precomp"}
    out.update({k: getattr(rs, k).grad for k in CAM})
    return out


def feature_grads(rs, t, tm, F, G):
    rs = rs._replace(**{k: getattr(rs, k).detach().clone().requires_grad_(True) for k in CAM})
    leaves = {k: v.detach().clone().requires_grad_(k != "colors_precomp") for k, v in t.items()}
    _, fmap = rasterize_features(rs, **leaves, features=F, tile_mask=tm, weight_grad=True)
    (fmap * G).sum().backward()
    out = {k: v.grad for k, v in leaves.items() if k != "colors_precomp"}
    out.update({k: getattr(rs, k).grad for k in CAM})
    return out


@pytest.mark.parametrize("cam_name,keep", [("replica", None), ("hd", None), ("replica", 0.5)])
def test_identities_with_the_rasterizer_backward(cuda_device, room_1m, cam_name, keep):
    """C = 3 with F = colors_precomp is the colour backward with dL/dcolor = G (bg 0, no depth term); C = 1 with F = 1 is
    the T_map backward with dL/dT = -G. Geometry and camera gradients within 10 x the rasterizer's run-to-run spread, or
    2e-5 of the tensor's largest entry where that is larger: the two backwards form dL/dalpha in different orders (back
    to front in float, front to back from a double suffix sum), so they differ by the float rounding of the per-pair terms,
    which on the T_map path is above the jitter of the atomics (measured on an H100 80GB HBM3 at 700 W: at most 6.5e-6 of
    the largest entry, dL/drotations of the T_map case at 1920x1080)."""
    dev = cuda_device
    g, inputs = room_1m
    cam = scene.make_camera(cam_name)
    mask = None if keep is None else scene.random_tile_mask(cam, keep, seed=11)
    tm = mask_t(mask, dev)
    rs = helpers.make_settings(cam, dev)
    t = tensors(inputs, dev)
    P = t["means3D"].shape[0]
    G = torch.rand((3, cam.height, cam.width), generator=torch.Generator(device=dev).manual_seed(7), device=dev)
    cases = {
        "colour": (t["colors_precomp"], G, lambda o: (o[0] * G).sum()),
        "T_map": (torch.ones((P, 1), device=dev), G[:1], lambda o: -(o[6] * G[:1]).sum()),
    }
    for label, (F, Gf, loss_of) in cases.items():
        ref, ref2 = rasterizer_grads(rs, t, tm, loss_of), rasterizer_grads(rs, t, tm, loss_of)
        ours = feature_grads(rs, t, tm, F, Gf)
        for k in ref:
            spread = float((ref[k] - ref2[k]).abs().max())
            d = float((ours[k] - ref[k]).abs().max())
            print(f"1M {cam_name} keep {keep} {label} d{k}: |ours - rasterizer| {d:.2e}, rasterizer run-to-run {spread:.2e}, "
                  f"max {float(ref[k].abs().max()):.2e}")
            assert d <= max(10 * spread, 2e-5 * float(ref[k].abs().max())), (label, k, d, spread)


# ------------------------------------------------------------------------------------------------ behaviour
def small(dev, name="masked"):
    cam, g, mask = gck.scene_case(name)
    inputs, _ = inputs_for(g, "sh")
    return cam, g, mask, inputs, helpers.make_settings(cam, dev), mask_t(mask, dev)


def test_default_is_unchanged(cuda_device):
    """weight_grad=False (the default) is the feature node of before: the same map bit for bit, no gradient to the
    geometry, and the same dL/dF as an explicit False."""
    dev = cuda_device
    cam, g, mask, inputs, rs, tm = small(dev)
    F = torch.randn((len(g["xyz"]), 5), generator=torch.Generator(device=dev).manual_seed(3), device=dev)
    Gf = torch.rand((5, cam.height, cam.width), generator=torch.Generator(device=dev).manual_seed(4), device=dev)
    res = []
    for kw in ({}, {"weight_grad": False}, {"weight_grad": True}):
        t = tensors(inputs, dev, grad=True)
        f = F.clone().requires_grad_(True)
        outs, fmap = rasterize_features(rs, **t, features=f, tile_mask=tm, **kw)
        (fmap * Gf).sum().backward()
        res.append((fmap.detach(), f.grad, {k: v.grad for k, v in t.items() if v.requires_grad}, outs))
    (m0, f0, g0, o0), (m1, f1, g1, o1), (m2, f2, g2, o2) = res
    assert torch.equal(m0, m1) and torch.equal(m0, m2)
    for a, b, c in zip(o0, o1, o2):
        assert torch.equal(a.detach(), b.detach()) and torch.equal(a.detach(), c.detach())
    assert all(v is None for v in g0.values()) and all(v is None for v in g1.values())
    assert all(v is not None and float(v.abs().max()) > 0 for v in g2.values())
    assert float((f0 - f1).abs().max()) <= 1e-6 * float(f0.abs().max())
    assert float((f0 - f2).abs().max()) <= 1e-6 * float(f0.abs().max())


def test_loss_without_the_map_and_sum_of_losses(cuda_device):
    """A loss that does not touch the map gets the rasterizer's gradients alone (the feature node does not run); a colour
    loss plus a feature loss gets the sum of the two."""
    dev = cuda_device
    cam, g, mask, inputs, rs, tm = small(dev)
    gc = torch.from_numpy(scene.upstream_grads(cam, seed=5)[0]).to(dev)
    F = torch.randn((len(g["xyz"]), 4), generator=torch.Generator(device=dev).manual_seed(3), device=dev)
    Gf = torch.rand((4, cam.height, cam.width), generator=torch.Generator(device=dev).manual_seed(4), device=dev) / 1e4

    def grads(colour, feature, weight_grad=True, via_features=True):
        t = tensors(inputs, dev, grad=True)
        if via_features:
            outs, fmap = rasterize_features(rs, **t, features=F, tile_mask=tm, weight_grad=weight_grad)
        else:
            outs, fmap = GaussianRasterizer(rs)(**t, tile_mask=tm), None
        loss = (outs[0] * gc).sum() * colour + ((fmap * Gf).sum() if feature else 0.0)
        loss.backward()
        return {k: v.grad for k, v in t.items() if v.requires_grad}

    ras, ras2 = grads(1, 0, via_features=False), grads(1, 0, via_features=False)
    no_map = grads(1, 0)
    feat, feat2, both = grads(0, 1), grads(0, 1), grads(1, 1)
    for k in ras:
        spread = float((ras[k] - ras2[k]).abs().max())
        fspread = float((feat[k] - feat2[k]).abs().max())
        d0 = float((no_map[k] - ras[k]).abs().max())
        d1 = float((both[k] - (ras[k] + feat[k])).abs().max())
        print(f"d{k}: no map {d0:.2e}, sum {d1:.2e}, run-to-run rasterizer {spread:.2e}, feature {fspread:.2e}")
        assert d0 <= 2 * spread + 1e-6 * float(ras[k].abs().max()), k
        assert d1 <= 2 * (spread + fspread) + 1e-6 * float(both[k].abs().max()), k
        assert float(feat[k].abs().max()) > 0


class _Spy:
    """Stands in for the library: records the arguments of rtg_splat_features_backward_geometry."""

    def __init__(self, lib):
        self.lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self.lib, name)
        if name != "rtg_splat_features_backward_geometry":
            return fn

        def wrapped(*a):
            self.calls.append(a)
            return fn(*a)
        return wrapped


def test_pose_only_and_visible_rows(cuda_device, monkeypatch):
    """Only the camera requires grad: the camera gradient of the full path, with no per-Gaussian output passed down.
    visible_rows_only: the flag is passed down and the visible rows are the dense call's."""
    dev = cuda_device
    cam, g, mask, inputs, rs, tm = small(dev)
    F = torch.randn((len(g["xyz"]), 3), generator=torch.Generator(device=dev).manual_seed(3), device=dev)
    Gf = torch.rand((3, cam.height, cam.width), generator=torch.Generator(device=dev).manual_seed(4), device=dev) / 1e4
    spy = _Spy(features_mod._lib.lib())
    monkeypatch.setattr(features_mod._lib, "lib", lambda: spy)

    def go(gaussians, vis=False):
        r = rs._replace(**{k: getattr(rs, k).detach().clone().requires_grad_(True) for k in CAM})
        t = tensors(inputs, dev, grad=gaussians)
        with visible_rows_only(vis):
            _, fmap = rasterize_features(r, **t, features=F, tile_mask=tm, weight_grad=True)
            (fmap * Gf).sum().backward()
        return {k: getattr(r, k).grad for k in CAM}, {k: v.grad for k, v in t.items() if v.requires_grad}, spy.calls[-1]

    full, gfull, call_full = go(True)
    full2, _, _ = go(True)
    pose, gpose, call_pose = go(False)
    assert not gpose and all(a is None for a in call_pose[16:21]) and call_pose[22] is not None
    assert all(a is not None for a in call_full[16:19])
    for k in ("viewmatrix", "projmatrix"):
        jit = float((full2[k] - full[k]).abs().max())
        d = float((pose[k] - full[k]).abs().max())
        assert d <= max(10 * jit, 1e-6 * float(full[k].abs().max())), (k, d, jit)
    _, gvis, call_vis = go(True, vis=True)
    assert call_vis[21] == 1 and call_full[21] == 0
    radii = gpu_forward(cam, inputs, dev, mask)["radii"]
    vis = torch.from_numpy(radii > 0).to(dev)
    for k, v in gvis.items():
        ref = gfull[k]
        assert float((v[vis] - ref[vis]).abs().max()) <= 1e-5 * float(ref.abs().max()), k


def test_no_gaussians_overflow_and_record_hook(cuda_device):
    dev = cuda_device
    cam = scene.make_camera("small")
    rs = helpers.make_settings(cam, dev)
    z = lambda *s: torch.zeros(s, device=dev, requires_grad=True)
    m, o, s, r = z(0, 3), z(0, 1), z(0, 3), z(0, 4)
    f = z(0, 2)
    _, fmap = rasterize_features(rs, m, o, f, shs=torch.zeros((0, 16, 3), device=dev), scales=s, rotations=r, weight_grad=True)
    fmap.sum().backward()
    assert m.grad.shape == (0, 3) and o.grad.shape == (0, 1) and f.grad.shape == (0, 2)

    cam, g, mask, inputs, rs, tm = small(dev, "small")
    st = rasterizer._state(dev)
    prev_mode, prev_hint = st.mode, st.r_hint
    rasterizer.set_capacity_checks("deferred", dev)
    st.r_hint = 16   # far too small: the forward overflows without waiting for its count
    try:
        t = tensors(inputs, dev, grad=True)
        _, fmap = rasterize_features(rs, **t, features=torch.ones((len(g["xyz"]), 2), device=dev), weight_grad=True)
        with pytest.raises(rasterizer.CapacityOverflow):
            fmap.sum().backward()
        assert t["means3D"].grad is None
    finally:
        rasterizer.set_capacity_checks(prev_mode, dev)
        st.r_hint = max(st.r_hint, prev_hint)

    prev = rasterizer.set_grad_record_hook(lambda rec: None)
    try:
        t = tensors(inputs, dev, grad=True)
        _, fmap = rasterize_features(rs, **t, features=torch.ones((len(g["xyz"]), 2), device=dev), weight_grad=True)
        with pytest.raises(RuntimeError, match="exchange hook"):
            fmap.sum().backward()
    finally:
        rasterizer.set_grad_record_hook(prev)


# ------------------------------------------------------------------------------------------------ expected depth
def z_view(means, vm):
    """View-space depth of each centre: the third column of the row-vector view transform."""
    return means @ vm[:3, 2] + vm[3, 2]


def test_expected_depth_recipe_matches_the_statement(cuda_device):
    """depth = map[0] / map[1] of F = (z_view, 1), an L1 loss against a shifted target: the means' gradient (through the
    weights and through z_view) and the other rows against the float64 statement plus dL/dF chained through z_view."""
    dev = cuda_device
    cam, g, mask = gck.scene_case("small")
    inputs, over = inputs_for(g, "sh")
    gg, kw = gck.oracle_args(inputs, mask, over)
    o32, o64 = (OracleRender(cam, gg, precision=p, tie_eps=1e-3, **kw) for p in ("f32", "f64"))
    fwd = gpu_forward(cam, inputs, dev, mask)
    dm = torch.from_numpy(gck.decision_mask(cam, gg, kw, gpu_forward=fwd, oracles=(o32, o64))).to(dev)
    rows, _ = gck.comparable_rows(cam, gg, kw, o32, o64, gpu_radii=fwd["radii"])
    rs = helpers.make_settings(cam, dev)

    def once():
        t = tensors(inputs, dev, grad=True)
        Fz = torch.stack([z_view(t["means3D"], rs.viewmatrix), torch.ones_like(t["means3D"][:, 0])], 1)
        _, fmap = rasterize_features(rs, **t, features=Fz, weight_grad=True)
        fmap.retain_grad()
        depth = fmap[0] / fmap[1].clamp_min(1e-6)
        keep = (fmap[1].detach() > 0.5) & ~dm
        ((depth - 2.0).abs() * keep).sum().div(cam.width * cam.height).backward()
        return {k: v.grad.cpu().numpy() for k, v in t.items() if v.requires_grad}, fmap.grad.cpu().numpy(), Fz.detach()

    a, G, Fz = once()
    b, _, _ = once()
    Fz = Fz.cpu().numpy().astype(np.float64)
    ref, _ = statement(cam, gg, kw, Fz, G)
    dF = feature_statement(o64, G=G)["grad"]
    ref["means3D"] = ref["means3D"] + dF[:, :1] * rs.viewmatrix[:3, 2].cpu().numpy().astype(np.float64)[None]
    gck.check_rows("expected depth", a, ref, rows, o64, gg, again=b)


def test_expected_depth_refines_the_pose_with_adam(cuda_device):
    """Target: the expected depth at a pose. Start 1 deg / 2 cm away (test_camera_grad_gpu's offset); Adam (lr 1e-3, 150
    steps) on a twist of the pose through the settings' camera tensors, L1 on expected depth only (the map frozen: the
    pose-only pass). Both errors must fall below a fifth of their start."""
    dev = cuda_device
    cam = scene.make_camera("small")
    g = {k: torch.from_numpy(v).to(dev) for k, v in scene.surfel_room(20_000, seed=7).items()}
    proj = torch.from_numpy(np.ascontiguousarray(cam.projection)).to(dev)
    base = helpers.make_settings(cam, dev)

    def expected_depth(w2c):
        vm = w2c.transpose(0, 1)
        rs = base._replace(viewmatrix=vm, projmatrix=vm @ proj, campos=torch.linalg.inv(w2c)[:3, 3])
        F = torch.stack([z_view(g["xyz"], vm), torch.ones_like(g["xyz"][:, 0])], 1)
        _, fmap = rasterize_features(rs, g["xyz"], g["opacity"], F, shs=g["shs"], scales=g["scales"],
                                     rotations=g["rotations"], weight_grad=True)
        return fmap[0] / fmap[1].clamp_min(1e-6), fmap[1]

    w2c_true = torch.from_numpy(np.linalg.inv(scene.small_pose()).astype(np.float32)).to(dev)
    with torch.no_grad():
        tgt, cover = expected_depth(w2c_true)
        valid = cover > 0.5
    off = torch.tensor([0.012, -0.010, 0.012, 0.010, -0.012, 0.008], device=dev)  # 2 cm, 1.0 deg
    w2c0 = se3_exp(off) @ w2c_true
    ang0, tr0 = pose_error(w2c0, w2c_true)
    xi = torch.zeros(6, device=dev, requires_grad=True)
    opt = torch.optim.Adam([xi], lr=1e-3)
    for _ in range(150):
        opt.zero_grad()
        d, _ = expected_depth(se3_exp(xi) @ w2c0)
        (d - tgt).abs()[valid].mean().backward()
        opt.step()
    with torch.no_grad():
        ang, tr = pose_error(se3_exp(xi) @ w2c0, w2c_true)
    print(f"expected-depth pose refinement: rotation {ang0:.3f} -> {ang:.3f} deg ({ang / ang0:.3f}), translation "
          f"{100 * tr0:.2f} -> {100 * tr:.2f} cm ({tr / tr0:.3f})")
    assert ang < 0.2 * ang0 and tr < 0.2 * tr0, (ang0, ang, tr0, tr)
