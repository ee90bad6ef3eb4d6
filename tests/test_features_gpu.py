"""GPU tests of per-Gaussian feature maps (rtg_splat_features / rtg_splat_features_backward through
features.rasterize_features): against the float64 statement (oracle/features_oracle.py) on the rasterizer's test scenes,
identities with the rasterizer's own outputs and backward at 1 M Gaussians, the behaviour of the call (the eight outputs
and their gradients untouched, reproducibility, the antialiased mode, P == 0, overflow) and a short fit of features.

Ties. A pixel whose alpha, T_threshold or opaque-hit decision lies within 1e-3 of its threshold may be decided differently
in float32 and float64 (gradcheck.decision_mask flags it). Flagged pixels are left out of the map comparison and get the
upstream gradient 0 for the backward. The upstream gradients are drawn from U(0, 1), so that a row's gradient is a sum of
non-negative terms and its relative bound means what it says; the features are N(0, 1), and the map is held to a bound
on sum_g w |F|, the size of the terms it sums."""
import numpy as np
import pytest
import torch

import gradcheck as gck
import helpers
from oracle.antialias_oracle import AntialiasedOracleRender
from oracle.features_oracle import features as feature_statement
from oracle.splat_oracle import OracleRender
from rtg_slam_b200 import mapstats, rasterizer, scene
from rtg_slam_b200.features import rasterize_features
from rtg_slam_b200.optim import FusedAdam
from rtg_slam_b200.rasterizer import GaussianRasterizer, antialiased
from test_camera_grad_gpu import KW, NAMES, inputs_for
from test_raster_grad_rows_gpu import gpu_forward

pytestmark = pytest.mark.gpu

CHANNELS = (1, 3, 16, 33, 128)


@pytest.fixture(scope="module", autouse=True)
def own_capacity_checks(cuda_device):
    prev = rasterizer._state(cuda_device).mode
    rasterizer.set_capacity_checks("sync", cuda_device)
    yield
    rasterizer.set_capacity_checks(prev, cuda_device)


def tensors(inputs, dev):
    return {KW[k]: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in inputs.items()}


def mask_t(mask, dev):
    return None if mask is None else torch.from_numpy(np.ascontiguousarray(mask, dtype=np.int32)).to(dev)


CONFIGS = [("small", "sh"), ("ragged", "sh"), ("masked", "sh"), ("dense", "sh"), ("small", "colors_precomp"),
           ("ragged", "cov3D_precomp"), ("small", "antialiased"), ("masked", "antialiased")]


@pytest.mark.parametrize("name,mode", CONFIGS)
def test_matches_the_f64_statement(cuda_device, name, mode):
    dev = cuda_device
    aa = mode == "antialiased"
    cam, g, mask = gck.scene_case(name)
    inputs, over = inputs_for(g, "sh" if aa else mode)
    gg, kw = gck.oracle_args(inputs, mask, over)
    cls = AntialiasedOracleRender if aa else OracleRender
    o32, o64 = (cls(cam, gg, precision=p, tie_eps=1e-3, **kw) for p in ("f32", "f64"))
    P, H, W = len(g["xyz"]), cam.height, cam.width
    rng = np.random.default_rng(sum(map(ord, name + mode)))
    Fs = [rng.standard_normal((P, c)).astype(np.float32) for c in CHANNELS]
    Gs = [rng.uniform(0.0, 1.0, (c, H, W)).astype(np.float32) for c in CHANNELS]
    rs = helpers.make_settings(cam, dev, **over)
    with antialiased(aa):
        fwd = gpu_forward(cam, inputs, dev, mask, **over)
        dm = gck.decision_mask(cam, gg, kw, gpu_forward=fwd, oracles=(o32, o64))
        assert dm.mean() <= gck.MAX_MASKED_SHARE.get(name, 0.01), (name, int(dm.sum()), dm.size)
        got = []
        for F, G in zip(Fs, Gs):
            G[:, dm] = 0.0
            f = torch.from_numpy(F).to(dev).requires_grad_(True)
            outs, fmap = rasterize_features(rs, **tensors(inputs, dev), features=f, tile_mask=mask_t(mask, dev))
            (fmap * torch.from_numpy(G).to(dev)).sum().backward()
            got.append((fmap.detach().cpu().numpy(), f.grad.cpu().numpy()))
            for k, o in zip(NAMES, outs):   # the call's forward is the forward
                assert np.array_equal(o.detach().cpu().numpy(), fwd[k]), k
    # one walk of the statement for every channel count: the features, their magnitudes and the upstream gradients side by side
    ref = feature_statement(o64, F=np.concatenate(Fs + [np.abs(F) for F in Fs], 1), G=np.concatenate(Gs, 0))
    rows = (o64.radii > 0) & (fwd["radii"] == o64.radii)
    assert (~rows & (o64.radii > 0)).sum() <= max(1, 1e-3 * (o64.radii > 0).sum())
    c0, n_all = 0, sum(CHANNELS)
    for (m, dF), c in zip(got, CHANNELS):
        rm, rabs, rg = ref["map"][c0:c0 + c], ref["map"][n_all + c0:n_all + c0 + c], ref["grad"][:, c0:c0 + c]
        c0 += c
        keep = ~dm
        err_m = np.abs(m.astype(np.float64) - rm)[:, keep]
        tol_m = 1e-4 * rabs[:, keep] + 1e-6
        assert rabs.max() > 0.1
        r, x = rg[rows], dF[rows].astype(np.float64)
        assert r.max() > 0
        tol_g = 1e-4 * np.abs(r) + 1e-6 * np.abs(r).max()
        ratio_g = np.where(np.abs(x - r) == 0, 0.0, np.abs(x - r) / tol_g)
        print(f"{name}/{mode} C={c}: {int(dm.sum())} of {dm.size} pixels flagged; map worst ratio {(err_m / tol_m).max():.3f}, "
              f"dL/dF worst ratio {ratio_g.max():.3f} over {int(rows.sum())} rows")
        assert np.all(err_m <= tol_m), (c, (err_m / tol_m).max())
        assert np.all(ratio_g <= 1.0), (c, ratio_g.max())
        assert np.all(dF[fwd["radii"] == 0] == 0)
        if mask is not None:   # masked-out tiles are 0
            pix = np.kron(mask, np.ones((16, 16), np.int32))[:H, :W] == 0
            assert np.all(m[:, pix] == 0)


# ------------------------------------------------------------------------------------------------ at the timed sizes
@pytest.fixture(scope="module")
def room_1m(cuda_device):
    g = scene.surfel_room(1_000_000, seed=2024)
    return g, inputs_for(g, "colors_precomp")[0]


@pytest.mark.parametrize("cam_name,keep", [("replica", None), ("hd", None), ("replica", 0.5)])
def test_frame_identities_at_timed_sizes(cuda_device, room_1m, cam_name, keep):
    dev = cuda_device
    g, inputs = room_1m
    cam = scene.make_camera(cam_name)
    mask = None if keep is None else scene.random_tile_mask(cam, keep, seed=11)
    tm = mask_t(mask, dev)
    rs = helpers.make_settings(cam, dev)
    t = tensors(inputs, dev)
    P = t["means3D"].shape[0]
    # F = 1: the covered fraction 1 - T_map
    with torch.no_grad():
        outs, ones_map = rasterize_features(rs, **t, features=torch.ones((P, 1), device=dev), tile_mask=tm)
    d_T = float((ones_map[0] - (1.0 - outs[6][0])).abs().max())
    # F = the colours: the forward's colour image (background 0); C = 3 backward against the rasterizer's dL/dcolors_precomp
    cols = t.pop("colors_precomp").requires_grad_(True)
    f = cols.detach().clone().requires_grad_(True)
    outs, fmap = rasterize_features(rs, **t, colors_precomp=cols, features=f, tile_mask=tm)
    G = torch.rand((3, cam.height, cam.width), generator=torch.Generator(device=dev).manual_seed(7), device=dev)
    ((outs[0] * G).sum() + (fmap * G).sum()).backward()
    d_C = float((fmap - outs[0]).abs().max())
    radii = outs[7].cpu().numpy()
    ref, x = cols.grad.cpu().numpy().astype(np.float64), f.grad.cpu().numpy().astype(np.float64)
    vis = radii > 0
    tol = 1e-4 * np.abs(ref[vis]) + 1e-6 * np.abs(ref[vis]).max()
    d = np.abs(x[vis] - ref[vis])
    ratio = np.where(d == 0, 0.0, d / tol)
    # adjoint identity, summed in float64
    lhs = float((fmap.detach().double() * G.double()).sum())
    rhs = float((f.detach().double() * f.grad.double()).sum())
    print(f"1M {cam_name} keep {keep}: |ones - (1 - T_map)| {d_T:.2e}, |colour map - color| {d_C:.2e}, dL/dF vs "
          f"dL/dcolors_precomp worst ratio {ratio.max():.3f}, adjoint rel {abs(lhs - rhs) / abs(lhs):.2e}")
    assert d_T <= 1e-5 and d_C <= 1e-5
    assert np.all(ratio <= 1.0)
    assert np.all(x[~vis] == 0)
    assert abs(lhs - rhs) <= 1e-5 * abs(lhs)
    if mask is not None:
        pix = torch.from_numpy(np.kron(mask, np.ones((16, 16), np.int32))[:cam.height, :cam.width] == 0).to(dev)
        assert int(pix.sum()) > 0
        assert float(fmap.detach()[:, pix].abs().max()) == 0.0 and float(ones_map[:, pix].abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------ behaviour of the call
def small_inputs(dev, name="masked"):
    cam, g, mask = gck.scene_case(name)
    inputs, _ = inputs_for(g, "sh")
    return cam, g, mask, inputs


def test_outputs_and_geometry_gradients_are_the_rasterizers(cuda_device):
    """The eight outputs equal GaussianRasterizer's bit for bit; the gradients of a colour + depth + T_map loss equal its own,
    with a loss on the feature map added (which has no geometry gradient), within twice the spread between two of its
    own backwards plus 1e-6 of the largest entry (the compositing backward sums with atomics in a varying order)."""
    dev = cuda_device
    cam, g, mask, inputs = small_inputs(dev)
    rs = helpers.make_settings(cam, dev)
    tm = mask_t(mask, dev)
    gc, gd = (torch.from_numpy(a).to(dev) for a in scene.upstream_grads(cam, seed=5))
    P = len(g["xyz"])
    F = torch.randn((P, 5), generator=torch.Generator(device=dev).manual_seed(3), device=dev)
    Gf = torch.rand((5, cam.height, cam.width), generator=torch.Generator(device=dev).manual_seed(4), device=dev)

    def run(ours):
        t = {k: v.requires_grad_(True) for k, v in tensors(inputs, dev).items()}
        if ours:
            f = F.clone().requires_grad_(True)
            outs, fmap = rasterize_features(rs, **t, features=f, tile_mask=tm)
            extra = (fmap * Gf).sum()
        else:
            outs = GaussianRasterizer(rs)(**t, tile_mask=tm)
            extra = 0.0
        ((outs[0] * gc).sum() + (outs[1] * gd).sum() + outs[6].sum() + extra).backward()
        return [o.detach() for o in outs], {k: v.grad for k, v in t.items()}

    ref_o, ref_g = run(False)
    ref2_o, ref2_g = run(False)
    our_o, our_g = run(True)
    for k, a, b in zip(NAMES, ref_o, our_o):
        assert torch.equal(a, b), k
    for k in ref_g:
        spread = float((ref_g[k] - ref2_g[k]).abs().max())
        d = float((our_g[k] - ref_g[k]).abs().max())
        bound = 2 * spread + 1e-6 * float(ref_g[k].abs().max())
        print(f"d{k}: |ours - rasterizer| {d:.2e}, rasterizer run-to-run {spread:.2e}, bound {bound:.2e}")
        assert d <= bound, k


def test_forward_is_reproducible_and_needs_no_grad(cuda_device):
    dev = cuda_device
    cam, g, mask, inputs = small_inputs(dev)
    rs = helpers.make_settings(cam, dev)
    F = torch.randn((len(g["xyz"]), 33), generator=torch.Generator(device=dev).manual_seed(8), device=dev)
    _, a = rasterize_features(rs, **tensors(inputs, dev), features=F, tile_mask=mask_t(mask, dev))
    with torch.no_grad():
        _, b = rasterize_features(rs, **tensors(inputs, dev), features=F, tile_mask=mask_t(mask, dev))
    assert not a.requires_grad and a.shape == (33, cam.height, cam.width) and a.dtype == torch.float32
    assert torch.equal(a, b) and float(a.abs().max()) > 0
    # a non-contiguous feature tensor renders as its contiguous copy
    Ft = F.t().contiguous().t()
    assert not Ft.is_contiguous()
    _, c = rasterize_features(rs, **tensors(inputs, dev), features=Ft, tile_mask=mask_t(mask, dev))
    assert torch.equal(a, c)


def test_stride_zero_upstream_gives_the_contribution_weight(cuda_device):
    """feature_map.sum() sends a stride-0 gradient of ones: dL/dF[:, c] is then sum_p w, the contribution weight."""
    dev = cuda_device
    cam, g, mask, inputs = small_inputs(dev)
    rs = helpers.make_settings(cam, dev)
    f = torch.zeros((len(g["xyz"]), 2), device=dev, requires_grad=True)
    _, fmap = rasterize_features(rs, **tensors(inputs, dev), features=f, tile_mask=mask_t(mask, dev))
    fmap.sum().backward()
    _, st = mapstats.gaussian_contributions(rs, **tensors(inputs, dev), tile_mask=mask_t(mask, dev))
    w = st["weight"]
    assert float(w.max()) > 0
    for c in range(2):
        assert float((f.grad[:, c] - w).abs().max()) <= 1e-6 * float(w.max())


def test_antialiased_mode_is_honoured(cuda_device):
    dev = cuda_device
    cam, g, mask, inputs = small_inputs(dev, "small")
    rs = helpers.make_settings(cam, dev)
    ones = torch.ones((len(g["xyz"]), 1), device=dev)
    maps = {}
    for aa in (False, True):
        with antialiased(aa), torch.no_grad():
            outs, m = rasterize_features(rs, **tensors(inputs, dev), features=ones)
        maps[aa] = m
        assert float((m[0] - (1.0 - outs[6][0])).abs().max()) <= 1e-5, aa
    assert float((maps[True] - maps[False]).abs().max()) > 1e-2


def test_no_gaussians(cuda_device):
    dev = cuda_device
    cam = scene.make_camera("small")
    rs = helpers.make_settings(cam, dev)
    z = lambda *s: torch.zeros(s, device=dev)
    f = z(0, 7).requires_grad_(True)
    outs, fmap = rasterize_features(rs, z(0, 3), z(0, 1), f, shs=z(0, 16, 3), scales=z(0, 3), rotations=z(0, 4))
    assert fmap.shape == (7, cam.height, cam.width) and float(fmap.abs().max()) == 0.0
    fmap.sum().backward()
    assert f.grad.shape == (0, 7)


def test_overflow_is_reported(cuda_device):
    """In the deferred mode an overflowed forward renders an empty frame and an empty feature map; the feature backward
    raises CapacityOverflow instead of returning the zero gradient of the empty render."""
    dev = cuda_device
    cam, g, mask, inputs = small_inputs(dev, "small")
    rs = helpers.make_settings(cam, dev)
    st = rasterizer._state(dev)
    prev_mode, prev_hint = st.mode, st.r_hint
    rasterizer.set_capacity_checks("deferred", dev)
    st.r_hint = 16   # far too small: the forward overflows without waiting for its count
    try:
        f = torch.ones((len(g["xyz"]), 4), device=dev, requires_grad=True)
        outs, fmap = rasterize_features(rs, **tensors(inputs, dev), features=f)
        assert float(fmap.abs().max()) == 0.0 and float(outs[0].abs().max()) == 0.0
        with pytest.raises(rasterizer.CapacityOverflow):
            fmap.sum().backward()
        assert f.grad is None
        raised_to = st.r_hint
    finally:
        rasterizer.set_capacity_checks(prev_mode, dev)
        st.r_hint = max(st.r_hint, prev_hint)
    assert raised_to > 16
    _, again = rasterize_features(rs, **tensors(inputs, dev), features=f.detach())   # rendered again, it succeeds
    assert float(again.abs().max()) > 0


# ------------------------------------------------------------------------------------------------ a short fit
def test_features_fit_a_target_map(cuda_device):
    """Features start at 0 and fit the map rendered from known features on a fixed geometry: 150 FusedAdam steps at
    lr 0.05 on the mean squared error bring the loss down by at least 10x."""
    dev = cuda_device
    cam, g, mask, inputs = small_inputs(dev, "small")
    rs = helpers.make_settings(cam, dev)
    t = tensors(inputs, dev)
    P, Cn = len(g["xyz"]), 8
    truth = torch.randn((P, Cn), generator=torch.Generator(device=dev).manual_seed(12), device=dev)
    with torch.no_grad():
        _, target = rasterize_features(rs, **t, features=truth)
    f = torch.zeros((P, Cn), device=dev, requires_grad=True)
    opt = FusedAdam([{"params": [f], "lr": 0.05}], lr=0.0, eps=1e-15)
    losses = []
    for _ in range(150):
        opt.zero_grad()
        _, fmap = rasterize_features(rs, **t, features=f)
        loss = ((fmap - target) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    print(f"fit: loss {losses[0]:.4e} -> {losses[-1]:.4e} ({losses[0] / losses[-1]:.1f}x)")
    assert losses[-1] * 10 <= losses[0]
