"""GPU tests of the per-Gaussian contribution statistics (rtg_splat_contributions through mapstats.gaussian_contributions):
against the float64 statement (oracle/contrib_oracle.py) on the rasterizer's test scenes, the frame identities and the
agreement with the existing backward at 1 M Gaussians, and the behaviour of the call (accumulation, reproducibility, the
forward left untouched, the overflow re-render).

Ties. A pixel whose alpha, T_threshold or opaque-hit decision lies within 1e-3 of its threshold may be decided differently
in float32 and float64 (gradcheck.decision_mask flags it). Such pixels get the error e = 0, every other pixel e = 1, so
`error` is the weight over the unflagged pixels, where both sides take the same decisions; it is held per row to
|error - ref| <= 1e-4 ref + 1e-6 max(ref). n_pixels may differ from the statement only through flagged pixels: by at most
the number of flagged pixels in whose tile list the Gaussian is (a tie at the last blended entry can lengthen or shorten
the walked prefix)."""
import numpy as np
import pytest
import torch

import gradcheck as gck
import helpers
from oracle.antialias_oracle import AntialiasedOracleRender
from oracle.contrib_oracle import contributions
from oracle.splat_oracle import OracleRender
from rtg_slam_b200 import mapstats, rasterizer, scene
from rtg_slam_b200.rasterizer import antialiased
from test_camera_grad_gpu import KW, NAMES, inputs_for
from test_raster_grad_rows_gpu import gpu_forward

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def own_capacity_checks(cuda_device):
    prev = rasterizer._state(cuda_device).mode
    rasterizer.set_capacity_checks("sync", cuda_device)
    yield
    rasterizer.set_capacity_checks(prev, cuda_device)


def tensors(inputs, dev):
    return {KW[k]: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in inputs.items()}


def stats_call(cam, inputs, dev, mask=None, pixel_error=None, out=None, **over):
    rs = helpers.make_settings(cam, dev, **over)
    tm = None if mask is None else torch.from_numpy(np.ascontiguousarray(mask, dtype=np.int32)).to(dev)
    pe = None if pixel_error is None else torch.from_numpy(np.ascontiguousarray(pixel_error, dtype=np.float32)).to(dev)
    outs, st = mapstats.gaussian_contributions(rs, **tensors(inputs, dev), tile_mask=tm, pixel_error=pe, out=out)
    return dict(zip(NAMES, [o.cpu().numpy() for o in outs])), {k: v.cpu().numpy() for k, v in st.items()}


def list_counts(o, pixels):
    """Per Gaussian: the pixels of `pixels` (boolean (H, W)) in whose tile list it is."""
    pl, rg = o.binning()
    tw = (o.W + 15) // 16
    ys, xs = np.nonzero(pixels)
    per_tile = np.bincount((ys // 16) * tw + xs // 16, minlength=len(rg))
    out = np.zeros(o.P, np.int64)
    for t in np.nonzero(per_tile)[0]:
        np.add.at(out, pl[rg[t, 0]:rg[t, 1]], per_tile[t])
    return out


CONFIGS = [("small", "sh"), ("ragged", "sh"), ("masked", "sh"), ("dense", "sh"), ("small", "colors_precomp"),
           ("ragged", "cov3D_precomp"), ("small", "antialiased"), ("masked", "antialiased")]


@pytest.mark.parametrize("name,mode", CONFIGS)
def test_matches_the_f64_statement(cuda_device, name, mode):
    aa = mode == "antialiased"
    cam, g, mask = gck.scene_case(name)
    inputs, over = inputs_for(g, "sh" if aa else mode)
    gg, kw = gck.oracle_args(inputs, mask, over)
    cls = AntialiasedOracleRender if aa else OracleRender
    o32, o64 = (cls(cam, gg, precision=p, tie_eps=1e-3, **kw) for p in ("f32", "f64"))
    with antialiased(aa):
        fwd = gpu_forward(cam, inputs, cuda_device, mask, **over)
        dm = gck.decision_mask(cam, gg, kw, gpu_forward=fwd, oracles=(o32, o64))
        assert dm.mean() <= gck.MAX_MASKED_SHARE.get(name, 0.01), (name, int(dm.sum()), dm.size)
        e = (~dm).astype(np.float32)
        outs, st = stats_call(cam, inputs, cuda_device, mask, pixel_error=e, **over)
    for k in NAMES:   # the stats call's forward is the forward
        assert np.array_equal(outs[k], fwd[k]), k
    ref = contributions(o64, e, pixels=dm)
    rows = (o64.radii > 0) & (fwd["radii"] == o64.radii)
    assert (~rows & (o64.radii > 0)).sum() <= max(1, 1e-3 * (o64.radii > 0).sum())
    assert np.all(st["n_pixels"][fwd["radii"] == 0] == 0) and np.all(st["weight"][fwd["radii"] == 0] == 0)
    r, x = ref["error"][rows], st["error"][rows].astype(np.float64)
    assert r.max() > 0
    tol = 1e-4 * r + 1e-6 * r.max()
    ratio = np.where(np.abs(x - r) == 0, 0.0, np.abs(x - r) / tol)
    dn = np.abs(st["n_pixels"].astype(np.int64) - ref["n_pixels"])[rows]
    allow = list_counts(o64, dm)[rows]
    strict = ref["in_prefix"][rows]
    print(f"{name}/{mode}: {int(dm.sum())} of {dm.size} pixels flagged, {int(rows.sum())} rows; error worst ratio "
          f"{ratio.max():.3f}; n_pixels differs on {int((dn > 0).sum())} rows (max {int(dn.max())}), beyond the flagged "
          f"prefix count on {int((dn > strict).sum())}; pairs {int(st['n_pixels'].sum())} vs {int(ref['n_pixels'].sum())}")
    assert np.all(ratio <= 1.0), (ratio.max(), np.argmax(ratio))
    assert np.all(dn <= allow), np.nonzero(dn > allow)[0][:10]


# ------------------------------------------------------------------------------------------------ at the timed sizes
@pytest.fixture(scope="module")
def room_1m(cuda_device):
    g = scene.surfel_room(1_000_000, seed=2024)
    return g, tensors(inputs_for(g, "sh")[0], cuda_device)


def frame_checks(cam, g_t, dev, mask, label):
    rs = helpers.make_settings(cam, dev)
    tm = None if mask is None else torch.from_numpy(mask).to(dev)
    outs, st = mapstats.gaussian_contributions(rs, **g_t, tile_mask=tm)
    n, w = st["n_pixels"].cpu().numpy().astype(np.int64), st["weight"].cpu().numpy().astype(np.float64)
    T = outs[6].cpu().numpy().astype(np.float64)
    hc, hcw, radii = outs[2].cpu().numpy().reshape(-1), outs[4].cpu().numpy().reshape(-1).astype(np.float64), outs[7].cpu().numpy()
    lhs, rhs = w.sum(), (1.0 - T).sum()
    rel = abs(lhs - rhs) / rhs
    won = hcw > 0   # a pixel with a colour contribution: its hit_color is the arg-max Gaussian
    wins = np.bincount(hc[won], minlength=len(n))
    win_w = np.bincount(hc[won], weights=hcw[won], minlength=len(n))
    print(f"{label}: sum weight {lhs:.6f} vs sum (1 - T_map) {rhs:.6f} (rel {rel:.2e}); {int((n > 0).sum())} of "
          f"{int((radii > 0).sum())} visible Gaussians add colour; {int(n.sum())} pairs")
    assert rel <= 1e-5
    assert np.all(n >= wins)
    assert np.all(w >= win_w * (1 - 1e-6))
    assert np.all(n[radii == 0] == 0) and np.all(w[radii == 0] == 0)
    return rs, tm


@pytest.mark.parametrize("cam_name,keep", [("replica", None), ("hd", None), ("replica", 0.5)])
def test_frame_identities_at_timed_sizes(cuda_device, room_1m, cam_name, keep):
    g, g_t = room_1m
    cam = scene.make_camera(cam_name)
    mask = None if keep is None else scene.random_tile_mask(cam, keep, seed=11)
    frame_checks(cam, g_t, cuda_device, mask, f"1M {cam_name} keep {keep}")


@pytest.mark.parametrize("cam_name,keep", [("replica", None), ("hd", 0.5)])
def test_error_is_the_backward_colour_gradient_at_timed_sizes(cuda_device, room_1m, cam_name, keep):
    """dL/dcolors_precomp[:, 0] of the existing backward under dL/dcolor = (e, 0, 0), random colours on the same geometry."""
    from rtg_slam_b200.rasterizer import GaussianRasterizer
    g, _ = room_1m
    dev = cuda_device
    cam = scene.make_camera(cam_name)
    mask = None if keep is None else scene.random_tile_mask(cam, keep, seed=11)
    inputs, _ = inputs_for(g, "colors_precomp")
    rng = np.random.default_rng(7)
    e = rng.uniform(0.0, 1.0, (cam.height, cam.width)).astype(np.float32)
    _, st = stats_call(cam, inputs, dev, mask, pixel_error=e)
    rs = helpers.make_settings(cam, dev)
    t = tensors(inputs, dev)
    t["colors_precomp"].requires_grad_(True)
    tm = None if mask is None else torch.from_numpy(mask).to(dev)
    out = GaussianRasterizer(rs)(**t, tile_mask=tm)
    (out[0][0] * torch.from_numpy(e).to(dev)).sum().backward()
    ref = t["colors_precomp"].grad[:, 0].cpu().numpy().astype(np.float64)
    x = st["error"].astype(np.float64)
    rows = out[7].cpu().numpy() > 0
    tol = 1e-4 * np.abs(ref[rows]) + 1e-6 * np.abs(ref[rows]).max()
    d = np.abs(x[rows] - ref[rows])
    ratio = np.where(d == 0, 0.0, d / tol)
    print(f"1M {cam_name} keep {keep}: error vs backward colour gradient, worst ratio {ratio.max():.3f}")
    assert np.all(ratio <= 1.0)
    assert np.all(x[~rows] == 0)


# ------------------------------------------------------------------------------------------------ behaviour of the call
def test_accumulates_reproduces_and_leaves_the_forward_alone(cuda_device):
    cam, g, mask = gck.scene_case("masked")
    inputs, _ = inputs_for(g, "sh")
    e = np.random.default_rng(9).uniform(0.0, 1.0, (cam.height, cam.width)).astype(np.float32)
    fwd = gpu_forward(cam, inputs, cuda_device, mask)
    outs_a, a = stats_call(cam, inputs, cuda_device, mask, pixel_error=e)
    outs_b, b = stats_call(cam, inputs, cuda_device, mask, pixel_error=e)
    for k in NAMES:
        assert np.array_equal(outs_a[k], fwd[k]) and np.array_equal(outs_b[k], fwd[k]), k
    assert np.array_equal(a["n_pixels"], b["n_pixels"])   # counts are exact
    P = len(g["xyz"])
    acc = {"n_pixels": torch.zeros(P, dtype=torch.int32, device=cuda_device),
           "weight": torch.zeros(P, dtype=torch.float32, device=cuda_device),
           "error": torch.zeros(P, dtype=torch.float32, device=cuda_device)}
    e2 = (e * 0.5).astype(np.float32)
    _, c = stats_call(cam, inputs, cuda_device, mask, pixel_error=e2)
    stats_call(cam, inputs, cuda_device, mask, pixel_error=e, out=acc)
    _, s = stats_call(cam, inputs, cuda_device, mask, pixel_error=e2, out=acc)
    assert np.array_equal(s["n_pixels"], a["n_pixels"] + c["n_pixels"])
    for k in ("weight", "error"):
        assert np.allclose(s[k], a[k] + c[k], rtol=1e-6, atol=1e-7 * np.abs(a[k]).max()), k
    assert a["n_pixels"].sum() > 0 and np.abs(a["weight"] - b["weight"]).max() <= 1e-6 * a["weight"].max()
    with pytest.raises(ValueError):
        stats_call(cam, inputs, cuda_device, mask, out={"n_pixels": acc["n_pixels"], "weight": acc["weight"]}, pixel_error=e)
    with pytest.raises(ValueError):
        stats_call(cam, inputs, cuda_device, mask, out={"n_pixels": acc["weight"], "weight": acc["weight"]})


def test_an_overflowed_forward_is_rendered_again(cuda_device):
    cam, g, mask = gck.scene_case("small")
    inputs, _ = inputs_for(g, "sh")
    _, want = stats_call(cam, inputs, cuda_device, mask)
    st = rasterizer._state(cuda_device)
    prev_mode, prev_hint = st.mode, st.r_hint
    rasterizer.set_capacity_checks("deferred", cuda_device)
    st.r_hint = 16   # far too small: the first forward overflows without waiting for its count
    try:
        _, got = stats_call(cam, inputs, cuda_device, mask)
        raised_to = st.r_hint
    finally:
        rasterizer.set_capacity_checks(prev_mode, cuda_device)
        st.r_hint = max(st.r_hint, prev_hint)
    assert raised_to > 16
    assert np.array_equal(got["n_pixels"], want["n_pixels"]) and got["n_pixels"].sum() > 0
