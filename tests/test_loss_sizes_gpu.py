"""GPU tests of the three frame losses (rtg_loss_l1, rtg_loss_l1_exposure, rtg_loss_mapping with the cosine normal term)
against their float64 statement (test_pose_exposure_cpu.loss_statement), through the C entry points, at every frame size
from one pixel to 1920x1080: the reduce and gradient kernels cap their grid at RTG_LOSS_MAX_BLOCKS x 256 = 270,336 pixels,
so 640x480 and up make a second grid-stride pass. Both layouts of the measured colour, with and without a render mask;
two calls give the same bits. Then the losses with nothing selected: an all-zero mask, no valid gt depth, no gt normal,
and the mapping loss without its normal weight."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_pose_exposure_cpu import loss_statement, mapping_frame

pytestmark = pytest.mark.gpu

SIZES = [(1, 1), (5, 7), (16, 16), (480, 640), (680, 1200), (1080, 1920)]
FORMS = ["l1", "exposure", "mapping"]
AB = (0.15, -0.03)                      # the exposure of the exposure form: residuals of either sign, mostly positive
WEIGHTS = dict(color_weight=0.8, depth_weight=1.0, normal_weight=0.1, depth_error_max=0.1)


def frame(dev, H, W, seed, channels_last=True, masked=False):
    """mapping_frame on the device in float32, the measured colour (H,W,3) or (3,H,W), and a 60 % render mask or None."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    render, depth, normal, depth_index, gt_color, gt_depth, gt_normal = mapping_frame(H, W, gen, torch.float32)
    if not channels_last:
        gt_color = gt_color.permute(2, 0, 1).contiguous()
    mask = (torch.rand(H, W, generator=gen, device=dev) < 0.6) if masked else None
    return dict(render=render, depth=depth, normal=normal, depth_index=depth_index, gt_color=gt_color, gt_depth=gt_depth,
                gt_normal=gt_normal, mask=mask)


def loss_call(form, f, ab=AB, normal_weight=WEIGHTS["normal_weight"]):
    """One call of the form's entry point on frame f. Every output starts as NaN. Returns parts (4 or 8), dL/dC (3,H,W),
    dL/ddepth (1,H,W), dL/dnormal (3,H,W) or None, dL/d(a, b) (2) or None, all on the device."""
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    dev = f["render"].device
    _, H, W = f["render"].shape
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    nan = lambda t: torch.full_like(t, float("nan"))
    g_color, g_depth = nan(f["render"]), nan(f["depth"])
    g_normal = nan(f["render"]) if form == "mapping" else None
    parts = torch.full((8 if form == "mapping" else 4,), float("nan"), device=dev)
    mask = None if f["mask"] is None else f["mask"].to(torch.uint8).contiguous()
    channels_last = int(tuple(f["gt_color"].shape) == (H, W, 3))
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    cw, dw, dem = WEIGHTS["color_weight"], WEIGHTS["depth_weight"], WEIGHTS["depth_error_max"]
    frame_args = (p(f["gt_color"]), p(f["gt_depth"]))
    if form == "mapping":
        ws = torch.zeros(L.rtg_loss_workspace_bytes(), dtype=torch.uint8, device=dev)
        _lib.check(L.rtg_loss_mapping(p(f["render"]), p(f["depth"]), p(f["normal"]), p(f["depth_index"]), *frame_args,
                                      p(f["gt_normal"]), p(mask), H, W, channels_last, cw, dw, normal_weight, dem, p(g_color), p(g_depth),
                                      p(g_normal), p(parts), p(ws), stream), "rtg_loss_mapping")
        return parts, g_color, g_depth, g_normal, None
    head = (p(f["render"]), p(f["depth"]), p(f["depth_index"]), *frame_args, p(mask), H, W, channels_last, cw, dw, dem)
    if form == "l1":
        ws = torch.zeros(L.rtg_loss_workspace_bytes(), dtype=torch.uint8, device=dev)
        _lib.check(L.rtg_loss_l1(*head, p(g_color), p(g_depth), p(parts), p(ws), stream), "rtg_loss_l1")
        return parts, g_color, g_depth, None, None
    ws = torch.zeros(L.rtg_loss_l1_exposure_workspace_bytes(), dtype=torch.uint8, device=dev)
    e = torch.tensor(ab, dtype=torch.float32, device=dev)
    g_e = torch.full((2,), float("nan"), device=dev)
    _lib.check(L.rtg_loss_l1_exposure(*head, p(e), p(g_color), p(g_depth), p(g_e), p(parts), p(ws), stream), "rtg_loss_l1_exposure")
    return parts, g_color, g_depth, None, g_e


def statement(form, f):
    """loss_statement on frame f in float64 on the device, with the selections formed from the float32 quantities the
    kernel compares. Returns the statement's outputs and the float64 colour residual (3, n) (zero off the mask)."""
    _, H, W = f["render"].shape
    n = H * W
    m = torch.ones(n, dtype=torch.bool, device=f["render"].device) if f["mask"] is None else f["mask"].reshape(n)
    gt_color = f["gt_color"].permute(2, 0, 1) if tuple(f["gt_color"].shape) == (H, W, 3) else f["gt_color"]
    gt_color = gt_color.reshape(3, n).double()
    depth, gt_depth = f["depth"].reshape(n), f["gt_depth"].reshape(n)
    near = (depth - gt_depth) < torch.tensor(WEIGHTS["depth_error_max"], dtype=torch.float32)      # float32, as the kernel forms it
    ab = (float(np.float32(AB[0])), float(np.float32(AB[1]))) if form == "exposure" else (0.0, 0.0)
    kw = {}
    if form == "mapping":
        kw = dict(normal=f["normal"].reshape(3, n).double(), gt_normal=f["gt_normal"].reshape(n, 3).t().double(),
                  normal_weight=WEIGHTS["normal_weight"])
    render = f["render"].reshape(3, n).double()
    out = loss_statement(render, depth.double(), f["depth_index"].reshape(n), gt_color, gt_depth.double(), m, WEIGHTS["color_weight"],
                         WEIGHTS["depth_weight"], WEIGHTS["depth_error_max"], ab, depth_near=near, **kw)
    r64 = torch.where(m[None], float(np.exp(ab[0])) * render + ab[1] - gt_color, torch.zeros_like(render))
    return out, r64, m


def rel_max(got, want, keep=None):
    """max |got - want| (over `keep` if given) and max |want|."""
    d = (got.double().reshape(want.shape) - want).abs()
    if keep is not None:
        d = d * keep
    return float(d.max()), float(want.abs().max())


@pytest.mark.parametrize("masked", [False, True], ids=["no_mask", "mask60"])
@pytest.mark.parametrize("channels_last", [True, False], ids=["HW3", "3HW"])
@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("form", FORMS)
def test_loss_matches_the_f64_statement_at_every_frame_size(cuda_device, form, H, W, channels_last, masked):
    f = frame(cuda_device, H, W, seed=H * W + 7 * masked + 3 * channels_last, channels_last=channels_last, masked=masked)
    got = loss_call(form, f)
    again = loss_call(form, f)
    for a, b in zip(got, again):                                   # fixed-order sums: the same bits from call to call
        assert (a is None and b is None) or torch.equal(a, b)
    parts, gC, gD, gN, gE = got
    for t in got:
        assert t is None or not bool(torch.isnan(t).any())        # every output element is written
    (want, wC, wD, wN, wE), r64, m = statement(form, f)
    parts = parts.cpu().double().tolist()
    n = H * W
    # counts exact; colour, depth and total to 1e-6 relative, the normal part to 1e-5
    assert parts[3] == want[3], (parts[3], want[3])
    for k in (0, 1, 2):
        assert abs(parts[k] - want[k]) <= 1e-6 * abs(want[k]), (k, parts[k], want[k])
    if form == "mapping":
        assert parts[5] == want[5] and parts[6:] == [0.0, 0.0], parts
        assert abs(parts[4] - want[4]) <= 1e-5 * abs(want[4]), (parts[4], want[4])
    if n > 10_000:        # the frame has every kind of pixel
        assert 0 < want[3] < float(m.sum()) and (form != "mapping" or 0 < want[5] < float(m.sum()))
    # a residual within float32 rounding of zero may take either sign: such pixels are left out of the sign comparisons
    unsure = r64.abs() <= 1e-6
    unsure &= m[None]
    err, top = rel_max(gC, wC, ~unsure)
    assert err <= 1e-6 * top, (err, top)
    err, top = rel_max(gD, wD)
    assert err <= 1e-6 * top, (err, top)
    if form == "mapping":
        err, top = rel_max(gN, wN)
        assert err <= 1e-5 * top, (err, top)
    if form == "exposure":
        # each unsure residual may move dL/da by 2 gcs e^a C and dL/db by 2 gcs
        gcs = WEIGHTS["color_weight"] / (3 * float(m.sum())) if float(m.sum()) > 0 else 0.0
        slack = 2 * gcs * float(np.exp(AB[0])) * max(1.0, float(f["render"].max())) * int(unsure.sum())
        err, top = rel_max(gE, wE)
        assert err <= 1e-5 * top + slack, (gE.cpu(), wE.cpu(), slack)
    print(f"{form} {H}x{W} {'HW3' if channels_last else '3HW'} mask={masked}: parts {parts[:4]} unsure {int(unsure.sum())}")


# ------------------------------------------------------------------------------------------------------ nothing selected
@pytest.mark.parametrize("H,W", [(5, 7), (680, 1200)])
@pytest.mark.parametrize("form", FORMS)
def test_loss_with_nothing_selected(cuda_device, form, H, W):
    """An all-zero render mask, no valid gt depth, no gt normal: the empty means and their gradients are exactly 0 (no NaN
    from 0 / 0), and the other terms are the ones of the full frame, bit for bit."""
    f = frame(cuda_device, H, W, seed=H + W, masked=True)
    parts, gC, gD, gN, gE = loss_call(form, f)
    assert float(parts[3]) > 0 and (form != "mapping" or float(parts[5]) > 0)
    # all-zero mask: every part and every gradient is 0
    z = loss_call(form, dict(f, mask=torch.zeros_like(f["mask"])))
    for t in z:
        assert t is None or torch.equal(t, torch.zeros_like(t)), t
    # gt depth all 0: no depth pixel; the colour (and normal) terms are unchanged
    zp, zC, zD, zN, zE = loss_call(form, dict(f, gt_depth=torch.zeros_like(f["gt_depth"])))
    assert float(zp[2]) == 0 and float(zp[3]) == 0 and torch.equal(zD, torch.zeros_like(zD))
    assert float(zp[1]) == float(parts[1]) and torch.equal(zC, gC)
    assert gE is None or torch.equal(zE, gE)
    want_total = WEIGHTS["color_weight"] * float(parts[1])
    if form == "mapping":
        assert torch.equal(zp[4:6], parts[4:6]) and torch.equal(zN, gN)
        want_total += WEIGHTS["normal_weight"] * float(parts[4])
    assert abs(float(zp[0]) - want_total) <= 1e-6 * want_total
    if form != "mapping":
        return
    # gt normals all 0: no normal pixel; the colour and depth terms are unchanged
    zp, zC, zD, zN, _ = loss_call(form, dict(f, gt_normal=torch.zeros_like(f["gt_normal"])))
    assert float(zp[4]) == 0 and float(zp[5]) == 0 and torch.equal(zN, torch.zeros_like(zN))
    assert torch.equal(zp[1:4], parts[1:4]) and torch.equal(zC, gC) and torch.equal(zD, gD)


@pytest.mark.parametrize("H,W", [(5, 7), (680, 1200)])
def test_mapping_loss_without_normal_weight_has_no_normal_term(cuda_device, H, W):
    """mapping_loss(normal_weight=0) with render and gt normals supplied: parts 4 and 5 are 0, the normal gets no gradient,
    and the colour and depth terms are the L1 loss's."""
    from rtg_slam_b200.loss import l1_color_depth_loss, mapping_loss
    f = frame(cuda_device, H, W, seed=2 * H + W, masked=True)
    normal = f["normal"].clone().requires_grad_(True)
    render = f["render"].clone().requires_grad_(True)
    out = {"render": render, "depth": f["depth"], "normal": normal, "depth_index_map": f["depth_index"]}
    loss, parts = mapping_loss(out, {"color_map": f["gt_color"], "depth_map": f["gt_depth"], "normal_map": f["gt_normal"]},
                               render_mask=f["mask"], color_weight=0.8, depth_weight=1.0, normal_weight=0.0, ssim_weight=0.0,
                               depth_error_max=0.1)
    loss.backward()
    assert float(parts[4]) == 0 and float(parts[5]) == 0 and normal.grad is None
    r2 = f["render"].clone().requires_grad_(True)
    l1, p1 = l1_color_depth_loss({"render": r2, "depth": f["depth"], "depth_index_map": f["depth_index"]}, f["gt_color"], f["gt_depth"],
                                 f["mask"], 0.8, 1.0, 0.1)
    l1.backward()
    assert float(parts[3]) == float(p1[3]) > 0
    for k in (0, 1, 2):
        assert abs(float(parts[k]) - float(p1[k])) <= 1e-6 * abs(float(p1[k]))
    assert torch.equal(render.grad, r2.grad)
