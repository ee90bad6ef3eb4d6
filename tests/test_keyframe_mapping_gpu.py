"""GPU tests of keyframe poses and exposures refined with the map: rtg_loss_mapping_exposure against rtg_loss_mapping at
(0, 0) bit for bit and against its float64 statement under an exposure; rtg_ssim_loss_exposure likewise; mapping_loss's
exposure gradient as the sum of its two terms'; KeyframeTable's cameras, steps and bookkeeping; pose and exposure
convergence against a frozen map; and a joint run with MapOptimizer, where refined exposures keep the keyframes'
brightness out of the map's colours."""
import ctypes as C

import numpy as np
import pytest
import torch

from rtg_slam_b200 import scene
from test_camera_grad_gpu import pose_error, se3_exp
from test_loss_sizes_gpu import WEIGHTS, frame, rel_max
from test_mapoptim_gpu import LRS
from test_pose_exposure_cpu import loss_statement
from test_pose_exposure_gpu import EXPOSURES
from test_pose_refine_gpu import ARGS, refiner_camera

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------- the mapping loss
def mapping_call(f, ab=None, normal_weight=WEIGHTS["normal_weight"]):
    """rtg_loss_mapping (ab None) or rtg_loss_mapping_exposure on frame f; every output starts as NaN. Returns parts (8),
    dL/dC, dL/ddepth, dL/dnormal, dL/d(a, b) or None, on the host."""
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    dev = f["render"].device
    _, H, W = f["render"].shape
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    nan = lambda t: torch.full_like(t, float("nan"))
    g_color, g_depth, g_normal = nan(f["render"]), nan(f["depth"]), nan(f["render"])
    parts = torch.full((8,), float("nan"), device=dev)
    mask = None if f["mask"] is None else f["mask"].to(torch.uint8).contiguous()
    channels_last = int(tuple(f["gt_color"].shape) == (H, W, 3))
    ws = torch.zeros(L.rtg_loss_workspace_bytes(), dtype=torch.uint8, device=dev)
    head = (p(f["render"]), p(f["depth"]), p(f["normal"]), p(f["depth_index"]), p(f["gt_color"]), p(f["gt_depth"]), p(f["gt_normal"]),
            p(mask), H, W, channels_last, WEIGHTS["color_weight"], WEIGHTS["depth_weight"], normal_weight, WEIGHTS["depth_error_max"])
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    g_e = None
    if ab is None:
        _lib.check(L.rtg_loss_mapping(*head, p(g_color), p(g_depth), p(g_normal), p(parts), p(ws), stream), "rtg_loss_mapping")
    else:
        e = torch.tensor(ab, dtype=torch.float32, device=dev)
        g_e = torch.full((2,), float("nan"), device=dev)
        _lib.check(L.rtg_loss_mapping_exposure(*head, p(e), p(g_color), p(g_depth), p(g_normal), p(g_e), p(parts), p(ws), stream),
                   "rtg_loss_mapping_exposure")
    if normal_weight == 0:
        g_normal = None
    return tuple(None if t is None else t.cpu() for t in (parts, g_color, g_depth, g_normal, g_e))


def same(a, b):
    return all((x is None and y is None) or torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("masked", [False, True], ids=["no_mask", "mask60"])
@pytest.mark.parametrize("normal_weight", [0.0, 0.1])
def test_mapping_loss_at_no_exposure_is_rtg_loss_mapping_bit_for_bit(cuda_device, normal_weight, masked):
    f = frame(cuda_device, 480, 640, seed=31 + int(masked), masked=masked)
    plain = mapping_call(f, None, normal_weight)
    got = mapping_call(f, (0.0, 0.0), normal_weight)
    again = mapping_call(f, (0.0, 0.0), normal_weight)
    assert same(got, again)
    assert same(got[:4], plain[:4]), "exposure (0, 0) must reproduce rtg_loss_mapping"
    assert not torch.isnan(got[4]).any()


@pytest.mark.parametrize("H,W", [(480, 640), (75, 100)], ids=["tum", "ragged"])
@pytest.mark.parametrize("ab", EXPOSURES)
def test_mapping_loss_under_an_exposure_matches_the_f64_statement(cuda_device, ab, H, W):
    f = frame(cuda_device, H, W, seed=H + W)
    parts, gC, gD, gN, gE = mapping_call(f, ab)
    assert same((parts, gC, gD, gN, gE), mapping_call(f, ab))
    n = H * W
    dev = f["render"].device
    m = torch.ones(n, dtype=torch.bool, device=dev)
    gt_color = f["gt_color"].permute(2, 0, 1).reshape(3, n).double()
    depth, gt_depth = f["depth"].reshape(n), f["gt_depth"].reshape(n)
    near = (depth - gt_depth) < torch.tensor(WEIGHTS["depth_error_max"], dtype=torch.float32)
    ab32 = (float(np.float32(ab[0])), float(np.float32(ab[1])))
    render = f["render"].reshape(3, n).double()
    want, wC, wD, wN, wE = loss_statement(render, depth.double(), f["depth_index"].reshape(n), gt_color, gt_depth.double(), m,
                                          WEIGHTS["color_weight"], WEIGHTS["depth_weight"], WEIGHTS["depth_error_max"], ab32,
                                          normal=f["normal"].reshape(3, n).double(), gt_normal=f["gt_normal"].reshape(n, 3).t().double(),
                                          normal_weight=WEIGHTS["normal_weight"], depth_near=near)
    wC, wD, wN, wE = (t.cpu() for t in (wC, wD, wN, wE))
    parts = parts.double().tolist()
    assert parts[3] == want[3] and parts[5] == want[5] and parts[6:] == [0.0, 0.0]
    for k in (0, 1, 2):
        assert abs(parts[k] - want[k]) <= 1e-6 * abs(want[k]), (k, parts[k], want[k])
    assert abs(parts[4] - want[4]) <= 1e-5 * abs(want[4])
    r64 = (float(np.exp(ab32[0])) * render + ab32[1] - gt_color).cpu()
    unsure = r64.abs() <= 1e-6                # a residual within float32 rounding of zero may take either sign
    err, top = rel_max(gC, wC, ~unsure)
    assert err <= 1e-6 * top, (err, top)
    err, top = rel_max(gD, wD)
    assert err <= 1e-6 * top, (err, top)
    err, top = rel_max(gN, wN)
    assert err <= 1e-5 * top, (err, top)
    gcs = WEIGHTS["color_weight"] / (3 * n)
    slack = 2 * gcs * float(np.exp(ab[0])) * max(1.0, float(f["render"].max())) * int(unsure.sum())
    err, top = rel_max(gE, wE)
    print(f"{H}x{W} ab={ab}: dL/d(a, b) {gE.numpy()} vs {wE.numpy()}, unsure {int(unsure.sum())}")
    assert err <= 1e-5 * top + slack, (gE, wE, slack)


# ------------------------------------------------------------------------------------------------------------- SSIM
def ssim_call(a, b, ab, grads=(True, True)):
    """rtg_ssim_loss (ab None) or rtg_ssim_loss_exposure on float32 (C,H,W) CUDA images. Returns loss_out, dL/dimg1 or
    None, dL/d(a, b) or None, on the host."""
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    dev = a.device
    Cn, H, W = a.shape
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    g = torch.full_like(a, float("nan")) if grads[0] else None
    out = torch.full((2,), float("nan"), device=dev)
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    g_e = None
    if ab is None:
        ws = torch.zeros(L.rtg_ssim_workspace_bytes(Cn, H, W), dtype=torch.uint8, device=dev)
        _lib.check(L.rtg_ssim_loss(p(a), p(b), Cn, H, W, p(g), p(out), p(ws), stream), "rtg_ssim_loss")
    else:
        ws = torch.zeros(L.rtg_ssim_exposure_workspace_bytes(Cn, H, W), dtype=torch.uint8, device=dev)
        e = torch.tensor(ab, dtype=torch.float32, device=dev)
        g_e = torch.full((2,), float("nan"), device=dev) if grads[1] else None
        _lib.check(L.rtg_ssim_loss_exposure(p(a), p(b), Cn, H, W, p(e), p(g), p(g_e), p(out), p(ws), stream), "rtg_ssim_loss_exposure")
    return tuple(None if t is None else t.cpu() for t in (out, g, g_e))


def ssim_pair(dev, name):
    import helpers
    a, b = helpers.ssim_inputs(name)
    return torch.from_numpy(a).to(dev), torch.from_numpy(b).to(dev)


@pytest.mark.parametrize("name", ["ragged", "strip", "smooth"])
def test_ssim_at_no_exposure_is_rtg_ssim_loss_bit_for_bit(cuda_device, name):
    a, b = ssim_pair(cuda_device, name)
    plain = ssim_call(a, b, None)
    got = ssim_call(a, b, (0.0, 0.0))
    assert torch.equal(got[0], plain[0]) and torch.equal(got[1], plain[1])
    assert not torch.isnan(got[2]).any()


@pytest.mark.parametrize("name", ["ragged", "strip"])
@pytest.mark.parametrize("ab", EXPOSURES)
def test_ssim_under_an_exposure_matches_the_f64_statement(cuda_device, ab, name):
    from rtg_slam_b200.loss import _ssim_term
    a, b = ssim_pair(cuda_device, name)
    assert a.shape[1] % 16 and a.shape[2] % 16
    out, gx, ge = ssim_call(a, b, ab)
    out2, gx2, ge2 = ssim_call(a, b, ab)
    assert torch.equal(out, out2) and torch.equal(gx, gx2) and torch.equal(ge, ge2)      # fixed-order sums
    # value only, and each gradient on its own, give the same bits
    assert torch.equal(ssim_call(a, b, ab, (False, False))[0], out)
    assert torch.equal(ssim_call(a, b, ab, (False, True))[2], ge) and torch.equal(ssim_call(a, b, ab, (True, False))[1], gx)
    x = a.double().requires_grad_(True)
    e = torch.tensor([float(np.float32(ab[0])), float(np.float32(ab[1]))], dtype=torch.float64, device=a.device, requires_grad=True)
    v = _ssim_term(torch.exp(e[0]) * x + e[1], b.double())
    wx, we = (t.cpu() for t in torch.autograd.grad(v, (x, e)))
    assert abs(float(out[0]) - float(v.detach())) < 1e-5, (float(out[0]), float(v.detach()))
    assert float((gx.double() - wx).abs().max()) <= 1e-4 * float(wx.abs().max())
    err = float((ge.double() - we).abs().max() / we.abs().max())
    print(f"{name} ab={ab}: dL/d(a, b) {ge.numpy()} vs {we.numpy()}, rel err {err:.2e}")
    assert err <= 1e-4, (ge, we)


def test_mapping_loss_exposure_gradient_is_the_sum_of_its_terms(cuda_device):
    """render_mask None, ssim_weight > 0: autograd's dL/d(a, b) is the colour L1's plus ssim_weight times the SSIM term's."""
    from rtg_slam_b200.loss import _ssim_term, mapping_loss
    f = frame(cuda_device, 75, 100, seed=5)
    e = torch.tensor([0.2, 0.05], device=cuda_device, requires_grad=True)
    out = {"render": f["render"].clone().requires_grad_(True), "depth": f["depth"], "depth_index_map": f["depth_index"]}
    loss, parts = mapping_loss(out, {"color_map": f["gt_color"], "depth_map": f["gt_depth"]}, None, ssim_weight=0.2, exposure=e)
    loss.backward()
    n = 75 * 100
    gt = f["gt_color"].permute(2, 0, 1).contiguous()
    e64 = e.detach().double().requires_grad_(True)
    x = f["render"].double()
    l1 = 0.8 * (torch.exp(e64[0]) * x + e64[1] - gt.double()).abs().mean()
    ssim = _ssim_term(torch.exp(e64[0]) * x + e64[1], gt.double())
    (g_l1,) = torch.autograd.grad(l1, (e64,))
    (g_ssim,) = torch.autograd.grad(ssim, (e64,))
    want = g_l1 + 0.2 * g_ssim
    assert float((e.grad.double() - want).abs().max()) <= 1e-4 * float(want.abs().max()), (e.grad, want, g_l1, g_ssim)
    assert abs(float(parts[6]) - float(ssim.detach())) < 1e-5 and n > 0
    # without the exposure: exactly the calls of before (rtg_loss_mapping and rtg_ssim_loss), the same value
    l0, p0 = mapping_loss(out, {"color_map": f["gt_color"], "depth_map": f["gt_depth"]}, None, ssim_weight=0.2)
    l00, _ = mapping_loss(out, {"color_map": f["gt_color"], "depth_map": f["gt_depth"]}, None, ssim_weight=0.2,
                          exposure=torch.zeros(2, device=cuda_device))
    assert float(l0.detach()) == float(l00.detach())


# --------------------------------------------------------------------------------------------------------- the table
def keyframe_scene(dev, P=20_000, cam_name="tum"):
    """The surfel room, three true poses around scene.small_pose() and their renders (the targets before the exposure)."""
    from rtg_slam_b200.render import Renderer
    from test_camera_grad_gpu import view_camera
    cam = scene.make_camera(cam_name)
    g = {k: torch.from_numpy(v).to(dev) for k, v in scene.surfel_room(P, seed=7).items()}
    base = torch.from_numpy(np.linalg.inv(scene.small_pose()).astype(np.float32)).to(dev)
    offsets = ([0.0] * 6, [0.05, 0.0, -0.03, 0.0, 0.02, 0.0], [-0.04, 0.02, 0.03, 0.01, -0.03, 0.0])
    truths = [se3_exp(torch.tensor(o, device=dev)) @ base for o in offsets]
    with torch.no_grad():
        targets = [Renderer(ARGS).render(view_camera(cam, w), g) for w in truths]
    return cam, g, truths, [{k: t[k].detach().clone() for k in ("render", "depth")} for t in targets]


def test_table_camera_renders_as_the_keyframe_camera(cuda_device):
    from rtg_slam_b200.keyframes import KeyframeTable
    from rtg_slam_b200.render import Renderer
    from rtg_slam_b200.tracking import camera_tensors
    cam, g, truths, _ = keyframe_scene(cuda_device, P=5000, cam_name="small")
    table = KeyframeTable(1e-3, 1e-3, 1e-2)
    k = table.add(refiner_camera(cam, truths[1]), exposure=(0.1, 0.02))
    kc = table.camera(k)
    pose = truths[1].double()
    projection = torch.from_numpy(np.ascontiguousarray(cam.projection)).to(cuda_device).float()
    view, proj, campos = camera_tensors(pose, projection)
    own = refiner_camera(cam, truths[1])
    own.full_proj_transform, own.camera_center, own.world_view_transform = proj, campos, view
    with torch.no_grad():
        a = Renderer(ARGS).render(kc, g)
        b = Renderer(ARGS).render(own, g)
    for key in ("render", "depth", "depth_index_map", "T_map"):
        assert torch.equal(a[key], b[key]), key
    assert kc.world_view_transform.requires_grad and kc.full_proj_transform.requires_grad and kc.camera_center.requires_grad
    assert torch.equal(table.pose(k), pose) and table.exposure(k).requires_grad and table.poses().shape == (1, 4, 4)


def table_with_grads(dev, cam, truths):
    """Three keyframes: 0 fixed (pose and exposure), 1 and 2 free, with exposures."""
    from rtg_slam_b200.keyframes import KeyframeTable
    table = KeyframeTable(1e-3, 2e-3, 1e-2)
    start = [truths[0]] + [se3_exp(torch.tensor([0.012, -0.010, 0.012, 0.010, -0.012, 0.008], device=dev)) @ w for w in truths[1:]]
    for k, w in enumerate(start):
        table.add(refiner_camera(cam, w), exposure=(0.0, 0.0), fix_pose=(k == 0), fix_exposure=(k == 0))
    return table


def snapshot(table, k):
    kf = table._kf[k]
    return (kf.pose.clone(), kf.moments.clone(), kf.exposure.detach().clone(), kf.step,
            None if kf.adam is None or not kf.adam.state else {n: v.clone() if torch.is_tensor(v) else v
                                                              for n, v in kf.adam.state[kf.exposure].items()})


def equal_snap(a, b):
    if not (torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]) and a[3] == b[3]):
        return False
    if (a[4] is None) != (b[4] is None):
        return False
    return a[4] is None or all((torch.equal(a[4][n], b[4][n]) if torch.is_tensor(a[4][n]) else a[4][n] == b[4][n]) for n in a[4])


def backward_at(table, k, g, target, ssim_weight=0.2):
    from rtg_slam_b200.loss import mapping_loss
    from rtg_slam_b200.render import Renderer
    out = Renderer(ARGS).render(table.camera(k), g)
    loss, _ = mapping_loss(out, {"color_map": target["render"], "depth_map": target["depth"]}, None, ssim_weight=ssim_weight,
                           exposure=table.exposure(k))
    if loss.requires_grad:                       # a fixed keyframe against a frozen map has nothing to differentiate
        loss.backward()


def test_a_step_moves_only_its_keyframe_and_equals_the_hand_sequence(cuda_device):
    from rtg_slam_b200 import _lib
    from rtg_slam_b200.optim import FusedAdam
    from rtg_slam_b200.tracking import apply_exposure
    dev = cuda_device
    cam, g, truths, targets = keyframe_scene(dev, P=5000, cam_name="small")
    seen = [dict(t, render=apply_exposure(t["render"], ab).contiguous()) for t, ab in zip(targets, [(0.0, 0.0)] + EXPOSURES)]
    table = table_with_grads(dev, cam, truths)
    twin = table_with_grads(dev, cam, truths)        # stepped by hand
    hand_adam = {k: FusedAdam([twin.exposure(k)], lr=1e-2, betas=(0.9, 0.999), eps=1e-8) for k in (1, 2)}
    counts = {0: 0, 1: 0, 2: 0}
    for k in (0, 2, 2, 1):
        before = [snapshot(table, j) for j in range(3)]
        backward_at(table, k, g, seen[k])
        kt = table._kf[k]
        # the camera gradients are summed with atomics: the twin takes these very gradients, not a backward of its own
        grads = [None if t.grad is None else t.grad.clone() for t in (kt.view, kt.proj, kt.campos, kt.exposure)]
        table.step(k)
        counts[k] += 1
        after = [snapshot(table, j) for j in range(3)]
        for j in range(3):
            if j != k or j == 0:
                assert equal_snap(before[j], after[j]), (k, j)
        if k != 0:
            assert not torch.equal(before[k][0], after[k][0]) and not torch.equal(before[k][2], after[k][2])
        for t in (table.camera(k).world_view_transform, table.camera(k).full_proj_transform, table.camera(k).camera_center,
                  table.exposure(k)):
            assert t.grad is None
        # the same sequence by hand on the twin
        kf = twin._kf[k]
        kf.view.grad, kf.proj.grad, kf.campos.grad, kf.exposure.grad = grads
        if k != 0:
            st = _lib.RtgPoseAdam()
            st.pose, st.projection = kf.pose.data_ptr(), kf.projection.data_ptr()
            st.exp_avg, st.exp_avg_sq = kf.moments[0].data_ptr(), kf.moments[1].data_ptr()
            st.viewmatrix, st.projmatrix, st.campos = (t.data_ptr() for t in (kf.view, kf.proj, kf.campos))
            st.dL_dviewmatrix, st.dL_dprojmatrix, st.dL_dcampos = (t.grad.data_ptr() for t in (kf.view, kf.proj, kf.campos))
            st.lr_trans, st.lr_rot, st.beta1, st.beta2, st.eps, st.step = 2e-3, 1e-3, 0.9, 0.999, 1e-8, counts[k]
            _lib.check(_lib.lib().rtg_pose_adam_step(C.byref(st), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "pose step")
            hand_adam[k].step()
        kf.view.grad = kf.proj.grad = kf.campos.grad = kf.exposure.grad = None
        kf.step = counts[k] if k != 0 else 0
        for j in range(3):
            assert torch.equal(table.pose(j), twin.pose(j)) and torch.equal(table.exposure(j), twin.exposure(j))
            assert torch.equal(table.moments(j), twin.moments(j))
    assert [table.step_count(k) for k in range(3)] == [0, 1, 2]
    assert torch.equal(table.pose(0), truths[0].double()) and torch.equal(table.exposure(0), torch.zeros(2, device=dev))
    # set_pose: the pose, its camera tensors, moments and count
    table.set_pose(2, truths[2])
    assert torch.equal(table.pose(2), truths[2].double()) and table.step_count(2) == 0 and not table.moments(2).any()
    assert torch.equal(table.camera(2).world_view_transform, truths[2].double().t().float())
    with pytest.raises(ValueError):
        table.set_pose(2, torch.eye(3))


# ---------------------------------------------------------------------------------------------------- convergence
CONVERGENCE_ITERS = 150


def test_poses_and_exposures_converge_against_a_frozen_map(cuda_device):
    """Keyframe 0 fixed at the truth; 1 and 2 start 1 deg / 2 cm away at exposure (0, 0) and are seen under EXPOSURES.
    Round-robin mapping-loss steps (colour L1 + depth L1 + SSIM) with the map frozen, 150 rounds at lr 1e-3 (rotation),
    2e-3 (translation) and 1e-2 (exposure). Measured on an H100: the largest remaining error of the eight (rotation,
    translation, a, b of keyframes 1 and 2), as a fraction of its start, is 0.018 (keyframe 1's rotation); the bar is
    0.05."""
    from rtg_slam_b200.tracking import apply_exposure
    dev = cuda_device
    cam, g, truths, targets = keyframe_scene(dev)
    seen = [dict(t, render=apply_exposure(t["render"], ab).contiguous()) for t, ab in zip(targets, [(0.0, 0.0)] + EXPOSURES)]
    table = table_with_grads(dev, cam, truths)
    start = [pose_error(table.pose(k), truths[k].double()) for k in (1, 2)]
    for _ in range(CONVERGENCE_ITERS):
        for k in range(3):
            backward_at(table, k, g, seen[k])
            table.step(k)
    worst = 0.0
    for i, k in enumerate((1, 2)):
        ang, tr = pose_error(table.pose(k), truths[k].double())
        ab = table.exposure(k).detach().cpu().double().numpy()
        fa, ft = ang / start[i][0], tr / start[i][1]
        fea, feb = abs(ab[0] - EXPOSURES[i][0]) / abs(EXPOSURES[i][0]), abs(ab[1] - EXPOSURES[i][1]) / abs(EXPOSURES[i][1])
        print(f"keyframe {k}: rotation {fa:.4f}, translation {ft:.4f} of the start; exposure {ab} vs {EXPOSURES[i]}: "
              f"a {fea:.4f}, b {feb:.4f} of the start")
        worst = max(worst, fa, ft, fea, feb)
    assert torch.equal(table.pose(0), truths[0].double())
    assert worst < CONVERGENCE_BAR, worst


CONVERGENCE_BAR = 0.05


def map_optimizer(g, dev):
    from rtg_slam_b200.mapoptim import MapOptimizer
    shs = g["shs"]
    return MapOptimizer(g["xyz"], shs[:, :1].contiguous(), shs[:, 1:].contiguous(), torch.logit(g["opacity"].clamp(1e-4, 1 - 1e-4)),
                        torch.log(g["scales"]), g["rotations"], dict(LRS, opacity=0.0))


def joint_run(dev, cam, g, truths, seen, exposures, iters, table_cams=True):
    """Round-robin map + keyframe steps at fixed poses; `exposures` None (no exposure leaves) or True (keyframes 1 and 2
    refine theirs, keyframe 0's is fixed at (0, 0)). `table_cams` False renders at plain camera tensors instead (today's
    loop). Returns the MapOptimizer."""
    from rtg_slam_b200.keyframes import KeyframeTable
    from rtg_slam_b200.loss import mapping_loss
    from rtg_slam_b200.render import Renderer
    from rtg_slam_b200.tracking import camera_tensors
    mo = map_optimizer(g, dev)
    table = KeyframeTable(1e-3, 1e-3, 1e-2)
    for k, w in enumerate(truths):
        table.add(refiner_camera(cam, w), exposure=None if exposures is None else (0.0, 0.0), fix_pose=True, fix_exposure=(k == 0))
    plain = []
    for w in truths:
        c = refiner_camera(cam, w)
        c.world_view_transform, c.full_proj_transform, c.camera_center = camera_tensors(
            w.double(), torch.from_numpy(np.ascontiguousarray(cam.projection)).to(dev).float())
        plain.append(c)
    for _ in range(iters):
        for k in range(3):
            camera = table.camera(k) if table_cams else plain[k]
            out = Renderer(ARGS).render(camera, mo.gaussian_data())
            loss, _ = mapping_loss(out, {"color_map": seen[k]["render"], "depth_map": seen[k]["depth"]}, None, ssim_weight=0.2,
                                   exposure=table.exposure(k) if table_cams else None)
            loss.backward()
            mo.step()
            if table_cams:
                table.step(k)
    return mo, table


def test_refined_exposures_keep_brightness_out_of_the_map(cuda_device):
    """The map starts at the truth's colours; keyframes 1 and 2 are seen under EXPOSURES at their true (fixed) poses.
    60 rounds of MapOptimizer (base.yaml rates) and keyframe steps. Measured on an H100: the mean |f_dc - truth| over the
    3877 Gaussians the keyframes see is 1.29e-2 without exposure leaves and 9.05e-3 with them, 1.42x less; the exposures
    reach (0.204, 0.050) and (-0.252, -0.030). The bar is 1.3x."""
    from rtg_slam_b200.render import Renderer
    from rtg_slam_b200.tracking import apply_exposure
    from test_camera_grad_gpu import view_camera
    dev = cuda_device
    cam, g, truths, targets = keyframe_scene(dev, P=20_000, cam_name="small")
    seen = [dict(t, render=apply_exposure(t["render"], ab).contiguous()) for t, ab in zip(targets, [(0.0, 0.0)] + EXPOSURES)]
    with torch.no_grad():
        vis = torch.zeros(g["xyz"].shape[0], dtype=torch.bool, device=dev)
        for w in truths:
            vis |= Renderer(ARGS).render(view_camera(cam, w), g)["radii"] > 0
    truth_dc = g["shs"][:, 0]
    drift = {}
    for name, ex in (("without", None), ("with", True)):
        mo, table = joint_run(dev, cam, g, truths, seen, ex, JOINT_ITERS)
        drift[name] = float((mo.features_dc[:, 0] - truth_dc)[vis].abs().mean())
        if ex:
            print(f"exposures {[table.exposure(k).detach().cpu().numpy() for k in range(3)]}")
    factor = drift["without"] / drift["with"]
    print(f"mean |f_dc - truth| over {int(vis.sum())} seen Gaussians: {drift['without']:.4e} without exposures, "
          f"{drift['with']:.4e} with them: {factor:.2f}x")
    assert factor > JOINT_FACTOR, drift


JOINT_ITERS = 60
JOINT_FACTOR = 1.3


def test_fixed_keyframes_without_exposures_leave_the_map_loop_unchanged(cuda_device, monkeypatch):
    """All keyframes fixed, no exposure leaves: the table hands the loop camera tensors bit-equal to the plain ones, which
    require no grad, and its step is a no-op, so the loop makes the same native calls, in the same order, on the same
    inputs as the plain MapOptimizer loop. (The backward sums gradients with atomics, so two runs of either loop are not
    compared bit for bit.)"""
    from rtg_slam_b200 import _lib
    from rtg_slam_b200.keyframes import KeyframeTable
    from rtg_slam_b200.render import Renderer
    from rtg_slam_b200.tracking import apply_exposure, camera_tensors
    dev = cuda_device
    cam, g, truths, targets = keyframe_scene(dev, P=5000, cam_name="small")
    seen = [dict(t, render=apply_exposure(t["render"], ab).contiguous()) for t, ab in zip(targets, [(0.0, 0.0)] + EXPOSURES)]
    table = KeyframeTable(1e-3, 1e-3, 1e-2)
    projection = torch.from_numpy(np.ascontiguousarray(cam.projection)).to(dev).float()
    for k, w in enumerate(truths):
        table.add(refiner_camera(cam, w), fix_pose=True)
        kc = table.camera(k)
        for got, want in zip((kc.world_view_transform, kc.full_proj_transform, kc.camera_center), camera_tensors(w.double(), projection)):
            assert torch.equal(got, want) and not got.requires_grad
        assert table.exposure(k) is None
        with torch.no_grad():
            a = Renderer(ARGS).render(kc, g)
            plain = refiner_camera(cam, w)
            plain.world_view_transform, plain.full_proj_transform, plain.camera_center = camera_tensors(w.double(), projection)
            b = Renderer(ARGS).render(plain, g)
        assert all(torch.equal(a[key], b[key]) for key in ("render", "depth", "depth_index_map", "T_map", "radii"))
    L = _lib.lib()

    class Calls:
        def __init__(self):
            self.names = []

        def __getattr__(self, name):
            self.names.append(name)
            return getattr(L, name)
    seqs = []
    for table_cams in (True, False):
        rec = Calls()
        monkeypatch.setattr(_lib, "lib", lambda: rec)
        _, t = joint_run(dev, cam, g, truths, seen, None, 2, table_cams=table_cams)
        monkeypatch.setattr(_lib, "lib", lambda: L)
        seqs.append(rec.names)
        if table_cams:
            assert all(t.step_count(k) == 0 and not t.moments(k).any() for k in range(3))
            assert all(torch.equal(t.pose(k), truths[k].double()) for k in range(3))
    assert seqs[0] == seqs[1] and "rtg_map_adam_step" in seqs[0] and "rtg_pose_adam_step" not in seqs[0], seqs
