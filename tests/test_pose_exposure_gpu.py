"""GPU tests of exposure estimation in the pose refiners: the 75-term tile rows of rtg_splat_pose_gn_step_exposure against
float64 sums over the tangent images, against the plain rows at (a, b) = (0, 0), from run to run, and one device step;
rtg_loss_l1_exposure against its float64 statement and against rtg_loss_l1; PoseRefiner.refine_gn and refine on frames
whose brightness differs from the map's, with and without the exposure unknowns; the default paths left as they were.

Targets are renders at the true pose seen under a known exposure (tracking.apply_exposure, not clamped)."""
import ctypes as C

import numpy as np
import pytest
import torch

from rtg_slam_b200 import scene
from test_camera_grad_gpu import pose_error, se3_exp, view_camera
from test_pose_exposure_cpu import exposure_gn_step, exposure_normal_equations, loss_statement
from test_pose_gn_gpu import gn_inputs
from test_pose_gn_pyramid_gpu import rows as plain_rows
from test_pose_refine_cpu import camera_arrays
from test_pose_refine_gpu import ARGS, refiner_camera

pytestmark = pytest.mark.gpu

EXPOSURES = [(0.2, 0.05), (-0.25, -0.03)]


def seen(tgt, ab):
    """The target frame under the exposure ab: the colour changes, the depth does not."""
    from rtg_slam_b200.tracking import apply_exposure
    return {"render": apply_exposure(tgt["render"], ab).contiguous(), "depth": tgt["depth"]}


# -------------------------------------------------------------------------------------------- rows and the device step
def rows(cam, g, tgt, w2c0, dev, render_mask, configs):
    """One forward and its tangent images J; then, per entry (ab0, deltas or None, color_weight) of `configs`, one
    rtg_splat_pose_gn_step_exposure on that same forward into fresh pose / camera arrays and a fresh exposure buffer.
    Returns J, the forward's outputs, the start pose and per config (per-tile rows, new pose, arrays, report, new ab)."""
    from rtg_slam_b200 import _lib, rasterizer
    from rtg_slam_b200.tracking import PoseRefiner, _native_args
    L = _lib.lib()
    _, pose, projection, view, proj, campos, rs, gg = PoseRefiner(ARGS)._setup(refiner_camera(cam, w2c0.double()), g,
                                                                              requires_grad=False)
    outs, saved, ins = rasterizer._forward_native(rs, gg["xyz"], gg["shs"], None, gg["opacity"], gg["scales"], gg["rotations"],
                                                  None, None)
    rasterizer._state(dev).read(saved.pending, block=True)
    assert not saved.pending.overflow
    H, W = cam.height, cam.width
    P = int(gg["xyz"].shape[0])
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    scratch = torch.empty((int(L.rtg_splat_pose_gn_exposure_scratch_bytes(P, H, W)),), dtype=torch.uint8, device=dev)
    J = torch.empty((6, 4, H, W), device=dev)
    _lib.check(L.rtg_splat_pose_tangents(*_native_args(rs, saved, ins, dev), C.c_void_p(outs[3].data_ptr()),
                                         C.c_void_p(scratch.data_ptr()), C.c_void_p(J.data_ptr()), stream), "tangents")
    mask = None if render_mask is None else render_mask.to(torch.uint8).contiguous()
    gt_color, gt_depth = tgt["render"].contiguous(), tgt["depth"].contiguous()
    res = []
    for ab0, deltas, color_weight in configs:
        new_pose = pose.clone()
        arrays = [torch.full_like(t, float("nan")) for t in (view, proj, campos)]
        report = torch.zeros(8, dtype=torch.float64, device=dev)
        ab = torch.tensor(ab0, dtype=torch.float64, device=dev)
        scratch.zero_()
        s = _lib.RtgPoseGN()
        s.pose, s.projection = new_pose.data_ptr(), projection.data_ptr()
        s.viewmatrix, s.projmatrix, s.campos = (a.data_ptr() for a in arrays)
        s.render, s.depth, s.hit_depth = outs[0].data_ptr(), outs[1].data_ptr(), outs[3].data_ptr()
        s.gt_color, s.gt_depth = gt_color.data_ptr(), gt_depth.data_ptr()
        s.render_mask = None if mask is None else mask.data_ptr()
        s.scratch, s.report = scratch.data_ptr(), report.data_ptr()
        s.color_weight, s.depth_weight, s.depth_error_max, s.damping = color_weight, 1.0, 0.1, 1e-4
        r = _lib.RtgPoseRobust()
        if deltas is not None:
            r.kernel, (r.color_delta, r.depth_delta) = _lib.RTG_ROBUST_HUBER, deltas
        e = _lib.RtgPoseExposure()
        e.ab = ab.data_ptr()
        _lib.check(L.rtg_splat_pose_gn_step_exposure(*_native_args(rs, saved, ins, dev), C.byref(s), C.byref(r), C.byref(e), stream),
                   "exposure step")
        off = (P * 192 + 255) // 256 * 256     # the per-tile rows sit after the tangent rows
        T = ((H + 15) // 16) * ((W + 15) // 16)
        partial = scratch[off:off + T * 75 * 8].view(torch.float64).view(T, 75).cpu()
        res.append((partial, new_pose.cpu(), [a.cpu() for a in arrays], report.cpu(), ab.cpu()))
    return J.cpu().double(), [o.cpu() for o in outs], pose.cpu(), res


def kernel_system(part, nc, nd, color_weight=0.8):
    """H (8, 8) and g (8) from the summed tile rows, and the colour and depth totals."""
    tot = part.sum(0)
    c, d = tot[:46], tot[46:]
    wc, wd = (color_weight / nc if nc > 0 else 0.0), 1.0 / nd
    Hk = torch.zeros((8, 8), dtype=torch.float64)
    iu = torch.triu_indices(8, 8)
    Hk[iu[0], iu[1]] = wc * c[:36]
    i6 = torch.triu_indices(6, 6)
    Hk[i6[0], i6[1]] += wd * d[:21]
    Hk = Hk + Hk.triu(1).t()
    gk = wc * c[36:44]
    gk[:6] += wd * d[21:27]
    return Hk, gk, c, d


@pytest.mark.parametrize("robust", [False, True])
@pytest.mark.parametrize("masks", ["none", "render_mask"])
def test_exposure_rows_and_step_match_f64_statements(cuda_device, masks, robust):
    dev = cuda_device
    cam, g, tgt, _, w2c0, kw = gn_inputs(dev, masks)
    tgt = seen(tgt, (0.2, 0.05))
    ab0 = (0.1, 0.02)                       # the estimate the step starts from: e^a != 1 and residuals of either sign
    _, outs0, _, _ = rows(cam, g, tgt, w2c0, dev, kw.get("render_mask"), [])
    H_, W_ = cam.height, cam.width
    m = torch.ones((H_, W_), dtype=torch.bool) if "render_mask" not in kw else kw["render_mask"].cpu().bool()
    gtc, gtd = tgt["render"].cpu(), tgt["depth"].cpu()[0]
    rc32 = (outs0[0] * float(np.float32(np.exp(ab0[0]))) + float(np.float32(ab0[1]))) - gtc     # float32, as the kernel forms it
    rd32 = outs0[1][0] - gtd
    sel_d = m & (outs0[3][0] != -1) & (gtd > 0) & (rd32 < torch.tensor(0.1, dtype=torch.float32))
    deltas = None
    if robust:
        deltas = (float(np.float32(rc32[:, m].abs().quantile(0.7))), float(np.float32(rd32[sel_d].abs().quantile(0.7))))
        frac_c = float((rc32[:, m].abs() > deltas[0]).double().mean())
        frac_d = float((rd32[sel_d].abs() > deltas[1]).double().mean())
        print(f"{masks}: deltas {deltas[0]:.3e} / {deltas[1]:.3e} down-weight {frac_c:.1%} colour, {frac_d:.1%} depth residuals")
        assert 0.1 <= frac_c <= 0.5 and 0.1 <= frac_d <= 0.5
    J, outs, pose0, ((part, pose1, arr1, rep1, ab1), (part2, pose2, arr2, rep2, ab2)) = rows(
        cam, g, tgt, w2c0, dev, kw.get("render_mask"), [(ab0, deltas, 0.8)] * 2)
    # bit-identical from run to run
    assert torch.equal(part, part2) and torch.equal(pose1, pose2) and torch.equal(rep1, rep2) and torch.equal(ab1, ab2)
    assert all(torch.equal(a, b) for a, b in zip(arr1, arr2))
    # the f64 statement from the tangent images, the forward's render and the same selection
    Jc, Jd = J[:, :3].reshape(6, 3, -1), J[:, 3].reshape(6, -1)
    Hm, gv, (E, ec, ed), nc, nd = exposure_normal_equations(Jc, outs[0].double().reshape(3, -1), gtc.double().reshape(3, -1),
                                                            m.reshape(-1), Jd, rd32.double().reshape(-1), sel_d.reshape(-1), 0.8,
                                                            1.0, ab0, deltas)
    Hk, gk, c, d = kernel_system(part, nc, nd)
    assert int(c[45]) * 3 == nc and int(d[28]) == nd and nd > 0
    for what, got, want in (("H", Hk, Hm), ("g", gk, gv)):
        err = float((got - want).abs().max() / want.abs().max())
        print(f"{masks} robust={robust}: {what} rel err {err:.2e}")
        assert err <= 1e-5, (what, err)
    # the exposure block on its own scale (the pose block's entries are orders of magnitude larger)
    for what, got, want in (("H[6:, 6:]", Hk[6:, 6:], Hm[6:, 6:]), ("H[:6, 6:]", Hk[:6, 6:], Hm[:6, 6:]), ("g[6:]", gk[6:], gv[6:])):
        err = float((got - want).abs().max() / want.abs().max())
        print(f"{masks} robust={robust}: {what} rel err {err:.2e}")
        assert err <= 1e-5, (what, err)
    assert abs(float(rep1[0]) - E) <= 1e-5 * E and abs(float(rep1[1]) - ec) <= 1e-5 * ec and abs(float(rep1[2]) - ed) <= 1e-5 * ed
    assert float(rep1[3]) == nc and float(rep1[4]) == nd and float(rep1[7]) == 0
    # the device step against the f64 statement, from the kernel's own H and g
    want, ab_want, x = exposure_gn_step(Hk, gk, 1e-4, pose0, ab0)
    assert float((pose1 - want).abs().max()) <= 1e-6, (pose1, want)
    assert float((ab1 - ab_want).abs().max()) <= 1e-9, (ab1, ab_want)
    assert float((ab1 - torch.tensor(ab0, dtype=torch.float64)).abs().max()) > 1e-3      # the exposure moved
    assert abs(float(rep1[5]) - float(x[:3].norm())) <= 1e-9 and abs(float(rep1[6]) - float(x[3:6].norm())) <= 1e-9
    view, proj, campos = camera_arrays(pose1, torch.from_numpy(cam.projection.astype(np.float64)))
    for got, r in zip(arr1, (view, proj, campos)):
        assert float((got.double().reshape(r.shape) - r).abs().max()) <= 1e-6 * max(1.0, float(r.abs().max()))


def test_at_no_exposure_the_pose_block_is_the_plain_one(cuda_device):
    """(a, b) = (0, 0): the leading 6x6 / 6 / E terms are TAN_NORMAL_EQ's (to rounding: the contraction may differ)."""
    dev = cuda_device
    cam, g, tgt, _, w2c0, _ = gn_inputs(dev)
    tgt = seen(tgt, (0.2, 0.05))
    _, _, _, ((part, _, _, rep, _),) = rows(cam, g, tgt, w2c0, dev, None, [((0.0, 0.0), None, 0.8)])
    _, _, _, ((plain, _, _, rep_pl),) = plain_rows(cam, g, tgt, w2c0, dev, None, [None])
    tot, ref = part.sum(0), plain.sum(0)
    lead = [sum(8 - i for i in range(a)) + (c - a) for a in range(6) for c in range(a, 6)]
    pairs = [(tot[lead], ref[:21]), (tot[36:42], ref[21:27]), (tot[44:46], ref[27:29]), (tot[46:], ref[29:])]
    for got, want in pairs:
        rel = float(((got - want).abs() / want.abs().max()).max())
        assert rel <= 1e-6, (rel, got, want)
    assert abs(float(rep[0]) - float(rep_pl[0])) <= 1e-6 * float(rep_pl[0])


def test_without_a_colour_term_the_exposure_is_kept(cuda_device):
    """color_weight = 0: the exposure columns are empty; the pose system is solved alone and the status stays OK."""
    dev = cuda_device
    cam, g, tgt, _, w2c0, _ = gn_inputs(dev)
    tgt = seen(tgt, (0.2, 0.05))
    _, _, pose0, ((part, pose1, arr1, rep, ab),) = rows(cam, g, tgt, w2c0, dev, None, [((0.1, 0.02), None, 0.0)])
    assert torch.equal(ab, torch.tensor([0.1, 0.02], dtype=torch.float64))
    assert float(rep[7]) == 0 and float(rep[1]) == 0 and float(rep[2]) > 0 and float(rep[5]) > 0
    nc, nd = float(rep[3]), float(rep[4])
    Hk, gk, _, _ = kernel_system(part, nc, nd, color_weight=0.0)
    want, ab_want, xi = exposure_gn_step(Hk, gk, 1e-4, pose0, (0.1, 0.02), exposed=False)
    assert float((pose1 - want).abs().max()) <= 1e-6
    view, proj, campos = camera_arrays(pose1, torch.from_numpy(cam.projection.astype(np.float64)))
    for got, r in zip(arr1, (view, proj, campos)):
        assert float((got.double().reshape(r.shape) - r).abs().max()) <= 1e-6 * max(1.0, float(r.abs().max()))


# --------------------------------------------------------------------------------------------------------- the L1 loss
def loss_call(dev, out, tgt, mask, ab, exposure=True):
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    H, W = out["render"].shape[1:]
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    g_color, g_depth = torch.full_like(out["render"], float("nan")), torch.full_like(out["depth"], float("nan"))
    parts = torch.zeros(4, device=dev)
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    head = (p(out["render"]), p(out["depth"]), p(out["depth_index_map"]), p(tgt["render"]), p(tgt["depth"]), p(mask), H, W, 0, 0.8,
            1.0, 0.1)
    if not exposure:
        ws = torch.zeros(L.rtg_loss_workspace_bytes(), dtype=torch.uint8, device=dev)
        _lib.check(L.rtg_loss_l1(*head, p(g_color), p(g_depth), p(parts), p(ws), stream), "rtg_loss_l1")
        return parts.cpu(), g_color.cpu(), g_depth.cpu(), None
    ws = torch.zeros(L.rtg_loss_l1_exposure_workspace_bytes(), dtype=torch.uint8, device=dev)
    e = torch.tensor(ab, dtype=torch.float32, device=dev)
    g_e = torch.full((2,), float("nan"), device=dev)
    _lib.check(L.rtg_loss_l1_exposure(*head, p(e), p(g_color), p(g_depth), p(g_e), p(parts), p(ws), stream), "rtg_loss_l1_exposure")
    return parts.cpu(), g_color.cpu(), g_depth.cpu(), g_e.cpu()


@pytest.mark.parametrize("masks", ["none", "render_mask"])
def test_loss_l1_exposure_matches_the_f64_statement(cuda_device, masks):
    from rtg_slam_b200.render import Renderer
    dev = cuda_device
    cam, g, tgt, _, w2c0, kw = gn_inputs(dev, masks)
    tgt = seen(tgt, (0.2, 0.05))
    with torch.no_grad():
        out = Renderer(ARGS).render(view_camera(cam, w2c0), g)
    out = {k: out[k].contiguous() for k in ("render", "depth", "depth_index_map")}
    mask = kw["render_mask"].to(torch.uint8).contiguous() if "render_mask" in kw else None
    ab = (0.1, 0.02)
    parts, gC, gD, gE = loss_call(dev, out, tgt, mask, ab)
    parts2, gC2, gD2, gE2 = loss_call(dev, out, tgt, mask, ab)
    for a, b in ((parts, parts2), (gC, gC2), (gD, gD2), (gE, gE2)):
        assert torch.equal(a, b)                                   # fixed-order sums: the same bits from call to call
    n = cam.height * cam.width
    m = torch.ones(n, dtype=torch.bool) if mask is None else mask.cpu().bool().reshape(-1)
    ab32 = (float(np.float32(ab[0])), float(np.float32(ab[1])))     # as the kernel holds them
    depth32, gtd32 = out["depth"].cpu().reshape(-1), tgt["depth"].cpu().reshape(-1)
    # the selection from the float32 depth error, as the kernel forms it
    sel32 = (depth32 - gtd32) < torch.tensor(0.1, dtype=torch.float32)
    hit = torch.where(sel32, out["depth_index_map"].cpu().reshape(-1), torch.full((n,), -1, dtype=torch.int32))
    (loss, cl, dl, nd, *_), wC, wD, _, wE = loss_statement(out["render"].cpu().double().reshape(3, -1), depth32.double(), hit,
                                                           tgt["render"].cpu().double().reshape(3, -1), gtd32.double(), m, 0.8, 1.0,
                                                           float("inf"), ab32)
    assert nd > 0 and float(parts[3]) == nd
    for got, want in ((parts[0], loss), (parts[1], cl), (parts[2], dl)):
        assert abs(float(got) - want) <= 1e-6 * abs(want), (got, want)
    # a residual within float32 rounding of zero may take either sign: such pixels are left out of the comparison
    r64 = out["render"].cpu().double().reshape(3, -1) * float(np.exp(ab32[0])) + ab32[1] - tgt["render"].cpu().double().reshape(3, -1)
    sure = r64.abs() > 1e-6
    assert float(sure.double().mean()) > 0.99
    assert float(((gC.double().reshape(3, -1) - wC).abs() * sure).max()) <= 1e-6 * float(wC.abs().max())
    assert float((gD.double().reshape(-1) - wD).abs().max()) <= 1e-6 * float(wD.abs().max())
    err = float((gE.double() - wE).abs().max() / wE.abs().max())
    print(f"{masks}: dL/dexposure {gE.numpy()} vs {wE.numpy()}, rel err {err:.2e}")
    assert err <= 1e-5
    # no exposure: rtg_loss_l1's loss and gradients, bit for bit
    p0, c0, d0, _ = loss_call(dev, out, tgt, mask, (0.0, 0.0))
    p1, c1, d1, _ = loss_call(dev, out, tgt, mask, None, exposure=False)
    p2, c2, d2, _ = loss_call(dev, out, tgt, mask, None, exposure=False)
    assert torch.equal(p1, p2) and torch.equal(c1, c2) and torch.equal(d1, d2)  # rtg_loss_l1's sums are fixed-order too
    assert torch.equal(c0, c1) and torch.equal(d0, d1)
    assert torch.equal(p0, p1)


def test_loss_is_differentiable_with_respect_to_the_exposure(cuda_device):
    """l1_color_depth_loss(exposure=t): autograd returns dL/dC and dL/dt, checked against the torch expression."""
    from rtg_slam_b200.loss import l1_color_depth_loss
    from rtg_slam_b200.render import Renderer
    dev = cuda_device
    cam, g, tgt, _, w2c0, _ = gn_inputs(dev)
    tgt = seen(tgt, (0.2, 0.05))
    with torch.no_grad():
        out = Renderer(ARGS).render(view_camera(cam, w2c0), g)
    render = out["render"].clone().requires_grad_(True)
    t = torch.tensor([0.1, 0.02], device=dev, requires_grad=True)
    loss, parts = l1_color_depth_loss({"render": render, "depth": out["depth"], "depth_index_map": out["depth_index_map"]},
                                      tgt["render"], tgt["depth"], None, 0.8, 0.0, exposure=t)
    (2 * loss).backward()
    r2 = out["render"].double().requires_grad_(True)
    t2 = t.detach().double().requires_grad_(True)
    (2 * 0.8 * (torch.exp(t2[0]) * r2 + t2[1] - tgt["render"].double()).abs().mean()).backward()
    assert float((t.grad.double() - t2.grad).abs().max()) <= 1e-5 * float(t2.grad.abs().max()), (t.grad, t2.grad)
    assert float((render.grad.double() - r2.grad).abs().max()) <= 1e-6 * float(r2.grad.abs().max())
    assert float(loss.detach()) == float(parts[0])


def test_a_two_float_tensor_takes_adams_tail_path(cuda_device):
    """The exposure's Adam step goes through optim.FusedAdam (rtg_adam_step): two elements, below the 128-bit width."""
    from rtg_slam_b200.optim import FusedAdam
    dev = cuda_device
    p = torch.tensor([0.1, -0.02], device=dev, requires_grad=True)
    q = p.detach().clone().requires_grad_(True)
    ours, ref = FusedAdam([p], lr=0.01, betas=(0.9, 0.999), eps=1e-8), torch.optim.Adam([q], lr=0.01, betas=(0.9, 0.999), eps=1e-8)
    gen = torch.Generator(device=dev).manual_seed(3)
    for _ in range(5):
        gr = torch.randn(2, device=dev, generator=gen)
        p.grad, q.grad = gr.clone(), gr.clone()
        ours.step()
        ref.step()
    assert float((p - q).abs().max()) <= 1e-7, (p, q)


# -------------------------------------------------------------------------------------------------------- refinement
def room_inputs(dev):
    """gn_inputs' camera, poses and start on the 3 - 12 cm surfel room, which renders alike at every pyramid level."""
    from rtg_slam_b200.render import Renderer
    cam = scene.make_camera("small")
    g = {k: torch.from_numpy(v).to(dev) for k, v in scene.surfel_room(20_000, seed=7, r_min=0.03, r_max=0.12).items()}
    w2c_true = torch.from_numpy(np.linalg.inv(scene.small_pose()).astype(np.float32)).to(dev)
    with torch.no_grad():
        tgt = Renderer(ARGS).render(view_camera(cam, w2c_true), g)
    w2c0 = se3_exp(torch.tensor([0.012, -0.010, 0.012, 0.010, -0.012, 0.008], device=dev)) @ w2c_true
    return cam, g, tgt, w2c_true, w2c0, {}


def fractions(w2c, w2c0, w2c_true):
    ang0, tr0 = pose_error(w2c0, w2c_true)
    ang, tr = pose_error(w2c, w2c_true.double())
    return ang / ang0, tr / tr0


GN_ITERS = 12


@pytest.mark.parametrize("depth_weight", [1.0, 0.0])
@pytest.mark.parametrize("ab", EXPOSURES)
def test_refine_gn_recovers_pose_and_exposure(cuda_device, ab, depth_weight):
    """The point of the feature. A frame brighter or darker than the map: without the exposure unknowns Gauss-Newton settles
    at a biased pose; with them it reaches a tenth of both errors and (a, b) to 1e-2. Measured on an H100, as fractions of
    the 1 deg / 2 cm start errors after 12 iterations: without the unknowns the translation error stays at 0.078 (depth
    weight 1) and 0.082 (colour only) under (0.2, 0.05), at 0.132 and 0.103 under (-0.25, -0.03), and the rotation error at
    0.029 - 0.052; with them 0.0000 and 0.020 (the float32 rounding of the true pose) in all four, the objective falling
    from 6e-3 - 8e-3 to below 1e-12. The plateau without the unknowns is asserted as measured: above 0.05 of the start
    translation error, where the estimate with them is below 0.01."""
    from rtg_slam_b200.tracking import PoseRefiner
    dev = cuda_device
    cam, g, tgt, w2c_true, w2c0, _ = gn_inputs(dev)
    frame = seen(tgt, ab)
    ref = PoseRefiner(ARGS)
    run = lambda **kw: ref.refine_gn(refiner_camera(cam, w2c0), g, frame["render"], frame["depth"], iters=GN_ITERS, color_weight=1.0,
                                     depth_weight=depth_weight, **kw)
    biased, report0 = run()
    fa0, ft0 = fractions(biased, w2c0, w2c_true)
    w2c, report, est = run(exposure=(0.0, 0.0))
    fa, ft = fractions(w2c, w2c0, w2c_true)
    est = est.cpu()
    print(f"exposure {ab}, depth weight {depth_weight}: without the unknowns {fa0:.3f} / {ft0:.3f} of the start errors, with them {fa:.4f} / {ft:.4f}, "
          f"estimate {est.numpy()}, E {float(report0[0]):.3e} -> {float(report[0]):.3e}")
    assert int(report[7]) == 0 and est.dtype == torch.float64 and est.shape == (2,)
    assert ft0 > 0.05 and float(report0[0]) > 1e-3, (fa0, ft0)   # the brightness change went into the pose
    assert fa < 0.1 and ft < 0.01 and float(report[0]) < 1e-9, (fa, ft)
    assert abs(float(est[0]) - ab[0]) < 1e-2 and abs(float(est[1]) - ab[1]) < 1e-2, est


@pytest.mark.parametrize("ab", EXPOSURES)
def test_pyramid_and_huber_weights_recover_pose_and_exposure(cuda_device, ab):
    from rtg_slam_b200.tracking import PoseRefiner
    dev = cuda_device
    cam, g, tgt, w2c_true, w2c0, _ = room_inputs(dev)
    frame = seen(tgt, ab)
    w2c, report, est = PoseRefiner(ARGS).refine_gn(refiner_camera(cam, w2c0), g, frame["render"], frame["depth"], iters=(4, 4, 6),
                                                   scales=(4, 2, 1), robust="huber", color_weight=1.0, depth_weight=1.0,
                                                   exposure=torch.zeros(2))
    fa, ft = fractions(w2c, w2c0, w2c_true)
    est = est.cpu()
    print(f"exposure {ab}, pyramid (4, 2, 1) + huber: {fa:.4f} / {ft:.4f} of the start errors, estimate {est.numpy()}")
    assert int(report[7]) == 0
    assert fa < 0.1 and ft < 0.1, (fa, ft)
    assert abs(float(est[0]) - ab[0]) < 1e-2 and abs(float(est[1]) - ab[1]) < 1e-2, est


@pytest.mark.parametrize("ab", EXPOSURES)
def test_refine_recovers_pose_and_exposure(cuda_device, ab):
    """The Adam refiner on the same frames: 150 steps at lr 1e-3 as test_pose_refine_gpu, the exposure at lr 1e-2."""
    from rtg_slam_b200.tracking import PoseRefiner
    dev = cuda_device
    cam, g, tgt, w2c_true, w2c0, _ = gn_inputs(dev)
    frame = seen(tgt, ab)
    ref = PoseRefiner(ARGS)
    run = lambda **kw: ref.refine(refiner_camera(cam, w2c0), g, frame["render"], frame["depth"], iters=150, lr_rot=1e-3,
                                  lr_trans=1e-3, color_weight=1.0, depth_weight=1.0, **kw)
    biased, _ = run()
    fa0, ft0 = fractions(biased, w2c0, w2c_true)
    w2c, parts, est = run(exposure=(0.0, 0.0), lr_exposure=1e-2)
    fa, ft = fractions(w2c, w2c0, w2c_true)
    est = est.cpu()
    print(f"refine, exposure {ab}: without the unknowns {fa0:.3f} / {ft0:.3f} of the start errors, with them {fa:.4f} / {ft:.4f}, "
          f"estimate {est.numpy()}, parts {parts.cpu().numpy()}")
    assert est.dtype == torch.float32 and est.shape == (2,) and not est.requires_grad and parts.shape == (4,)
    assert fa < 0.1 and ft < 0.1, (fa, ft)
    assert abs(float(est[0]) - ab[0]) < 1e-2 and abs(float(est[1]) - ab[1]) < 1e-2, est


def test_on_an_unchanged_frame_the_extra_unknowns_cost_nothing(cuda_device):
    from rtg_slam_b200.tracking import PoseRefiner
    dev = cuda_device
    cam, g, tgt, w2c_true, w2c0, _ = gn_inputs(dev)
    ref = PoseRefiner(ARGS)
    run = lambda **kw: ref.refine_gn(refiner_camera(cam, w2c0), g, tgt["render"], tgt["depth"], iters=GN_ITERS, color_weight=1.0,
                                     depth_weight=1.0, **kw)
    plain, _ = run()
    w2c, report, est = run(exposure=(0.0, 0.0))
    fa0, ft0 = fractions(plain, w2c0, w2c_true)
    fa, ft = fractions(w2c, w2c0, w2c_true)
    print(f"no exposure change: {fa0:.4f} / {ft0:.4f} without, {fa:.4f} / {ft:.4f} with the unknowns, estimate {est.cpu().numpy()}")
    assert fa0 < 0.1 and ft0 < 0.1 and fa < 0.1 and ft < 0.1
    assert float(est.abs().max()) < 1e-3


# ------------------------------------------------------------------------------------------- the default paths stay put
class _Calls:
    """Stands in for the loaded library and records which of the step and loss entry points are fetched."""
    WATCHED = ("rtg_splat_pose_gn_step", "rtg_splat_pose_gn_step_robust", "rtg_splat_pose_gn_step_exposure", "rtg_loss_l1",
               "rtg_loss_l1_exposure")

    def __init__(self, L):
        self.L, self.calls = L, []

    def __getattr__(self, name):
        if name in self.WATCHED:
            self.calls.append(name)
        return getattr(self.L, name)


def test_without_exposure_the_entry_points_are_those_of_before(cuda_device, monkeypatch):
    from rtg_slam_b200 import _lib
    from rtg_slam_b200.tracking import PoseRefiner
    dev = cuda_device
    cam, g, tgt, _, w2c0, _ = gn_inputs(dev)
    s = _Calls(_lib.lib())
    monkeypatch.setattr(_lib, "lib", lambda: s)
    ref = PoseRefiner(ARGS)
    camera = refiner_camera(cam, w2c0)

    def calls(fn, **kw):
        s.calls.clear()
        out = fn(camera, g, tgt["render"], tgt["depth"], color_weight=1.0, depth_weight=1.0, **kw)
        return len(out), set(s.calls)
    assert calls(ref.refine_gn, iters=2) == (2, {"rtg_splat_pose_gn_step"})
    assert calls(ref.refine_gn, iters=2, robust="huber") == (2, {"rtg_splat_pose_gn_step_robust"})
    assert calls(ref.refine_gn, iters=(1, 1), scales=(2, 1)) == (2, {"rtg_splat_pose_gn_step"})
    assert calls(ref.refine, iters=2, lr_rot=1e-3, lr_trans=1e-3) == (2, {"rtg_loss_l1"})
    assert calls(ref.refine_gn, iters=2, exposure=(0.0, 0.0)) == (3, {"rtg_splat_pose_gn_step_exposure"})
    assert calls(ref.refine_gn, iters=2, robust="huber", exposure=(0.0, 0.0)) == (3, {"rtg_splat_pose_gn_step_exposure"})
    assert calls(ref.refine, iters=2, lr_rot=1e-3, lr_trans=1e-3, exposure=(0.0, 0.0)) == (3, {"rtg_loss_l1_exposure"})


def test_refine_gn_with_exposure_renders_an_overflowed_iteration_again(cuda_device):
    """The first render meets a binning buffer sized too small for it (a handled status): it is rendered again with the
    capacity raised, and pose and exposure go on from where they were."""
    from rtg_slam_b200 import rasterizer
    from rtg_slam_b200.tracking import PoseRefiner
    dev = cuda_device
    cam, g, tgt, w2c_true, w2c0, _ = gn_inputs(dev)
    frame = seen(tgt, EXPOSURES[0])
    st = rasterizer._state(dev)
    prev_mode, prev_hint = st.mode, st.r_hint
    rasterizer.set_capacity_checks("deferred", dev)
    st.r_hint = 1024
    try:
        w2c, report, est = PoseRefiner(ARGS).refine_gn(refiner_camera(cam, w2c0), g, frame["render"], frame["depth"], iters=GN_ITERS,
                                                       color_weight=1.0, depth_weight=1.0, exposure=(0.0, 0.0))
        raised_to = st.r_hint
    finally:
        rasterizer.set_capacity_checks(prev_mode, dev)
        st.r_hint = max(st.r_hint, prev_hint)
    assert raised_to > 1024
    assert int(report[7]) == 0 and float(report[4]) > 0
    fa, ft = fractions(w2c, w2c0, w2c_true)
    assert fa < 0.1 and ft < 0.1, (fa, ft)
    assert abs(float(est[0]) - EXPOSURES[0][0]) < 1e-2 and abs(float(est[1]) - EXPOSURES[0][1]) < 1e-2, est
