"""GPU tests of coarse-to-fine, robust Gauss-Newton tracking: rtg_frame_downsample against its numpy statement; the
Huber-weighted normal equations of rtg_splat_pose_gn_step_robust against float64 sums over the tangent images, against the
plain rows below the threshold, from run to run, and one device step; PoseRefiner.refine_gn with robust weights on a
partial map, with an image pyramid from outside the single-scale basin, and through a binning overflow at a coarse level."""
import ctypes as C

import numpy as np
import pytest
import torch

from rtg_slam_b200 import scene
from test_camera_grad_gpu import pose_error, se3_exp, view_camera
from test_pose_gn_cpu import gn_step
from test_pose_gn_gpu import gn_inputs
from test_pose_gn_pyramid_cpu import downsample_statement, huber_normal_equations
from test_pose_refine_cpu import camera_arrays
from test_pose_refine_gpu import ARGS, refiner_camera

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------ downsampling
@pytest.mark.parametrize("name", ["small", "ragged", "tum"])
@pytest.mark.parametrize("s", [2, 4])
@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("masks", [False, True])
def test_downsample_matches_the_numpy_statement(cuda_device, name, s, channels_last, masks):
    from rtg_slam_b200.tracking import downsample_frame
    cam = scene.make_camera(name)
    H, W = cam.height, cam.width
    rng = np.random.default_rng(17 + s)
    color = rng.uniform(size=(3, H, W)).astype(np.float32)
    depth = rng.uniform(0.3, 5.0, size=(H, W)).astype(np.float32)
    depth[rng.uniform(size=(H, W)) < 0.03] = 0.0
    mask = rng.uniform(size=(H, W)) < 0.95 if masks else None
    tiles = scene.random_tile_mask(cam, 0.3, seed=5 + s) if masks else None
    c_in = color.transpose(1, 2, 0) if channels_last else color
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device)
    got = downsample_frame(t(c_in), t(depth), s, t(mask), t(tiles))
    want = downsample_statement(c_in, depth, s, mask, tiles, channels_last=channels_last)
    c, d, m, tm = [None if x is None else x.cpu().numpy() for x in got]
    assert c.shape == want[0].shape and d.shape == want[1].shape
    assert np.abs(c - want[0]).max() <= 1e-6
    assert np.array_equal(d > 0, want[1] > 0) and np.abs(d - want[1]).max() <= 1e-6 * np.abs(want[1]).max()
    assert 0 < (d == 0).sum() < d.size
    if masks:
        assert m.dtype == np.uint8 and np.array_equal(m, want[2]) and 0 < m.sum() < m.size
        assert tm.dtype == np.int32 and np.array_equal(tm, want[3])
    else:
        assert m is None and tm is None


# ---------------------------------------------------------------------------------------- robust normal equations
def rows(cam, g, tgt, w2c0, dev, render_mask, configs):
    """One forward and its tangent images J; then, per entry of `configs` (None: rtg_splat_pose_gn_step, (dc, dd):
    rtg_splat_pose_gn_step_robust with Huber thresholds), one step on that same forward into fresh pose / camera arrays.
    Returns J, the forward's outputs, the start pose and per config (per-tile rows, new pose, arrays, report)."""
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
    scratch = torch.empty((int(L.rtg_splat_pose_gn_scratch_bytes(P, H, W)),), dtype=torch.uint8, device=dev)
    J = torch.empty((6, 4, H, W), device=dev)
    _lib.check(L.rtg_splat_pose_tangents(*_native_args(rs, saved, ins, dev), C.c_void_p(outs[3].data_ptr()),
                                         C.c_void_p(scratch.data_ptr()), C.c_void_p(J.data_ptr()), stream), "tangents")
    mask = None if render_mask is None else render_mask.to(torch.uint8).contiguous()
    res = []
    for cfg in configs:
        new_pose = pose.clone()
        arrays = [torch.full_like(t, float("nan")) for t in (view, proj, campos)]
        report = torch.zeros(8, dtype=torch.float64, device=dev)
        scratch.zero_()
        s = _lib.RtgPoseGN()
        s.pose, s.projection = new_pose.data_ptr(), projection.data_ptr()
        s.viewmatrix, s.projmatrix, s.campos = (a.data_ptr() for a in arrays)
        s.render, s.depth, s.hit_depth = outs[0].data_ptr(), outs[1].data_ptr(), outs[3].data_ptr()
        s.gt_color, s.gt_depth = tgt["render"].contiguous().data_ptr(), tgt["depth"].contiguous().data_ptr()
        s.render_mask = None if mask is None else mask.data_ptr()
        s.scratch, s.report = scratch.data_ptr(), report.data_ptr()
        s.color_weight, s.depth_weight, s.depth_error_max, s.damping = 0.8, 1.0, 0.1, 1e-4
        if cfg is None:
            _lib.check(L.rtg_splat_pose_gn_step(*_native_args(rs, saved, ins, dev), C.byref(s), stream), "step")
        else:
            r = _lib.RtgPoseRobust()
            r.kernel, (r.color_delta, r.depth_delta) = _lib.RTG_ROBUST_HUBER, cfg
            _lib.check(L.rtg_splat_pose_gn_step_robust(*_native_args(rs, saved, ins, dev), C.byref(s), C.byref(r), stream),
                       "robust step")
        off = (P * 192 + 255) // 256 * 256     # the per-tile rows sit after the tangent rows
        T = ((H + 15) // 16) * ((W + 15) // 16)
        partial = scratch[off:off + T * 58 * 8].view(torch.float64).view(T, 58).cpu()
        res.append((partial, new_pose.cpu(), [a.cpu() for a in arrays], report.cpu()))
    return J.cpu().double(), [o.cpu() for o in outs], pose.cpu(), res


def kernel_system(part, nc, nd):
    tot = part.sum(0)
    c, d = tot[:29], tot[29:]
    wc, wd = 0.8 / nc, 1.0 / nd
    iu = torch.triu_indices(6, 6)
    Hk = torch.zeros((6, 6), dtype=torch.float64)
    Hk[iu[0], iu[1]] = wc * c[:21] + wd * d[:21]
    Hk = Hk + Hk.triu(1).t()
    return Hk, wc * c[21:27] + wd * d[21:27], c, d


@pytest.mark.parametrize("masks", ["none", "render_mask"])
def test_robust_normal_equations_and_step_match_f64_statements(cuda_device, masks):
    dev = cuda_device
    cam, g, tgt, _, w2c0, kw = gn_inputs(dev, masks)
    # the residuals and selection of the step, in float32 as the kernel forms them
    _, outs0, _, _ = rows(cam, g, tgt, w2c0, dev, kw.get("render_mask"), [])
    H_, W_ = cam.height, cam.width
    m = torch.ones((H_, W_), dtype=torch.bool) if "render_mask" not in kw else kw["render_mask"].cpu().bool()
    rc32 = outs0[0] - tgt["render"].cpu()
    rd32 = outs0[1][0] - tgt["depth"].cpu()[0]
    sel_d = m & (outs0[3][0] != -1) & (tgt["depth"].cpu()[0] > 0) & (rd32 < torch.tensor(0.1, dtype=torch.float32))
    dc = float(np.float32(rc32[:, m].abs().quantile(0.7)))  # as the kernel holds them
    dd = float(np.float32(rd32[sel_d].abs().quantile(0.7)))
    frac_c = float((rc32[:, m].abs() > dc).double().mean())
    frac_d = float((rd32[sel_d].abs() > dd).double().mean())
    print(f"{masks}: deltas {dc:.3e} / {dd:.3e} down-weight {frac_c:.1%} of the colour and {frac_d:.1%} of the depth residuals")
    assert 0.1 <= frac_c <= 0.5 and 0.1 <= frac_d <= 0.5
    big = (2 * float(rc32[:, m].abs().max()) + 1, 2 * float(rd32[sel_d].abs().max()) + 1)
    J, outs, pose0, ((p_r, pose_r, arr_r, rep_r), (p_r2, pose_r2, arr_r2, rep_r2), (p_big, pose_big, _, rep_big),
                     (p_pl, pose_pl, _, rep_pl)) = rows(cam, g, tgt, w2c0, dev, kw.get("render_mask"), [(dc, dd), (dc, dd), big, None])
    for a, b in zip(outs, outs0):
        assert torch.equal(a, b)  # the same forward as the one the residuals came from
    # bit-identical from run to run
    assert torch.equal(p_r, p_r2) and torch.equal(pose_r, pose_r2) and torch.equal(rep_r, rep_r2)
    assert all(torch.equal(a, b) for a, b in zip(arr_r, arr_r2))
    # below the threshold the robust rows are the plain ones
    scale = p_pl.abs().amax(0).clamp_min(1e-300)
    rel = float(((p_big - p_pl).abs() / scale).max())
    print(f"{masks}: robust rows with delta >= max |r| vs plain rows: rel {rel:.2e}, bit-identical {torch.equal(p_big, p_pl)}")
    assert rel <= 1e-6
    assert float((pose_big - pose_pl).abs().max()) <= 1e-9
    # the f64 statement with Huber weights from the same float32 residuals
    Jc, Jd = J[:, :3].reshape(6, 3, -1), J[:, 3].reshape(6, -1)
    Hm, gv, (E, ec, ed), nc, nd = huber_normal_equations(Jc, rc32.double().reshape(3, -1), m.reshape(-1), Jd,
                                                         rd32.double().reshape(-1), sel_d.reshape(-1), 0.8, 1.0, dc, dd)
    Hk, gk, c, d = kernel_system(p_r, nc, nd)
    assert int(c[28]) * 3 == nc and int(d[28]) == nd and nd > 0
    for what, got, want in (("H", Hk, Hm), ("g", gk, gv)):
        err = float((got - want).abs().max() / want.abs().max())
        print(f"{masks}: robust {what} rel err {err:.2e}")
        assert err <= 1e-5, (what, err)
    assert abs(float(rep_r[0]) - E) <= 1e-5 * E and abs(float(rep_r[1]) - ec) <= 1e-5 * ec and abs(float(rep_r[2]) - ed) <= 1e-5 * ed
    assert float(rep_r[3]) == nc and float(rep_r[4]) == nd and float(rep_r[7]) == 0
    assert float(rep_r[0]) < float(rep_pl[0])  # rho(r) < r^2 / 2 beyond the threshold
    # the device step against the f64 statement, from the kernel's own H and g
    want, xi = gn_step(Hk, gk, 1e-4, pose0)
    assert float((pose_r - want).abs().max()) <= 1e-6, (pose_r, want)
    assert abs(float(rep_r[5]) - float(xi[:3].norm())) <= 1e-9 and abs(float(rep_r[6]) - float(xi[3:].norm())) <= 1e-9
    view, proj, campos = camera_arrays(pose_r, torch.from_numpy(cam.projection.astype(np.float64)))
    for got, r in zip(arr_r, (view, proj, campos)):
        assert float((got.double().reshape(r.shape) - r).abs().max()) <= 1e-6 * max(1.0, float(r.abs().max()))


# -------------------------------------------------------------------------------------------------------- refinement
def converge(ref, cam, g, tgt, w2c_true, w2c0, max_iters, label, **kw):
    """The first iteration count (1 .. max_iters) at which refine_gn reaches a tenth of both errors, or None; and the
    errors (fractions of the start) at that count or at max_iters."""
    ang0, tr0 = pose_error(w2c0, w2c_true)
    for it in range(1, max_iters + 1):
        w2c, report = ref.refine_gn(refiner_camera(cam, w2c0), g, tgt["render"], tgt["depth"], iters=it, color_weight=1.0,
                                    depth_weight=1.0, **kw)
        ang, tr = pose_error(w2c, w2c_true.double())
        print(f"{label} {it}: rotation {ang0:.3f} -> {ang:.4f} deg ({ang / ang0:.3f}), translation {100 * tr0:.2f} -> "
              f"{100 * tr:.3f} cm ({tr / tr0:.3f}), status {int(report[7])}")
        assert int(report[7]) == 0
        if ang < 0.1 * ang0 and tr < 0.1 * tr0:
            return it, (ang / ang0, tr / tr0)
    return None, (ang / ang0, tr / tr0)


def test_huber_weights_absorb_the_silhouette_of_a_partial_map(cuda_device):
    """The partial-map case of test_pose_gn_gpu.test_refine_gn_converges, where the squared residuals plateau at 0.056 of
    the rotation and 0.147 of the translation error: with Huber weights (the default thresholds) at a single scale both
    errors fall below a tenth within 10 iterations. Measured on an H100: 0.031 / 0.069 after 7 iterations, settling at
    0.024 / 0.045."""
    from rtg_slam_b200.tracking import PoseRefiner
    cam, g, tgt, w2c_true, w2c0, kw = gn_inputs(cuda_device, "render_mask")
    reached, frac = converge(PoseRefiner(ARGS), cam, g, tgt, w2c_true, w2c0, 10, "huber (render_mask)", robust="huber", **kw)
    assert reached is not None, frac


# The basin scene and start. The pyramid needs a map that renders alike at every level: the rasterizer widens every
# splat by 0.3 px^2 of the level it renders at, at full opacity, so a Gaussian much smaller than a coarse pixel covers
# more of the coarse render than of the block-averaged frame. gn_inputs' room (surfel radii 0.4-5 cm, most of them below
# a pixel at s = 4) differs from its 4x-downsampled target by 0.20 in mean absolute colour (mean colour 0.28); with radii of
# 3-12 cm the difference is 0.035 (mean colour 0.49), measured on an H100. On that room, BASIN times the 1 deg / 2 cm twist
# of gn_inputs (4 deg / 7.9 cm) was chosen by measurement: single-scale Gauss-Newton diverges from it (to 5.5x / 23x the
# start errors without masks, 6.0x / 18x with the tile mask, in 12 iterations) and the pyramid reaches 0.032 / 0.061 and
# 0.028 / 0.053 of them; from 3 deg / 5.9 cm single scale still converges without masks.
BASIN = 4.0
PYRAMID = (4, 2, 1)
PYRAMID_ITERS = (4, 4, 4)


def basin_inputs(dev, masks):
    from rtg_slam_b200.render import Renderer
    cam = scene.make_camera("small")
    g = {k: torch.from_numpy(v).to(dev) for k, v in scene.surfel_room(20_000, seed=7, r_min=0.03, r_max=0.12).items()}
    w2c_true = torch.from_numpy(np.linalg.inv(scene.small_pose()).astype(np.float32)).to(dev)
    with torch.no_grad():
        tgt = Renderer(ARGS).render(view_camera(cam, w2c_true), g)
    w2c0 = se3_exp(BASIN * torch.tensor([0.012, -0.010, 0.012, 0.010, -0.012, 0.008], device=dev)) @ w2c_true
    kw = {"tile_mask": torch.from_numpy(scene.random_tile_mask(cam, 0.5, seed=143)).to(dev)} if masks == "tile_mask" else {}
    return cam, g, tgt, w2c_true, w2c0, kw


@pytest.mark.parametrize("masks", ["none", "tile_mask"])
def test_the_pyramid_widens_the_basin(cuda_device, masks):
    from rtg_slam_b200.tracking import PoseRefiner
    cam, g, tgt, w2c_true, w2c0, kw = basin_inputs(cuda_device, masks)
    ang0, tr0 = pose_error(w2c0, w2c_true)
    assert ang0 >= 3.0 and tr0 >= 0.06, (ang0, tr0)
    ref = PoseRefiner(ARGS)
    total = sum(PYRAMID_ITERS)
    run = lambda **a: ref.refine_gn(refiner_camera(cam, w2c0), g, tgt["render"], tgt["depth"], color_weight=1.0, depth_weight=1.0,
                                    **kw, **a)
    single, _ = run(iters=total)
    pyramid, report = run(iters=PYRAMID_ITERS, scales=PYRAMID)
    a1, t1 = pose_error(single, w2c_true.double())
    a3, t3 = pose_error(pyramid, w2c_true.double())
    print(f"basin ({masks}) from {ang0:.2f} deg / {100 * tr0:.2f} cm, {total} iterations: single scale {a1 / ang0:.3f} / "
          f"{t1 / tr0:.3f}, pyramid {PYRAMID} {a3 / ang0:.4f} / {t3 / tr0:.4f} of the start errors")
    assert int(report[7]) == 0
    assert not (a1 < 0.1 * ang0 and t1 < 0.1 * tr0)
    assert a3 < 0.1 * ang0 and t3 < 0.1 * tr0


def test_a_pyramid_renders_an_overflowed_coarse_iteration_again(cuda_device):
    """gn_inputs' room from 1 deg / 2 cm, where the Huber-weighted pyramid reaches 0.02 / 0.00 of the start errors (the
    plain one does not: see basin_inputs), with a binning buffer too small for the first, coarsest render."""
    from rtg_slam_b200 import rasterizer
    from rtg_slam_b200.tracking import PoseRefiner
    dev = cuda_device
    cam, g, tgt, w2c_true, w2c0, _ = gn_inputs(dev)
    st = rasterizer._state(dev)
    prev_mode, prev_hint = st.mode, st.r_hint
    rasterizer.set_capacity_checks("deferred", dev)
    st.r_hint = 1024
    try:
        w2c, report = PoseRefiner(ARGS).refine_gn(refiner_camera(cam, w2c0), g, tgt["render"], tgt["depth"], iters=(4, 4, 4),
                                                  scales=(4, 2, 1), robust="huber", color_weight=1.0, depth_weight=1.0)
        raised_to = st.r_hint
    finally:
        rasterizer.set_capacity_checks(prev_mode, dev)
        st.r_hint = max(st.r_hint, prev_hint)
    assert raised_to > 1024
    assert int(report[7]) == 0 and float(report[4]) > 0
    ang0, tr0 = pose_error(w2c0, w2c_true)
    ang, tr = pose_error(w2c, w2c_true.double())
    assert ang < 0.1 * ang0 and tr < 0.1 * tr0, (ang0, ang, tr0, tr)
