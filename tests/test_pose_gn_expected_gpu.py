"""GPU tests of the expected-depth Gauss-Newton residual (rtg_splat_pose_tangents_expected, rtg_splat_pose_gn_step_expected,
tracking.pose_jacobian(depth="expected"), PoseRefiner.refine_gn(depth="expected")): the replayed (D, m1) map against
rasterize_features(F = (z_view, 1)); the tangents against central differences of the float64 oracle and, by the adjoint
identity, against the reverse-mode twist gradient of the feature map; the normal equations and the step against float64
statements (plain, Huber, exposure); convergence; depth="hit" left as it was."""
import ctypes as C

import numpy as np
import pytest
import torch

import helpers
from oracle.antialias_oracle import AntialiasedOracleRender
from oracle.features_oracle import features as feature_statement
from oracle.splat_oracle import OracleRender
from rtg_slam_b200 import rasterizer, scene
from test_camera_grad_gpu import CAM, KW, inputs_for, pose_error, scene_case
from test_pose_exposure_cpu import exposure_gn_step, exposure_normal_equations
from test_pose_gn_cpu import gn_step, normal_equations
from test_pose_gn_gpu import expm, gn_inputs
from test_pose_gn_pyramid_cpu import huber_normal_equations
from test_pose_refine_cpu import camera_arrays, tangent_grad
from test_pose_refine_gpu import ARGS, refiner_camera

pytestmark = pytest.mark.gpu


def z_view(means, vm):
    return means @ vm[:3, 2] + vm[3, 2]


def expected_jacobian(rs, t, tm=None, aa=False):
    from rtg_slam_b200.tracking import pose_jacobian
    with rasterizer.antialiased(aa):
        return pose_jacobian(rs, tile_mask=tm, depth="expected", **t)


def feature_map(rs, t, tm=None, aa=False):
    from rtg_slam_b200.features import rasterize_features
    F = torch.stack([z_view(t["means3D"], rs.viewmatrix), torch.ones_like(t["means3D"][:, 0])], 1).contiguous()
    with torch.no_grad(), rasterizer.antialiased(aa):
        _, fmap = rasterize_features(rs, features=F, tile_mask=tm, **t)
    return fmap


def room_tensors(g, dev):
    return {"means3D": g["xyz"], "opacities": g["opacity"], "shs": g["shs"], "scales": g["scales"], "rotations": g["rotations"]}


# ------------------------------------------------------------------------------------------ 1. the map is the feature map
@pytest.mark.parametrize("case", ["plain", "antialiased", "tile_mask", "render_mask"])
def test_the_replayed_map_is_the_feature_map(cuda_device, case):
    """(D, m1) of the tangent replay against m0 / m1, m1 of rasterize_features(F = (z_view, 1)) on the same forward. m1 is the
    same float sum in the same order: it must be bit-equal. m0 differs only by the rounding of z (the hit record's float
    z against torch's z_view of the same centre, an ulp each): D within 4 float32 ulps of its value (5e-7 relative).
    render_mask: the partial map of gn_inputs (the mask only selects the step's pixels, not the map)."""
    dev = cuda_device
    masks = {"tile_mask": "tile_mask", "render_mask": "render_mask"}.get(case, "none")
    cam, g, _, _, _, kw = gn_inputs(dev, masks)
    rs = helpers.make_settings(cam, dev)
    t = room_tensors(g, dev)
    tm, aa = kw.get("tile_mask"), case == "antialiased"
    outs, J, ex = expected_jacobian(rs, t, tm, aa)
    fmap = feature_map(rs, t, tm, aa)
    m1f = fmap[1]
    Df = torch.where(m1f > 0, fmap[0] / m1f, torch.zeros_like(m1f))
    assert torch.equal(ex[1], m1f), float((ex[1] - m1f).abs().max())
    err = float(((ex[0] - Df).abs() / Df.abs().clamp_min(1e-30)).max())
    cover = float((m1f > 0).float().mean())
    print(f"{case}: coverage > 0 on {cover:.1%} of the pixels, D rel err {err:.2e}")
    assert err <= 5e-7 and cover > 0.3
    assert torch.all(J[:, 3][:, m1f == 0] == 0)
    if tm is not None:  # masked-out tiles: nothing
        off = ~tm.bool().repeat_interleave(16, 0).repeat_interleave(16, 1)[:cam.height, :cam.width]
        assert torch.all(ex[:, off] == 0) and torch.all(J[:, :, off] == 0)


# ------------------------------------------------------------------------------- 2. tangents against the float64 oracle
def oracle_expected(cam, inputs, w2c, mask, over, aa):
    """The f64 oracle's expected depth and coverage at the pose w2c: F = (z_view, 1), z formed in double."""
    projection = cam.projection.astype(np.float64)
    view = w2c.T
    import types
    c = types.SimpleNamespace(height=cam.height, width=cam.width, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, cx=cam.cx, cy=cam.cy,
                              viewmatrix=view, projmatrix=view @ projection, campos=-(w2c[:3, :3].T @ w2c[:3, 3]))
    g = {k: (None if inputs.get(k) is None else inputs[k].astype(np.float64)) for k in ("xyz", "opacity", "shs", "scales", "rotations")}
    cls = AntialiasedOracleRender if aa else OracleRender
    o = cls(c, g, tile_mask=mask, precision="f64", **over)
    z = g["xyz"] @ w2c[2, :3] + w2c[2, 3]
    fm = feature_statement(o, F=np.stack([z, np.ones_like(z)], 1))["map"]
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(fm[1] > 0, fm[0] / fm[1], 0.0), fm[1]


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("name", ["small", "masked"])
def test_expected_depth_tangents_match_f64_oracle(cuda_device, name, aa):
    """Central differences of the oracle's expected depth along each twist direction, steps h and h/4; pixels where the
    two disagree (a pair's decision flipped inside the step) or whose coverage is below 1e-3 (where D is ill-conditioned)
    are skipped. The rest agree within 1e-3 of each direction's largest entry."""
    dev = cuda_device
    cam, g, mask = scene_case(name)
    inputs, over = inputs_for(g, "sh")
    t = {KW[k]: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in inputs.items()}
    tm = None if mask is None else torch.from_numpy(np.ascontiguousarray(mask, dtype=np.int32)).to(dev)
    _, J, ex = expected_jacobian(helpers.make_settings(cam, dev, **over), t, tm, aa)
    J, ex = J.cpu().numpy().astype(np.float64), ex.cpu().numpy()
    w2c = np.linalg.inv(cam.c2w)
    _, m1 = oracle_expected(cam, inputs, w2c, mask, over, aa)
    h = 1e-4
    skipped = total = 0
    for k in range(6):
        fd = []
        for step in (h, h / 4):
            e = np.zeros(6)
            e[k] = step
            dp, _ = oracle_expected(cam, inputs, expm(e) @ w2c, mask, over, aa)
            dm, _ = oracle_expected(cam, inputs, expm(-e) @ w2c, mask, over, aa)
            fd.append((dp - dm) / (2 * step))
        a, b, got = fd[0], fd[1], J[k, 3]
        keep = (m1 > 1e-3) & (ex[1] > 1e-3)
        scale = np.abs(b[keep]).max()
        keep &= np.abs(a - b) <= 2e-4 * scale
        skipped += int(((m1 > 1e-3) & ~keep).sum())
        total += int((m1 > 1e-3).sum())
        err = np.abs(got - b)[keep].max() / scale
        print(f"{name} aa={aa} direction {k}: max err {err:.2e} of the block max {scale:.3e}, kept {keep.sum()} pixels")
        assert err <= 1e-3, (name, aa, k, err)
    frac = skipped / total
    print(f"{name} aa={aa}: skipped fraction {frac:.3%}")
    assert frac < 0.03, frac


# ------------------------------------------------------------------ 3. adjoint identity against the merged reverse path
@pytest.fixture(scope="module")
def room_1m():
    return scene.surfel_room(1_000_000, seed=2024)


@pytest.mark.parametrize("cam_name", ["replica", "hd"])
def test_adjoint_identity_against_the_feature_map_gradient(cuda_device, room_1m, cam_name):
    """u^T (J_D v) for v the six unit twists against the twist gradient of sum u D, D = m0 / m1 of rasterize_features(F =
    (z_view, 1), weight_grad=True) with camera gradients (z_view itself differentiated through the viewmatrix), mapped to
    the twist as test_pose_gn_gpu.reverse_twist_grad maps it."""
    from rtg_slam_b200.features import rasterize_features
    dev = cuda_device
    cam = scene.make_camera(cam_name, c2w=scene.small_pose())
    t = {KW[k]: torch.from_numpy(np.ascontiguousarray(room_1m[k])).to(dev) for k in ("xyz", "opacity", "shs", "scales", "rotations")}
    gen = torch.Generator(device=dev).manual_seed(21)
    u = torch.randn((cam.height, cam.width), device=dev, generator=gen)
    _, J, ex = expected_jacobian(helpers.make_settings(cam, dev), t)
    fwd = torch.einsum("khw,hw->k", J[:, 3].double(), u.double()).cpu().numpy()

    def reverse():
        rs = helpers.make_settings(cam, dev)
        for k in CAM:
            getattr(rs, k).requires_grad_(True)
        F = torch.stack([z_view(t["means3D"], rs.viewmatrix), torch.ones_like(t["means3D"][:, 0])], 1)
        _, fmap = rasterize_features(rs, features=F, weight_grad=True, **t)
        cov = fmap[1] > 0
        D = torch.where(cov, fmap[0] / torch.where(cov, fmap[1], torch.ones_like(fmap[1])), torch.zeros_like(fmap[1]))
        (D * u).sum().backward()
        d = [getattr(rs, k).grad.double().cpu() for k in CAM]
        w2c = torch.from_numpy(np.linalg.inv(cam.c2w))
        return tangent_grad(d[0].view(4, 4), d[1].view(4, 4), d[2], w2c, torch.from_numpy(cam.projection.astype(np.float64))).numpy()

    rev, rev2 = reverse(), reverse()
    scale = np.abs(rev).max()
    spread = np.abs(rev - rev2).max() / scale
    err = np.abs(fwd - rev).max() / scale
    print(f"{cam_name}: forward-mode vs reverse-mode expected-depth twist gradient {err:.2e} (reverse run-to-run "
          f"{spread:.2e}), coverage > 0 on {float((ex[1] > 0).float().mean()):.1%}\n  fwd {fwd}\n  rev {rev}")
    assert err <= max(1e-4, 10 * spread), (err, spread)


# ------------------------------------------------------------------------------------ 4. normal equations and the step
def expected_rows(cam, g, tgt, w2c0, dev, render_mask, configs, min_coverage=0.5):
    """One forward, its expected tangent images and map; then per (deltas or None, ab0 or None) of `configs` one
    rtg_splat_pose_gn_step_expected on that same forward into fresh pose / camera arrays (and exposure). Returns J, the
    map, the start pose and per config (tile rows, new pose, arrays, report, new ab or None)."""
    from rtg_slam_b200 import _lib
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
    ex = torch.empty((2, H, W), device=dev)
    _lib.check(L.rtg_splat_pose_tangents_expected(*_native_args(rs, saved, ins, dev), C.c_void_p(scratch.data_ptr()),
                                                  C.c_void_p(J.data_ptr()), C.c_void_p(ex.data_ptr()), stream), "tangents")
    mask = None if render_mask is None else render_mask.to(torch.uint8).contiguous()
    gt_color, gt_depth = tgt["render"].contiguous(), tgt["depth"].contiguous()
    res = []
    for deltas, ab0 in configs:
        new_pose = pose.clone()
        arrays = [torch.full_like(t, float("nan")) for t in (view, proj, campos)]
        report = torch.zeros(8, dtype=torch.float64, device=dev)
        scratch.zero_()
        s = _lib.RtgPoseGN()
        s.pose, s.projection = new_pose.data_ptr(), projection.data_ptr()
        s.viewmatrix, s.projmatrix, s.campos = (a.data_ptr() for a in arrays)
        s.render, s.depth, s.hit_depth = outs[0].data_ptr(), outs[1].data_ptr(), outs[3].data_ptr()
        s.gt_color, s.gt_depth = gt_color.data_ptr(), gt_depth.data_ptr()
        s.render_mask = None if mask is None else mask.data_ptr()
        s.scratch, s.report = scratch.data_ptr(), report.data_ptr()
        s.color_weight, s.depth_weight, s.depth_error_max, s.damping = 0.8, 1.0, 0.1, 1e-4
        r = _lib.RtgPoseRobust()
        if deltas is not None:
            r.kernel, (r.color_delta, r.depth_delta) = _lib.RTG_ROBUST_HUBER, deltas
        ab, e = None, None
        if ab0 is not None:
            ab = torch.tensor(ab0, dtype=torch.float64, device=dev)
            e = _lib.RtgPoseExposure()
            e.ab = ab.data_ptr()
        _lib.check(L.rtg_splat_pose_gn_step_expected(*_native_args(rs, saved, ins, dev), C.byref(s), C.byref(r),
                                                     None if e is None else C.byref(e), min_coverage, stream), "step")
        nt = 75 if ab0 is not None else 58
        off = (P * 192 + 255) // 256 * 256
        T = ((H + 15) // 16) * ((W + 15) // 16)
        partial = scratch[off:off + T * nt * 8].view(torch.float64).view(T, nt).cpu()
        res.append((partial, new_pose.cpu(), [a.cpu() for a in arrays], report.cpu(), None if ab is None else ab.cpu()))
    return J.cpu().double(), ex.cpu(), [o.cpu() for o in outs], pose.cpu(), res


@pytest.mark.parametrize("kind", ["plain", "huber", "exposure"])
@pytest.mark.parametrize("masks", ["none", "render_mask"])
def test_normal_equations_and_step_match_f64_statements(cuda_device, masks, kind):
    dev = cuda_device
    cam, g, tgt, _, w2c0, kw = gn_inputs(dev, masks)
    J, ex, outs, pose0, _ = expected_rows(cam, g, tgt, w2c0, dev, kw.get("render_mask"), [])
    H_, W_ = cam.height, cam.width
    m = torch.ones((H_, W_), dtype=torch.bool) if "render_mask" not in kw else kw["render_mask"].cpu().bool()
    gtc, gtd = tgt["render"].cpu(), tgt["depth"].cpu()[0]
    D, m1 = ex[0], ex[1]
    rd32 = D - gtd                                          # float32, as the kernel forms it
    sel_d = m & (m1 >= 0.5) & (gtd > 0) & (rd32 < torch.tensor(0.1, dtype=torch.float32))
    rc32 = outs[0] - gtc
    deltas = ab0 = None
    if kind == "huber":
        deltas = (float(np.float32(rc32[:, m].abs().quantile(0.7))), float(np.float32(rd32[sel_d].abs().quantile(0.7))))
    if kind == "exposure":
        ab0 = (0.1, 0.02)
    J2, ex2, outs2, _, ((part, pose1, arr1, rep1, ab1), (part2, pose2, arr2, rep2, ab2)) = expected_rows(
        cam, g, tgt, w2c0, dev, kw.get("render_mask"), [(deltas, ab0)] * 2)
    assert torch.equal(J2, J) and torch.equal(ex2, ex) and all(torch.equal(a, b) for a, b in zip(outs, outs2))
    # bit-identical from run to run
    assert torch.equal(part, part2) and torch.equal(pose1, pose2) and torch.equal(rep1, rep2)
    assert all(torch.equal(a, b) for a, b in zip(arr1, arr2))
    if ab1 is not None:
        assert torch.equal(ab1, ab2)
    Jc, Jd = J[:, :3].reshape(6, 3, -1), J[:, 3].reshape(6, -1)
    rd, sd, mc = rd32.double().reshape(-1), sel_d.reshape(-1), m.reshape(-1)
    n6 = 8 if kind == "exposure" else 6
    tot = part.sum(0)
    if kind == "exposure":
        Hm, gv, (E, ec, ed), nc, nd = exposure_normal_equations(Jc, outs[0].double().reshape(3, -1), gtc.double().reshape(3, -1),
                                                                mc, Jd, rd, sd, 0.8, 1.0, ab0, None)
        c, d = tot[:46], tot[46:]
        assert int(c[45]) * 3 == nc
        wc, wd = 0.8 / nc, 1.0 / nd
        Hk = torch.zeros((8, 8), dtype=torch.float64)
        iu = torch.triu_indices(8, 8)
        Hk[iu[0], iu[1]] = wc * c[:36]
        i6 = torch.triu_indices(6, 6)
        Hk[i6[0], i6[1]] += wd * d[:21]
        gk = wc * c[36:44]
        gk[:6] += wd * d[21:27]
    else:
        rc = rc32.double().reshape(3, -1)
        if kind == "huber":
            Hm, gv, (E, ec, ed), nc, nd = huber_normal_equations(Jc, rc, mc, Jd, rd, sd, 0.8, 1.0, *deltas)
        else:
            Hm, gv, (E, ec, ed), nc, nd = normal_equations(Jc, rc, mc, Jd, rd, sd, 0.8, 1.0)
        c, d = tot[:29], tot[29:]
        assert int(c[28]) * 3 == nc
        wc, wd = 0.8 / nc, 1.0 / nd
        Hk = torch.zeros((6, 6), dtype=torch.float64)
        iu = torch.triu_indices(6, 6)
        Hk[iu[0], iu[1]] = wc * c[:21] + wd * d[:21]
        gk = wc * c[21:27] + wd * d[21:27]
    Hk = Hk + Hk.triu(1).t()
    assert int(d[28]) == nd and nd > 0
    print(f"{masks}/{kind}: N_d = {nd} ({nd / (H_ * W_):.1%} of the pixels; hit-depth set "
          f"{int((m & (outs[3][0] != -1)).sum())})")
    for what, got, want in (("H", Hk, Hm), ("g", gk, gv)):
        err = float((got - want).abs().max() / want.abs().max())
        print(f"{masks}/{kind}: {what} ({n6}x{n6}) rel err {err:.2e}")
        assert err <= 1e-5, (what, err)
    assert abs(float(rep1[0]) - E) <= 1e-5 * E and abs(float(rep1[1]) - ec) <= 1e-5 * ec and abs(float(rep1[2]) - ed) <= 1e-5 * ed
    assert float(rep1[3]) == nc and float(rep1[4]) == nd and float(rep1[7]) == 0
    if kind == "exposure":
        want, ab_want, x = exposure_gn_step(Hk, gk, 1e-4, pose0, ab0)
        assert float((ab1 - ab_want).abs().max()) <= 1e-9, (ab1, ab_want)
        xi = x[:6]
    else:
        want, xi = gn_step(Hk, gk, 1e-4, pose0)
    assert float((pose1 - want).abs().max()) <= 1e-6, (pose1, want)
    assert abs(float(rep1[5]) - float(xi[:3].norm())) <= 1e-9 and abs(float(rep1[6]) - float(xi[3:6].norm())) <= 1e-9
    view, proj, campos = camera_arrays(pose1, torch.from_numpy(cam.projection.astype(np.float64)))
    for got, r in zip(arr1, (view, proj, campos)):
        assert float((got.double().reshape(r.shape) - r).abs().max()) <= 1e-6 * max(1.0, float(r.abs().max()))


# -------------------------------------------------------------------------------------------------------- 5. convergence
def errors_after(ref, cam, g, tgt, w2c_true, w2c0, **kw):
    w2c, report = ref.refine_gn(refiner_camera(cam, w2c0), g, tgt["render"], tgt["depth"], **kw)
    ang0, tr0 = pose_error(w2c0, w2c_true)
    ang, tr = pose_error(w2c, w2c_true.double())
    return ang / ang0, tr / tr0, report


# Not met. Measured on an H100 (10 iterations, fractions of the start errors, hit depth beside): colour + depth 0.150 /
# 0.259 (hit 0.020 / 0.000), depth only 0.861 / 1.625 (hit 27.9 / 121). The target depth is the hit depth of a render at
# the true pose; the expected depth of that render differs from it at silhouettes and inside sub-pixel surfel stacks, so
# the expected-depth residual is not zero at the true pose. The bar stays; strict, so that meeting it shows.
@pytest.mark.xfail(strict=True, reason="measured 0.150 / 0.259 (colour + depth) and 0.861 / 1.625 (depth only)")
@pytest.mark.parametrize("color_weight", [1.0, 0.0])
def test_refine_gn_expected_converges(cuda_device, color_weight):
    """gn_inputs' 1 deg / 2 cm start: depth="expected" reaches a tenth of both errors within 10 iterations, colour + depth
    and depth only. The hit-depth result is printed beside it."""
    from rtg_slam_b200.tracking import PoseRefiner
    cam, g, tgt, w2c_true, w2c0, _ = gn_inputs(cuda_device)
    ref = PoseRefiner(ARGS)
    res = {}
    for depth in ("hit", "expected"):
        fa, ft, report = errors_after(ref, cam, g, tgt, w2c_true, w2c0, iters=10, color_weight=color_weight, depth_weight=1.0,
                                      depth=depth)
        res[depth] = (fa, ft, report)
        print(f"single scale, color_weight {color_weight}, depth={depth}: rotation {fa:.4f}, translation {ft:.4f} of the "
              f"start, report {report.cpu().numpy()}")
    fa, ft, report = res["expected"]
    assert int(report[7]) == 0 and float(report[4]) > 0
    assert fa < 0.1 and ft < 0.1, (fa, ft)


# Not met. Measured on an H100: 5.93 / 31.2 of the start errors (hit depth: 76.6 / 104, singular last step).
@pytest.mark.xfail(strict=True, reason="measured 5.93 / 31.2 of the start errors")
def test_refine_gn_expected_pyramid_antialiased_depth_only(cuda_device):
    """scales (4, 2, 1) with coarse_antialias, depth only: depth="expected" reaches a tenth of both errors. The hit-depth
    result is printed beside it."""
    from rtg_slam_b200.tracking import PoseRefiner
    cam, g, tgt, w2c_true, w2c0, _ = gn_inputs(cuda_device)
    ref = PoseRefiner(ARGS)
    res = {}
    for depth in ("hit", "expected"):
        fa, ft, report = errors_after(ref, cam, g, tgt, w2c_true, w2c0, iters=(4, 4, 4), scales=(4, 2, 1), coarse_antialias=True,
                                      color_weight=0.0, depth_weight=1.0, depth=depth)
        res[depth] = (fa, ft, report)
        print(f"pyramid (4, 2, 1) antialiased, depth only, depth={depth}: rotation {fa:.4f}, translation {ft:.4f} of the start, "
              f"report {report.cpu().numpy()}")
    fa, ft, report = res["expected"]
    assert int(report[7]) == 0
    assert fa < 0.1 and ft < 0.1, (fa, ft)


# ------------------------------------------------------------------------------------------------ 6. the default path
def test_depth_hit_is_the_default_bit_for_bit(cuda_device):
    from rtg_slam_b200.tracking import PoseRefiner
    cam, g, tgt, _, w2c0, kw = gn_inputs(cuda_device, "tile_mask")
    ref = PoseRefiner(ARGS)
    for extra in ({}, {"robust": "huber"}, {"exposure": (0.0, 0.0)}, {"scales": (2, 1), "iters": (2, 2)}):
        a = dict(iters=3, color_weight=1.0, depth_weight=1.0, **kw)
        a.update(extra)
        r0 = ref.refine_gn(refiner_camera(cam, w2c0), g, tgt["render"], tgt["depth"], **a)
        r1 = ref.refine_gn(refiner_camera(cam, w2c0), g, tgt["render"], tgt["depth"], depth="hit", **a)
        assert len(r0) == len(r1) and all(torch.equal(x, y) for x, y in zip(r0, r1)), extra
    from rtg_slam_b200.tracking import pose_jacobian
    rs = helpers.make_settings(cam, cuda_device)
    t = room_tensors(g, cuda_device)
    o0, J0 = pose_jacobian(rs, **t)
    o1, J1 = pose_jacobian(rs, depth="hit", **t)
    assert torch.equal(J0, J1) and all(torch.equal(x, y) for x, y in zip(o0, o1))


def test_expected_renders_an_overflowed_iteration_again(cuda_device):
    from rtg_slam_b200.tracking import PoseRefiner
    dev = cuda_device
    cam, g, tgt, w2c_true, w2c0, _ = gn_inputs(dev)
    st = rasterizer._state(dev)
    prev_mode, prev_hint = st.mode, st.r_hint
    rasterizer.set_capacity_checks("deferred", dev)
    st.r_hint = 1024
    try:
        w2c, report = PoseRefiner(ARGS).refine_gn(refiner_camera(cam, w2c0), g, tgt["render"], tgt["depth"], iters=10,
                                                  color_weight=1.0, depth_weight=1.0, depth="expected")
        raised_to = st.r_hint
    finally:
        rasterizer.set_capacity_checks(prev_mode, dev)
        st.r_hint = max(st.r_hint, prev_hint)
    assert raised_to > 1024
    assert int(report[7]) == 0 and float(report[4]) > 0
