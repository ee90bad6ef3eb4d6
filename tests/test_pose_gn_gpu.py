"""GPU tests of the Gauss-Newton pose step: the forward-mode tangent images (rtg_splat_pose_tangents through
tracking.pose_jacobian) against central differences of the float64 oracle and, by the adjoint identity, against the pinned
reverse-mode camera gradient; the normal equations and the device step (rtg_splat_pose_gn_step) against float64
statements; the forward left unchanged; PoseRefiner.refine_gn."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

import helpers
from oracle.splat_oracle import OracleRender
from rtg_slam_b200 import scene
from test_camera_grad_gpu import CAM, KW, inputs_for, pose_error, scene_case, se3_exp, view_camera
from test_pose_gn_cpu import gn_step, normal_equations
from test_pose_refine_cpu import camera_arrays, hat, tangent_grad
from test_pose_refine_gpu import ARGS, refiner_camera

pytestmark = pytest.mark.gpu


def jacobian(cam, inputs, dev, mask=None, **over):
    from rtg_slam_b200.tracking import pose_jacobian
    t = {KW[k]: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in inputs.items()}
    tm = None if mask is None else torch.from_numpy(np.ascontiguousarray(mask, dtype=np.int32)).to(dev)
    outs, J = pose_jacobian(helpers.make_settings(cam, dev, **over), tile_mask=tm, **t)
    return [o.cpu().numpy() for o in outs], J.cpu().numpy().astype(np.float64)


# ------------------------------------------------------------------------------------------- tangents vs the f64 oracle
def oracle_at(cam, inputs, w2c, mask, over):
    """f64 oracle forward at the pose w2c (camera arrays formed in double, not rounded to float32)."""
    projection = cam.projection.astype(np.float64)
    view = w2c.T
    c = types.SimpleNamespace(height=cam.height, width=cam.width, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, cx=cam.cx, cy=cam.cy,
                              viewmatrix=view, projmatrix=view @ projection, campos=-(w2c[:3, :3].T @ w2c[:3, 3]))
    g = {k: (None if inputs.get(k) is None else inputs[k].astype(np.float64)) for k in ("xyz", "opacity", "shs", "scales", "rotations")}
    cp, cv = inputs.get("colors_precomp"), inputs.get("cov3D_precomp")
    o = OracleRender(c, g, tile_mask=mask, precision="f64", colors_precomp=None if cp is None else cp.astype(np.float64),
                     cov3D_precomp=None if cv is None else cv.astype(np.float64), **over).outputs()
    return o[0], o[1][0], o[3][0]


def expm(xi):
    return torch.matrix_exp(hat(torch.from_numpy(xi))).numpy()


TAN_CONFIGS = [("small", "sh"), ("masked", "sh"), ("ragged", "sh"), ("small", "colors_precomp"), ("ragged", "cov3D_precomp"),
               ("masked", "M4")]


@pytest.mark.parametrize("name,mode", TAN_CONFIGS)
def test_tangent_images_match_f64_oracle(cuda_device, name, mode):
    """Central differences of the f64 oracle along each twist direction, steps h and h/4; a pixel where the two disagree
    (a decision flipped inside the step) or whose depth hit differs is skipped. The rest agree within 1e-3 of each
    (direction, colour | depth) block's largest entry."""
    cam, g, mask = scene_case(name)
    inputs, over = inputs_for(g, mode)
    outs, J = jacobian(cam, inputs, cuda_device, mask, **over)
    w2c = np.linalg.inv(cam.c2w)
    _, _, hit0 = oracle_at(cam, inputs, w2c, mask, over)
    kernel_hit = outs[3][0]
    h = 1e-4
    skipped = total = 0
    for k in range(6):
        fd = []
        hits = [hit0]
        for step in (h, h / 4):
            e = np.zeros(6)
            e[k] = step
            cp, dp, hp = oracle_at(cam, inputs, expm(e) @ w2c, mask, over)
            cm, dm, hm = oracle_at(cam, inputs, expm(-e) @ w2c, mask, over)
            fd.append((np.concatenate([cp, dp[None]]) - np.concatenate([cm, dm[None]])) / (2 * step))
            hits += [hp, hm]
        same_hit = np.all([hh == hit0 for hh in hits], axis=0) & (kernel_hit == hit0)
        for blk, sl in (("colour", slice(0, 3)), ("depth", slice(3, 4))):
            a, b, got = fd[0][sl], fd[1][sl], J[k, sl]
            scale = np.abs(b).max()
            if scale == 0:  # e.g. centre depths under a rotation about the optical axis at the identity pose
                assert np.abs(got).max() <= 1e-6, (name, mode, k, blk, np.abs(got).max())
                continue
            keep = np.abs(a - b) <= 2e-4 * scale
            if blk == "depth":
                keep &= same_hit[None]
            skipped += int((~keep).sum())
            total += keep.size
            err = np.abs(got - b)[keep].max() / scale
            print(f"{name}/{mode} direction {k} {blk}: max err {err:.2e} of the block max {scale:.3e}, "
                  f"skipped {(~keep).mean():.2%}")
            assert err <= 1e-3, (name, mode, k, blk, err)
    frac = skipped / total
    print(f"{name}/{mode}: skipped fraction {frac:.3%}")
    assert frac < 0.02, frac


# ------------------------------------------------------------------------------- adjoint identity vs the reverse path
@pytest.fixture(scope="module")
def room_1m():
    return scene.surfel_room(1_000_000, seed=2024)


def reverse_twist_grad(cam, inputs, dev, uc, ud, mask):
    """The existing pose-only backward fed the upstreams (uc, ud), mapped to dL/dxi by tangent_grad."""
    from rtg_slam_b200.rasterizer import GaussianRasterizer
    rs = helpers.make_settings(cam, dev)
    for k in CAM:
        getattr(rs, k).requires_grad_(True)
    t = {KW[k]: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in inputs.items()}
    tm = None if mask is None else torch.from_numpy(np.ascontiguousarray(mask, dtype=np.int32)).to(dev)
    out = GaussianRasterizer(rs)(**t, tile_mask=tm)
    ((out[0] * uc).sum() + (out[1] * ud).sum()).backward()
    d = [getattr(rs, k).grad.double().cpu() for k in CAM]
    w2c = torch.from_numpy(np.linalg.inv(cam.c2w))
    return tangent_grad(d[0].view(4, 4), d[1].view(4, 4), d[2], w2c, torch.from_numpy(cam.projection.astype(np.float64))).numpy()


@pytest.mark.parametrize("cam_name,masked", [("replica", False), ("hd", False), ("replica", True)])
def test_adjoint_identity_against_the_reverse_path(cuda_device, room_1m, cam_name, masked):
    dev = cuda_device
    cam = scene.make_camera(cam_name, c2w=scene.small_pose())
    mask = scene.random_tile_mask(cam, 0.5, seed=143) if masked else None
    inputs = {k: room_1m[k] for k in ("xyz", "opacity", "shs", "scales", "rotations")}
    gen = torch.Generator(device=dev).manual_seed(21)
    uc = torch.randn((3, cam.height, cam.width), device=dev, generator=gen)
    ud = torch.randn((1, cam.height, cam.width), device=dev, generator=gen)
    _, J = jacobian(cam, inputs, dev, mask)
    fwd = np.einsum("kqhw,qhw->k", J, np.concatenate([uc.cpu().numpy(), ud.cpu().numpy()]).astype(np.float64))
    rev = reverse_twist_grad(cam, inputs, dev, uc, ud, mask)
    rev2 = reverse_twist_grad(cam, inputs, dev, uc, ud, mask)
    scale = np.abs(rev).max()
    spread = np.abs(rev - rev2).max() / scale
    err = np.abs(fwd - rev).max() / scale
    print(f"{cam_name}{' masked' if masked else ''}: forward-mode vs reverse-mode twist gradient {err:.2e} "
          f"(reverse run-to-run {spread:.2e})\n  fwd {fwd}\n  rev {rev}")
    assert err <= max(1e-4, 10 * spread), (err, spread)


# ------------------------------------------------------------------------------------ normal equations and the step
def gn_inputs(dev, masks="none"):
    """The refiner's test scene: targets rendered at the true pose, the start 1 deg / 2 cm away."""
    from rtg_slam_b200.render import Renderer
    cam = scene.make_camera("small")
    g = {k: torch.from_numpy(v).to(dev) for k, v in scene.surfel_room(20_000, seed=7).items()}
    w2c_true = torch.from_numpy(np.linalg.inv(scene.small_pose()).astype(np.float32)).to(dev)
    with torch.no_grad():
        tgt = Renderer(ARGS).render(view_camera(cam, w2c_true), g)
    w2c0 = se3_exp(torch.tensor([0.012, -0.010, 0.012, 0.010, -0.012, 0.008], device=dev)) @ w2c_true
    kw, gm = {}, g
    if masks == "render_mask":
        keep = g["xyz"][:, 0] < 0.5
        gm = {k: v[keep] for k, v in g.items()}
        with torch.no_grad():
            kw["render_mask"] = Renderer(ARGS).render(view_camera(cam, w2c0), gm)["T_map"][0] != 1
    elif masks == "tile_mask":
        kw["tile_mask"] = torch.from_numpy(scene.random_tile_mask(cam, 0.5, seed=143)).to(dev)
    return cam, gm, tgt, w2c_true, w2c0, kw


def run_step(refiner, cam, g, tgt, w2c0, dev, render_mask=None, damping=1e-4):
    """One forward + tangent images + rtg_splat_pose_gn_step on that same forward, writing to fresh pose / camera arrays
    (so the forward's own arrays are not touched). Returns J, outputs, the per-tile partial sums, the new pose, arrays
    and report."""
    from rtg_slam_b200 import _lib, rasterizer
    from rtg_slam_b200.tracking import _native_args
    L = _lib.lib()
    _, pose, projection, view, proj, campos, rs, gg = refiner._setup(refiner_camera(cam, w2c0.double()), g, requires_grad=False)
    outs, saved, ins = rasterizer._forward_native(rs, gg["xyz"], gg["shs"], None, gg["opacity"], gg["scales"], gg["rotations"],
                                                  None, None)
    rasterizer._state(dev).read(saved.pending, block=True)
    assert not saved.pending.overflow
    H, W = cam.height, cam.width
    P = int(gg["xyz"].shape[0])
    nbytes = int(L.rtg_splat_pose_gn_scratch_bytes(P, H, W))
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    scratch = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
    J = torch.empty((6, 4, H, W), device=dev)
    _lib.check(L.rtg_splat_pose_tangents(*_native_args(rs, saved, ins, dev), C.c_void_p(outs[3].data_ptr()),
                                         C.c_void_p(scratch.data_ptr()), C.c_void_p(J.data_ptr()), stream), "tangents")
    res = []
    for _ in range(2):
        new_pose = pose.clone()
        arrays = [torch.full_like(t, float("nan")) for t in (view, proj, campos)]
        report = torch.zeros(8, dtype=torch.float64, device=dev)
        scratch.zero_()
        mask = None if render_mask is None else render_mask.to(torch.uint8).contiguous()
        s = _lib.RtgPoseGN()
        s.pose, s.projection = new_pose.data_ptr(), projection.data_ptr()
        s.viewmatrix, s.projmatrix, s.campos = (a.data_ptr() for a in arrays)
        s.render, s.depth, s.hit_depth = outs[0].data_ptr(), outs[1].data_ptr(), outs[3].data_ptr()
        s.gt_color, s.gt_depth = tgt["render"].contiguous().data_ptr(), tgt["depth"].contiguous().data_ptr()
        s.render_mask = None if mask is None else mask.data_ptr()
        s.scratch, s.report = scratch.data_ptr(), report.data_ptr()
        s.color_weight, s.depth_weight, s.depth_error_max, s.damping = 0.8, 1.0, 0.1, damping
        _lib.check(L.rtg_splat_pose_gn_step(*_native_args(rs, saved, ins, dev), C.byref(s), stream), "step")
        # the per-tile partial sums sit after the tangent rows (rtg_splat_pose_gn_scratch_bytes)
        off = (P * 192 + 255) // 256 * 256
        T = ((H + 15) // 16) * ((W + 15) // 16)
        partial = scratch[off:off + T * 58 * 8].view(torch.float64).view(T, 58).cpu()
        res.append((partial, new_pose.cpu(), [a.cpu() for a in arrays], report.cpu()))
    return J.cpu().double(), [o.cpu() for o in outs], res, pose.cpu()


@pytest.mark.parametrize("masks", ["none", "render_mask"])
def test_normal_equations_and_step_match_f64_statements(cuda_device, masks):
    from rtg_slam_b200.tracking import PoseRefiner
    dev = cuda_device
    cam, g, tgt, _, w2c0, kw = gn_inputs(dev, masks)
    J, outs, ((part, pose1, arr1, rep1), (part2, pose2, arr2, rep2)), pose0 = run_step(PoseRefiner(ARGS), cam, g, tgt, w2c0, dev,
                                                                                        kw.get("render_mask"))
    # bit-identical from run to run
    assert torch.equal(part, part2) and torch.equal(pose1, pose2) and torch.equal(rep1, rep2)
    assert all(torch.equal(a, b) for a, b in zip(arr1, arr2))
    # the f64 statement from the MODE_IMAGES output, the same residuals and the same selection
    color, depth, hit = outs[0].double(), outs[1][0].double(), outs[3][0]
    H_, W_ = cam.height, cam.width
    gtc, gtd = tgt["render"].cpu().double(), tgt["depth"].cpu().double()[0]
    m = torch.ones((H_, W_), dtype=torch.bool) if "render_mask" not in kw else kw["render_mask"].cpu().bool()
    rd = depth - gtd
    sel_d = m & (hit != -1) & (gtd > 0) & ((outs[1][0] - tgt["depth"].cpu()[0]) < torch.tensor(0.1, dtype=torch.float32))
    Jc, Jd = J[:, :3].reshape(6, 3, -1), J[:, 3].reshape(6, -1)
    Hm, gv, (E, ec, ed), nc, nd = normal_equations(Jc, (color - gtc).reshape(3, -1), m.reshape(-1), Jd, rd.reshape(-1),
                                                   sel_d.reshape(-1), 0.8, 1.0)
    tot = part.sum(0)
    c, d = tot[:29], tot[29:]
    assert int(c[28]) * 3 == nc and int(d[28]) == nd and nd > 0
    wc, wd = 0.8 / nc, 1.0 / nd
    iu = torch.triu_indices(6, 6)
    Hk = torch.zeros((6, 6), dtype=torch.float64)
    Hk[iu[0], iu[1]] = wc * c[:21] + wd * d[:21]
    Hk = Hk + Hk.triu(1).t()
    gk = wc * c[21:27] + wd * d[21:27]
    for what, got, want in (("H", Hk, Hm), ("g", gk, gv)):
        err = float((got - want).abs().max() / want.abs().max())
        print(f"{masks}: {what} rel err {err:.2e}")
        assert err <= 1e-5, (what, err)
    assert abs(float(rep1[0]) - E) <= 1e-5 * E and abs(float(rep1[1]) - ec) <= 1e-5 * ec and abs(float(rep1[2]) - ed) <= 1e-5 * ed
    assert float(rep1[3]) == nc and float(rep1[4]) == nd and float(rep1[7]) == 0
    # the device step against the f64 statement, from the kernel's own H and g
    want, xi = gn_step(Hk, gk, 1e-4, pose0)
    assert float((pose1 - want).abs().max()) <= 1e-6, (pose1, want)
    assert abs(float(rep1[5]) - float(xi[:3].norm())) <= 1e-9 and abs(float(rep1[6]) - float(xi[3:].norm())) <= 1e-9
    view, proj, campos = camera_arrays(pose1, torch.from_numpy(cam.projection.astype(np.float64)))
    for got, ref in zip(arr1, (view, proj, campos)):
        assert float((got.double().reshape(ref.shape) - ref).abs().max()) <= 1e-6 * max(1.0, float(ref.abs().max()))


def test_the_forward_is_unchanged(cuda_device):
    """The outputs of a render are bit-identical with and without the tangent pass run after it."""
    from rtg_slam_b200.rasterizer import GaussianRasterizer
    cam, g, mask = scene_case("masked")
    inputs, _ = inputs_for(g, "sh")
    t = {KW[k]: torch.from_numpy(np.ascontiguousarray(v)).to(cuda_device) for k, v in inputs.items()}
    tm = torch.from_numpy(np.ascontiguousarray(mask, dtype=np.int32)).to(cuda_device)
    with torch.no_grad():
        plain = [o.cpu().numpy() for o in GaussianRasterizer(helpers.make_settings(cam, cuda_device))(**t, tile_mask=tm)]
    with_tan, _ = jacobian(cam, inputs, cuda_device, mask)
    for a, b in zip(plain, with_tan):
        assert np.array_equal(a, b)


# -------------------------------------------------------------------------------------------------------- refinement
GN_ITERS = 10
# Iterations measured on an H100 to reach a tenth of both errors: 7 without masks, 6 with the tile mask. With the render
# mask (a partial map whose silhouette pixels disagree with the full-map target) the squared-residual optimum sits off the
# true pose: after 10 iterations the rotation error is at 0.056 of its start and the translation error at 0.147 (0.29 cm),
# where it stays; that case asserts the measured plateau (rotation below a tenth, translation below a fifth).
PLATEAU = {"render_mask": (0.1, 0.2)}


@pytest.mark.parametrize("masks", ["none", "render_mask", "tile_mask"])
def test_refine_gn_converges(cuda_device, masks):
    """The Adam refiner's 1 deg / 2 cm scene: Gauss-Newton reaches a tenth of both errors within GN_ITERS iterations
    (PLATEAU: the measured bound of the partial-map case)."""
    from rtg_slam_b200.tracking import PoseRefiner
    dev = cuda_device
    cam, g, tgt, w2c_true, w2c0, kw = gn_inputs(dev, masks)
    ang0, tr0 = pose_error(w2c0, w2c_true)
    fa, ft = PLATEAU.get(masks, (0.1, 0.1))
    ref = PoseRefiner(ARGS)
    reached = None
    for it in range(1, GN_ITERS + 1):
        w2c, report = ref.refine_gn(refiner_camera(cam, w2c0), g, tgt["render"], tgt["depth"], iters=it, color_weight=1.0,
                                    depth_weight=1.0, **kw)
        ang, tr = pose_error(w2c, w2c_true.double())
        print(f"refine_gn ({masks}) {it} iterations: rotation {ang0:.3f} -> {ang:.4f} deg, translation {100 * tr0:.2f} -> "
              f"{100 * tr:.3f} cm, report {report.cpu().numpy()}")
        assert int(report[7]) == 0
        if ang < fa * ang0 and tr < ft * tr0:
            reached = it
            break
    assert w2c.shape == (4, 4) and w2c.dtype == torch.float64 and w2c.is_cuda
    assert reached is not None, (masks, ang0, ang, tr0, tr)


def test_refine_gn_renders_an_overflowed_iteration_again(cuda_device):
    from rtg_slam_b200 import rasterizer
    from rtg_slam_b200.tracking import PoseRefiner
    dev = cuda_device
    cam, g, tgt, w2c_true, w2c0, _ = gn_inputs(dev)
    st = rasterizer._state(dev)
    prev_mode, prev_hint = st.mode, st.r_hint
    rasterizer.set_capacity_checks("deferred", dev)
    st.r_hint = 1024
    try:
        w2c, report = PoseRefiner(ARGS).refine_gn(refiner_camera(cam, w2c0), g, tgt["render"], tgt["depth"], iters=8,
                                                  color_weight=1.0, depth_weight=1.0)
        raised_to = st.r_hint
    finally:
        rasterizer.set_capacity_checks(prev_mode, dev)
        st.r_hint = max(st.r_hint, prev_hint)
    assert raised_to > 1024
    assert int(report[7]) == 0 and float(report[4]) > 0
    ang0, tr0 = pose_error(w2c0, w2c_true)
    ang, tr = pose_error(w2c, w2c_true.double())
    assert ang < 0.1 * ang0 and tr < 0.1 * tr0, (ang0, ang, tr0, tr)
