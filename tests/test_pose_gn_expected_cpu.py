"""CPU tests of the expected-depth Gauss-Newton residual: the float64 statement of the alpha-blended depth's pose tangents
(the one rtg_splat_pose_tangents_expected and rtg_splat_pose_gn_step_expected compute), pinned by central differences of
exp(h xi^) W2C; host-side validation of the two entry points and of the Python switches.

With the pairs a pixel blends, w_i = alpha_i T_i and z_i the view-space z of Gaussian i's centre:
  m1 = sum w_i,  m0 = sum w_i z_i,  D = m0 / m1,
  dz_i = (0, 0, 1, p_y, -p_x, 0),  dm1 = sum dw_i,  dm0 = sum (dw_i z_i + w_i dz_i),  dD = (dm0 - D dm1) / m1,
with dw_i = d alpha_i T_i + alpha_i dT_i as the colour tangents form it. The kernel carries dm1 as -dT_final (the sum
telescopes); the statement checks that identity too."""
import ctypes as C

import pytest
import torch

from test_pose_gn_cpu import STEPS, TWIST_POSES, _view, central
from test_pose_refine_cpu import POSES

FOCAL, CX, CY = 300.0, 80.0, 56.0


def _camera_points(w2c, pw):
    return pw @ w2c[:3, :3].t() + w2c[:3, 3]


def _alpha(pc, opacity, sigma, pix):
    """alpha of each Gaussian at pixel `pix`: opacity exp(-|u - pix|^2 / (2 sigma^2)), u the projected centre."""
    u = torch.stack([FOCAL * pc[:, 0] / pc[:, 2] + CX, FOCAL * pc[:, 1] / pc[:, 2] + CY], 1)
    d = u - pix
    return opacity * torch.exp(-0.5 * (d * d).sum(1) / sigma ** 2), u, d


def expected_depth(w2c, pw, opacity, sigma, pix):
    """(D, m1) of the blend in list order (front to back at the base pose)."""
    pc = _camera_points(w2c, pw)
    alpha, _, _ = _alpha(pc, opacity, sigma, pix)
    T, m0, m1 = 1.0, 0.0, 0.0
    for i in range(len(alpha)):
        w = alpha[i] * T
        m0, m1 = m0 + w * pc[i, 2], m1 + w
        T = T * (1 - alpha[i])
    return torch.stack([m0 / m1, torch.as_tensor(m1, dtype=torch.float64)])


def expected_depth_tangent(w2c, pw, opacity, sigma, pix):
    """The statement: dD (6,), dz (n, 6), and (sum dw, -dT_final) (6,) each."""
    pc = _camera_points(w2c, pw)
    alpha, u, d = _alpha(pc, opacity, sigma, pix)
    n = len(alpha)
    dz = torch.zeros((n, 6), dtype=torch.float64)
    dz[:, 2], dz[:, 3], dz[:, 4] = 1.0, pc[:, 1], -pc[:, 0]
    dD = torch.zeros(6, dtype=torch.float64)
    dm1_sum, dm1_tel = torch.zeros(6, dtype=torch.float64), torch.zeros(6, dtype=torch.float64)
    for k in range(6):
        rho, phi = torch.zeros(3, dtype=torch.float64), torch.zeros(3, dtype=torch.float64)
        (rho if k < 3 else phi)[k % 3] = 1.0
        dp = rho[None] + torch.linalg.cross(phi.expand(n, 3), pc)      # a view-space point moves as rho + phi x p_c
        du = FOCAL * (dp[:, :2] / pc[:, 2:3] - pc[:, :2] * dp[:, 2:3] / pc[:, 2:3] ** 2)
        dalpha = alpha * (-(d * du).sum(1) / sigma ** 2)
        T, dT, m0, m1, dm0, dm1 = 1.0, 0.0, 0.0, 0.0, 0.0, 0.0
        for i in range(n):
            w, dw = alpha[i] * T, dalpha[i] * T + alpha[i] * dT
            m0, m1 = m0 + w * pc[i, 2], m1 + w
            dm0, dm1 = dm0 + dw * pc[i, 2] + w * dz[i, k], dm1 + dw
            T, dT = T * (1 - alpha[i]), dT * (1 - alpha[i]) - T * dalpha[i]
        D = m0 / m1
        dD[k] = (dm0 - D * dm1) / m1
        dm1_sum[k], dm1_tel[k] = dm1, -dT
    return dD, dz, (dm1_sum, dm1_tel)


def ray_scene(w2c, coverage=None):
    """Three Gaussians near one pixel's ray at view depths 1.5, 2.0 and 2.6, a little off it; with `coverage`, their
    opacities are scaled (bisection) so that the pixel's m1 is that value."""
    pix = torch.tensor([70.0, 60.0], dtype=torch.float64)
    ray = torch.tensor([(pix[0] - CX) / FOCAL, (pix[1] - CY) / FOCAL, 1.0], dtype=torch.float64)
    z = torch.tensor([1.5, 2.0, 2.6], dtype=torch.float64)
    off = torch.tensor([[0.004, -0.003, 0.0], [-0.005, 0.002, 0.0], [0.003, 0.006, 0.0]], dtype=torch.float64)
    pc = z[:, None] * ray[None] + off
    c2w = torch.linalg.inv(w2c)
    pw = pc @ c2w[:3, :3].t() + c2w[:3, 3]
    opacity = torch.tensor([0.5, 0.6, 0.7], dtype=torch.float64)
    sigma = torch.tensor([2.0, 2.5, 3.0], dtype=torch.float64)
    if coverage is not None:
        lo, hi = 0.0, 1.0 / float(opacity.max())
        for _ in range(80):
            mid = 0.5 * (lo + hi)
            if float(expected_depth(w2c, pw, mid * opacity, sigma, pix)[1]) < coverage:
                lo = mid
            else:
                hi = mid
        opacity = hi * opacity
    return pw, opacity, sigma, pix


@pytest.mark.parametrize("coverage", [None, 0.5001])
@pytest.mark.parametrize("name", TWIST_POSES)
def test_expected_depth_tangent_matches_finite_differences(name, coverage):
    """dz and dD of the statement against central differences at steps h and h/4 (both must agree), at three poses and at
    a pixel whose coverage is just above the default min_coverage of 0.5; dm1 = sum dw_i equals -dT_final."""
    w2c = POSES[name]
    pw, opacity, sigma, pix = ray_scene(w2c, coverage)
    D, m1 = expected_depth(w2c, pw, opacity, sigma, pix)
    if coverage is not None:
        assert 0.5 < float(m1) < 0.5002
    dD, dz, (dm1_sum, dm1_tel) = expected_depth_tangent(w2c, pw, opacity, sigma, pix)
    assert float((dm1_sum - dm1_tel).abs().max()) <= 1e-12 * max(1.0, float(dm1_sum.abs().max()))
    for k in range(6):
        fz = [central(lambda m: _camera_points(m, pw)[:, 2], w2c, k, h) for h in STEPS]
        assert float((fz[1] - dz[:, k]).abs().max()) <= 1e-8, (k, fz[1], dz[:, k])
        fd = [central(lambda m: expected_depth(m, pw, opacity, sigma, pix)[0], w2c, k, h) for h in STEPS]
        scale = max(1.0, float(dD.abs().max()))
        assert abs(float(fd[0] - fd[1])) <= 1e-6 * scale, (k, fd)
        assert abs(float(fd[1] - dD[k])) <= 1e-6 * scale, (name, coverage, k, float(fd[1]), float(dD[k]))
    print(f"{name} coverage {float(m1):.4f}: D {float(D):.4f}, dD {dD.numpy()}")


# ------------------------------------------------------------------------------------------------- host-side validation
def test_pose_tangents_expected_validates_before_touching_cuda():
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    ok = C.c_void_p(256)
    view = _view()

    def call(v=C.byref(view), P=4, M=16, shs=ok, colors=None, scales=ok, rots=ok, cov=None, ws=ok, scratch=ok, J=ok, exp=ok):
        return L.rtg_splat_pose_tangents_expected(v, P, M, ok, shs, colors, scales, rots, cov, ws, ws, ws, 1024, ok, scratch, J,
                                                  exp, None)
    assert call(v=None) == -1 and b"view is NULL" in L.rtg_last_error()
    assert call(P=0) == -1 and b"P must be >= 1" in L.rtg_last_error()
    for kw in (dict(ws=None), dict(scratch=None)):
        assert call(**kw) == -1 and b"NULL pointer" in L.rtg_last_error(), kw
    for kw in (dict(J=None), dict(exp=None)):
        assert call(**kw) == -1 and b"J / expected is NULL" in L.rtg_last_error(), kw
    for kw in (dict(J=C.c_void_p(258)), dict(exp=C.c_void_p(258))):
        assert call(**kw) == -1 and b"4-byte aligned" in L.rtg_last_error(), kw
    assert call(colors=ok) == -1 and b"excatly one of either SHs" in L.rtg_last_error()
    assert call(cov=ok) == -1 and b"scale/rotation pair" in L.rtg_last_error()
    assert call(M=4) == -1 and b"M must hold" in L.rtg_last_error()
    assert call(scratch=C.c_void_p(264)) == -1 and b"16-byte aligned" in L.rtg_last_error()


def test_pose_gn_step_expected_validates_before_touching_cuda():
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    ok = C.c_void_p(256)
    view = _view()

    def state(**over):
        s = _lib.RtgPoseGN()
        for k in ("pose", "projection", "viewmatrix", "projmatrix", "campos", "render", "depth", "hit_depth", "gt_color", "gt_depth",
                  "scratch", "report"):
            setattr(s, k, 256)
        s.color_weight, s.depth_weight, s.depth_error_max, s.damping = 0.8, 1.0, 0.1, 1e-4
        for k, v in over.items():
            setattr(s, k, v)
        return s

    def robust(kernel=_lib.RTG_ROBUST_NONE, cd=0.1, dd=0.05):
        r = _lib.RtgPoseRobust()
        r.kernel, r.color_delta, r.depth_delta = kernel, cd, dd
        return r

    def exposure(ab):
        e = _lib.RtgPoseExposure()
        e.ab = ab
        return e

    def call(s, r=None, e=None, min_coverage=0.5, P=4, no_robust=False):
        r = robust() if r is None else r
        return L.rtg_splat_pose_gn_step_expected(C.byref(view), P, 16, ok, ok, None, ok, ok, None, ok, ok, ok, 1024, ok,
                                                 None if s is None else C.byref(s), None if no_robust else C.byref(r),
                                                 None if e is None else C.byref(e), min_coverage, None)
    assert call(None) == -1 and b"state is NULL" in L.rtg_last_error()
    assert call(state(), no_robust=True) == -1 and b"robust is NULL" in L.rtg_last_error()
    assert call(state(), r=robust(kernel=7)) == -1 and b"unknown robust kernel" in L.rtg_last_error()
    for cd, dd in ((0.0, 0.05), (0.1, -1.0), (float("inf"), 0.05), (0.1, float("nan"))):
        assert call(state(), r=robust(_lib.RTG_ROBUST_HUBER, cd, dd)) == -1 and b"positive and finite" in L.rtg_last_error()
    for mc in (0.0, -0.5, 1.0001, float("nan"), float("inf")):
        assert call(state(), min_coverage=mc) == -1 and b"min_coverage must be in (0, 1]" in L.rtg_last_error(), mc
    assert call(state(), e=exposure(None)) == -1 and b"exposure ab is NULL" in L.rtg_last_error()
    assert call(state(), e=exposure(260)) == -1 and b"8-byte aligned" in L.rtg_last_error()
    assert call(state(), P=0) == -1 and b"P must be >= 1" in L.rtg_last_error()
    for k in ("hit_depth", "scratch"):
        assert call(state(**{k: None})) == -1 and b"NULL pointer" in L.rtg_last_error(), k
    for k in ("pose", "projection", "viewmatrix", "projmatrix", "campos", "report"):
        assert call(state(**{k: None})) == -1 and b"NULL pose / projection" in L.rtg_last_error(), k
    for k in ("render", "depth", "gt_color", "gt_depth"):
        assert call(state(**{k: None})) == -1 and b"NULL render" in L.rtg_last_error(), k
    for k in ("damping", "color_weight", "depth_weight"):
        assert call(state(**{k: -1.0})) == -1 and b">= 0" in L.rtg_last_error(), k


def test_python_switches_raise_before_cuda_work():
    """`depth` and `min_coverage` are checked before any tensor is touched (the map and frame here are not tensors)."""
    from rtg_slam_b200.tracking import PoseRefiner, pose_jacobian
    with pytest.raises(ValueError, match="depth must be"):
        pose_jacobian(None, None, None, depth="median")
    ref = PoseRefiner.__new__(PoseRefiner)
    for kw, msg in ((dict(depth="median"), "depth must be"), (dict(depth="expected", min_coverage=0.0), "min_coverage"),
                    (dict(depth="expected", min_coverage=1.5), "min_coverage"),
                    (dict(depth="expected", min_coverage=float("nan")), "min_coverage")):
        with pytest.raises(ValueError, match=msg):
            ref.refine_gn(None, None, None, None, iters=1, **kw)
