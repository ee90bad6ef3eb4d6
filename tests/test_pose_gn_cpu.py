"""CPU tests of the Gauss-Newton pose step: the twist statements the forward-mode tangents rest on, pinned by central
finite differences of exp(h xi^) W2C; a float64 statement of the device step (`gn_step`), checked against an independent
formulation and reused by the GPU tests; host-side validation of the three new entry points.

Pose and twist as in rtg_pose_adam_step: W2C(xi) = exp(xi^) W2C with xi = (rho, phi). Under it a view-space point moves as
dp_c = rho + phi x p_c, a view-space direction as dn = phi x n, the view rotation as dW = [phi]x W and the camera centre as
d campos = -W^T rho."""
import ctypes as C
import math

import pytest
import torch

from test_pose_refine_cpu import POSES, hat

TWIST_POSES = ("identity", "rotated", "half_turn")   # identity, 35 and 150 degree rotations
STEPS = (1e-5, 2.5e-6)


def cross(a, b):
    return torch.linalg.cross(a, b)


def central(fn, w2c, k, h):
    e = torch.zeros(6, dtype=torch.float64)
    e[k] = h
    return (fn(torch.matrix_exp(hat(e)) @ w2c) - fn(torch.matrix_exp(hat(-e)) @ w2c)) / (2 * h)


def check_tangent(fn, w2c, want, tol=1e-8):
    """want(k) is the claimed tangent along direction k; both difference steps must agree with it."""
    for k in range(6):
        claimed = want(k)
        scale = max(1.0, float(claimed.abs().max()))
        fd = [central(fn, w2c, k, h) for h in STEPS]
        assert float((fd[0] - fd[1]).abs().max()) <= tol * scale, (k, fd)
        assert float((fd[1] - claimed).abs().max()) <= tol * scale, (k, fd[1], claimed)


def unit(k):
    e = torch.zeros(6, dtype=torch.float64)
    e[k] = 1.0
    return e[:3], e[3:]


def plane_depth(pc, n, ray):
    """The rasterizer's plane depth of a surfel hit along `ray`: ray.z (n . p_c) / (n . ray + 1e-8)."""
    return ray[2] * torch.dot(n, pc) / (torch.dot(n, ray) + 1e-8)


def plane_depth_tangent(pc, n, ray):
    """d D / d xi (6): d(n . p_c) = n . rho (a rotation moves n and p_c alike), d(n . ray) = phi . (n x ray)."""
    nr = torch.dot(n, ray) + 1e-8
    return torch.cat([ray[2] * n / nr, -ray[2] * torch.dot(n, pc) * cross(n, ray) / nr ** 2])


@pytest.mark.parametrize("name", TWIST_POSES)
def test_twist_statements_match_finite_differences(name):
    w2c = POSES[name]
    gen = torch.Generator().manual_seed(11)
    p = torch.randn(3, generator=gen, dtype=torch.float64) + torch.tensor([0.0, 0.0, 3.0], dtype=torch.float64)
    n_w = torch.randn(3, generator=gen, dtype=torch.float64)
    n_w = n_w / n_w.norm()
    R = w2c[:3, :3]
    pc = R @ p + w2c[:3, 3]
    nc = R @ n_w
    # view-space point, view-space direction, view rotation, camera centre
    check_tangent(lambda T: T[:3, :3] @ p + T[:3, 3], w2c, lambda k: unit(k)[0] + cross(unit(k)[1], pc))
    check_tangent(lambda T: T[:3, :3] @ n_w, w2c, lambda k: cross(unit(k)[1], nc))
    check_tangent(lambda T: T[:3, :3], w2c, lambda k: hat(torch.cat([torch.zeros(3, dtype=torch.float64), unit(k)[1]]))[:3, :3] @ R)
    check_tangent(lambda T: -(T[:3, :3].t() @ T[:3, 3]), w2c, lambda k: -(R.t() @ unit(k)[0]))
    # the plane depth of a surfel at world point p with world normal n_w, seen along a fixed pixel ray
    ray = torch.tensor([0.1, -0.2, 1.0], dtype=torch.float64)
    ray = ray / ray.norm()
    J = plane_depth_tangent(pc, nc, ray)
    check_tangent(lambda T: plane_depth(T[:3, :3] @ p + T[:3, 3], T[:3, :3] @ n_w, ray), w2c, lambda k: J[k], tol=1e-7)
    # the centre depth: (rho + phi x p_c).z
    check_tangent(lambda T: (T[:3, :3] @ p + T[:3, 3])[2], w2c, lambda k: (unit(k)[0] + cross(unit(k)[1], pc))[2])


# ------------------------------------------------------------------------------------------------- the step statement
def se3_exp_closed(xi):
    """exp(xi^) in closed form, as the device computes it (R = I + a K + b K^2, V = I + b K + c K^2)."""
    rho, phi = xi[:3], xi[3:]
    th2 = float(phi @ phi)
    if th2 < 1e-4:
        a = 1 - th2 / 6 * (1 - th2 / 20)
        b = 0.5 - th2 / 24 * (1 - th2 / 30)
        c = 1 / 6 - th2 / 120 * (1 - th2 / 42)
    else:
        th = math.sqrt(th2)
        a, b, c = math.sin(th) / th, (1 - math.cos(th)) / th2, (th - math.sin(th)) / (th2 * th)
    K = hat(torch.cat([torch.zeros(3, dtype=xi.dtype), phi]))[:3, :3]
    I = torch.eye(3, dtype=xi.dtype)
    E = torch.eye(4, dtype=xi.dtype)
    E[:3, :3] = I + a * K + b * K @ K
    E[:3, 3] = (I + b * K + c * K @ K) @ rho
    return E


def normal_equations(Jc, rc, sel_c, Jd, rd, sel_d, color_weight, depth_weight):
    """H (6,6), g (6), (E, E_colour, E_depth), N_c, N_d of E = 1/2 [w_c/N_c sum_{S_c} sum_ch r^2 + w_d/N_d sum_{S_d} r^2].
    Jc (6, 3, n), rc (3, n), Jd (6, n), rd (n); sel_* boolean (n,). Float64."""
    nc, nd = 3.0 * float(sel_c.sum()), float(sel_d.sum())
    wc = color_weight / nc if nc > 0 else 0.0
    wd = depth_weight / nd if nd > 0 else 0.0
    Jc, rc = Jc[..., sel_c], rc[:, sel_c]
    Jd, rd = Jd[:, sel_d], rd[sel_d]
    H = wc * torch.einsum("acn,bcn->ab", Jc, Jc) + wd * Jd @ Jd.t()
    g = wc * torch.einsum("acn,cn->a", Jc, rc) + wd * Jd @ rd
    ec, ed = 0.5 * wc * float((rc * rc).sum()), 0.5 * wd * float((rd * rd).sum())
    return H, g, (ec + ed, ec, ed), nc, nd


def gn_step(H, g, damping, w2c):
    """The device step from H and g: trace damping, Cholesky solve, closed-form exponential, left update. Returns
    (new W2C, xi) or (w2c, None) when the damped system is not positive definite."""
    A = H + damping * torch.trace(H) * torch.eye(6, dtype=H.dtype)
    L, info = torch.linalg.cholesky_ex(A)
    if int(info) != 0:
        return w2c, None
    xi = torch.cholesky_solve(-g[:, None], L)[:, 0]
    return se3_exp_closed(xi) @ w2c, xi


def random_problem(seed, n=500):
    gen = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
    return r(6, 3, n), r(3, n), torch.rand(n, generator=gen) < 0.7, r(6, n), r(n) * 0.1, torch.rand(n, generator=gen) < 0.4


@pytest.mark.parametrize("name,scale", [("identity", 1e-2), ("rotated", 1.0), ("half_turn", 30.0)])
def test_step_statement_matches_solve_and_matrix_exp(name, scale):
    """H and g against autograd of E through xi (E is quadratic in xi for fixed J), the step against torch.linalg.solve and
    torch.matrix_exp. `scale` spans both branches of the closed-form exponential."""
    w2c = POSES[name]
    Jc, rc, sel_c, Jd, rd, sel_d = random_problem(3)
    rc, rd = rc * scale, rd * scale
    H, g, (E, ec, ed), nc, nd = normal_equations(Jc, rc, sel_c, Jd, rd, sel_d, 0.8, 1.0)
    xi0 = torch.zeros(6, dtype=torch.float64, requires_grad=True)
    rcl = rc[:, sel_c] + torch.einsum("a,acn->cn", xi0, Jc[..., sel_c])
    rdl = rd[sel_d] + xi0 @ Jd[:, sel_d]
    El = 0.5 * (0.8 / nc * (rcl ** 2).sum() + 1.0 / nd * (rdl ** 2).sum())
    (gl,) = torch.autograd.grad(El, xi0, create_graph=True)
    Hl = torch.stack([torch.autograd.grad(gl[k], xi0, retain_graph=True)[0] for k in range(6)])
    assert abs(float(El.detach()) - E) <= 1e-12 * abs(E) and abs(ec + ed - E) <= 1e-15 * abs(E)
    assert float((gl - g).abs().max()) <= 1e-12 * float(g.abs().max())
    assert float((Hl - H).abs().max()) <= 1e-12 * float(H.abs().max())
    damping = 1e-4
    new, xi = gn_step(H, g, damping, w2c)
    xi_ref = torch.linalg.solve(H + damping * torch.trace(H) * torch.eye(6, dtype=torch.float64), -g)
    assert float((xi - xi_ref).abs().max()) <= 1e-12 * float(xi_ref.abs().max())
    ref = torch.matrix_exp(hat(xi_ref)) @ w2c
    assert float((new - ref).abs().max()) <= 1e-12 * max(1.0, float(ref.abs().max()))


def test_step_statement_edge_cases():
    """An empty depth set contributes nothing; an all-zero system is singular and leaves the pose."""
    Jc, rc, sel_c, Jd, rd, _ = random_problem(4)
    none = torch.zeros_like(sel_c)
    H, g, (E, ec, ed), nc, nd = normal_equations(Jc, rc, sel_c, Jd, rd, none, 0.8, 1.0)
    H2, g2, _, _, _ = normal_equations(Jc, rc, sel_c, Jd, rd, none, 0.8, 0.0)
    assert nd == 0 and ed == 0.0 and torch.equal(H, H2) and torch.equal(g, g2)
    w2c = POSES["rotated"]
    new, xi = gn_step(torch.zeros((6, 6), dtype=torch.float64), torch.zeros(6, dtype=torch.float64), 1e-4, w2c)
    assert xi is None and torch.equal(new, w2c)


# ------------------------------------------------------------------------------------------------- host-side validation
def _view():
    from rtg_slam_b200 import _lib
    view = _lib.RtgSplatView()
    view.image_height, view.image_width, view.sh_degree = 48, 64, 3
    view.viewmatrix = view.projmatrix = view.campos = view.bg = 256  # never dereferenced: validation fails first
    return view


def test_scratch_bytes_is_host_only():
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    tiles = 3 * 4
    assert L.rtg_splat_pose_gn_scratch_bytes(1000, 48, 64) == ((1000 * 192 + 255) // 256) * 256 + tiles * 58 * 8
    assert L.rtg_splat_pose_gn_scratch_bytes(-1, 48, 64) == 0 and L.rtg_splat_pose_gn_scratch_bytes(10, 0, 64) == 0


def test_pose_tangents_validates_before_touching_cuda():
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    ok = C.c_void_p(256)
    view = _view()

    def call(v=C.byref(view), P=4, M=16, shs=ok, colors=None, scales=ok, rots=ok, cov=None, ws=ok, hit=ok, scratch=ok, J=ok):
        return L.rtg_splat_pose_tangents(v, P, M, ok, shs, colors, scales, rots, cov, ws, ws, ws, 1024, ok, hit, scratch, J, None)
    assert call(v=None) == -1 and b"view is NULL" in L.rtg_last_error()
    assert call(P=0) == -1 and b"P must be >= 1" in L.rtg_last_error()
    for kw in (dict(ws=None), dict(hit=None), dict(scratch=None)):
        assert call(**kw) == -1 and b"NULL pointer" in L.rtg_last_error(), kw
    assert call(J=None) == -1 and b"J is NULL" in L.rtg_last_error()
    assert call(colors=ok) == -1 and b"excatly one of either SHs" in L.rtg_last_error()
    assert call(cov=ok) == -1 and b"scale/rotation pair" in L.rtg_last_error()
    assert call(M=4) == -1 and b"M must hold" in L.rtg_last_error()
    assert call(scratch=C.c_void_p(264)) == -1 and b"16-byte aligned" in L.rtg_last_error()


def test_pose_gn_step_validates_before_touching_cuda():
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

    def call(s, P=4):
        return L.rtg_splat_pose_gn_step(C.byref(view), P, 16, ok, ok, None, ok, ok, None, ok, ok, ok, 1024, ok,
                                        None if s is None else C.byref(s), None)
    assert call(None) == -1 and b"state is NULL" in L.rtg_last_error()
    assert call(state(), P=0) == -1 and b"P must be >= 1" in L.rtg_last_error()
    for k in ("hit_depth", "scratch"):
        assert call(state(**{k: None})) == -1 and b"NULL pointer" in L.rtg_last_error(), k
    for k in ("pose", "projection", "viewmatrix", "projmatrix", "campos", "report"):
        assert call(state(**{k: None})) == -1 and b"NULL pose / projection" in L.rtg_last_error(), k
    for k in ("render", "depth", "gt_color", "gt_depth"):
        assert call(state(**{k: None})) == -1 and b"NULL render" in L.rtg_last_error(), k
    assert call(state(pose=260)) == -1 and b"8-byte aligned" in L.rtg_last_error()
    assert call(state(report=260)) == -1 and b"8-byte aligned" in L.rtg_last_error()
    for k in ("damping", "color_weight", "depth_weight"):
        assert call(state(**{k: -1.0})) == -1 and b">= 0" in L.rtg_last_error(), k
    assert call(state(damping=float("nan"))) == -1
