"""CPU tests of pose refinement: a float64 torch statement of rtg_pose_adam_step's tangent gradient, pinned by central
finite differences, and host-side validation of rtg_splat_backward_pose and rtg_pose_adam_step.

The pose is W2C (world to camera); the rasterizer reads viewmatrix = W2C^T, projmatrix = viewmatrix @ projection and
campos = -R^T t. A left twist xi = (rho, phi) moves it to exp(xi^) W2C. `tangent_grad` turns the three camera gradients
of the rasterizer into dL/dxi at xi = 0; the GPU test holds the kernel to it."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from rtg_slam_b200 import scene


def hat(xi):
    """4x4 matrix of the twist xi = (rho, phi): [[phi]x, rho], [0, 0]]."""
    rho, phi = xi[:3], xi[3:]
    m = torch.zeros((4, 4), dtype=xi.dtype)
    m[0, 1], m[0, 2], m[1, 2] = -phi[2], phi[1], -phi[0]
    m[1, 0], m[2, 0], m[2, 1] = phi[2], -phi[1], phi[0]
    m[:3, 3] = rho
    return m


def camera_arrays(w2c, projection):
    """(viewmatrix, projmatrix, campos) the rasterizer reads for the pose W2C."""
    view = w2c.t()
    return view, view @ projection, -(w2c[:3, :3].t() @ w2c[:3, 3])


def tangent_grad(d_view, d_proj, d_campos, w2c, projection):
    """dL/dxi at xi = 0 for W2C(xi) = exp(xi^) W2C, from dL/dviewmatrix, dL/dprojmatrix, dL/dcampos (float64 torch):
    G = dL/dW2C through the three arrays, A = G W2C^T, dL/drho_k = A[k][3], dL/dphi = (A21 - A12, A02 - A20, A10 - A01)."""
    G = d_view.t() + projection @ d_proj.t()
    R, t = w2c[:3, :3], w2c[:3, 3]
    G = G.clone()
    G[:3, :3] -= torch.outer(t, d_campos)
    G[:3, 3] -= R @ d_campos
    A = G @ w2c.t()
    return torch.stack([A[0, 3], A[1, 3], A[2, 3], A[2, 1] - A[1, 2], A[0, 2] - A[2, 0], A[1, 0] - A[0, 1]])


def rot(axis, deg):
    a = torch.tensor(axis, dtype=torch.float64)
    a = a / a.norm()
    return torch.matrix_exp(hat(torch.cat([torch.zeros(3, dtype=torch.float64), a * math.radians(deg)]))[:3, :3])


def pose(axis, deg, t):
    T = torch.eye(4, dtype=torch.float64)
    T[:3, :3] = rot(axis, deg)
    T[:3, 3] = torch.tensor(t, dtype=torch.float64)
    return T


POSES = {
    "identity": torch.eye(4, dtype=torch.float64),
    "small": torch.from_numpy(np.linalg.inv(scene.small_pose())),
    "rotated": pose((0.3, -1.0, 0.4), 35.0, (0.4, -1.2, 2.5)),
    "half_turn": pose((1.0, 0.2, -0.5), 150.0, (-3.0, 0.7, 1.1)),
}


def smooth_loss(view, proj, campos, seed=3):
    """A smooth nonlinear function of all 35 camera floats, standing in for the render loss."""
    g = torch.Generator().manual_seed(seed)
    wv, wp, wc = (torch.randn(s, generator=g, dtype=torch.float64) for s in ((4, 4), (4, 4), (3,)))
    return (torch.sin(view * wv).sum() + (proj * wp).sum() + 0.3 * ((proj * wp) ** 2).sum() + torch.cos(campos * wc).sum()
            + 0.2 * (campos ** 2).sum())


@pytest.mark.parametrize("name", list(POSES))
def test_tangent_gradient_matches_finite_differences(name):
    w2c = POSES[name]
    projection = torch.from_numpy(scene.make_camera("small").projection.astype(np.float64))
    arrays = [a.clone().requires_grad_(True) for a in camera_arrays(w2c, projection)]
    smooth_loss(*arrays).backward()
    g = tangent_grad(*(a.grad for a in arrays), w2c, projection)

    def L(xi):
        return float(smooth_loss(*camera_arrays(torch.matrix_exp(hat(xi)) @ w2c, projection)))
    scale = float(g.abs().max())
    assert scale > 1e-2
    for k in range(6):
        fd = []
        for h in (1e-5, 2.5e-6):
            e = torch.zeros(6, dtype=torch.float64)
            e[k] = h
            fd.append((L(e) - L(-e)) / (2 * h))
        assert abs(fd[0] - fd[1]) <= 1e-8 * scale, (name, k, fd)   # both steps agree: the difference quotient has converged
        assert abs(fd[1] - float(g[k])) <= 1e-8 * scale, (name, k, fd[1], float(g[k]))


def test_tangent_gradient_of_a_pure_view_loss_is_the_left_jacobian():
    """L = <U, W2C>: dL/dxi = the left-invariant pairing of U with xi^ W2C, checked entry by entry at a rotated pose."""
    w2c = POSES["rotated"]
    U = torch.randn((4, 4), generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    z = torch.zeros((4, 4), dtype=torch.float64)
    g = tangent_grad(U.t(), z, torch.zeros(3, dtype=torch.float64), w2c, torch.eye(4, dtype=torch.float64))
    for k in range(6):
        e = torch.zeros(6, dtype=torch.float64)
        e[k] = 1.0
        assert abs(float((U * (hat(e) @ w2c)).sum()) - float(g[k])) <= 1e-12 * float(U.abs().sum() * w2c.abs().max())


# ------------------------------------------------------------------------------------------------- host-side validation
def test_backward_pose_validates_before_touching_cuda():
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    nul = [None]
    # view, P, M, 6 inputs, radii, 3 workspaces, R_cap, counters, final_T, hit_image, dL_dcolor, dL_ddepth, dL_dT, scratch,
    # dL_dcamera, camera_scratch, stream
    tail = lambda P, dcam, scratch, dT=None: (P, 16, *(nul * 6), *(nul * 4), 0, *(nul * 5), dT, None, dcam, scratch, None)
    ok = C.c_void_p(256)
    assert L.rtg_splat_backward_pose(None, *tail(1, ok, ok)) == -1
    assert b"view is NULL" in L.rtg_last_error()
    view = _lib.RtgSplatView()
    view.image_height, view.image_width, view.sh_degree = 48, 64, 3
    view.viewmatrix = view.projmatrix = view.campos = view.bg = 256  # never dereferenced: validation fails first
    assert L.rtg_splat_backward_pose(C.byref(view), *tail(-1, ok, ok)) == -1
    assert b"P < 0" in L.rtg_last_error()
    assert L.rtg_splat_backward_pose(C.byref(view), *tail(1, None, ok)) == -1
    assert b"dL_dcamera / camera_scratch is NULL" in L.rtg_last_error()
    assert L.rtg_splat_backward_pose(C.byref(view), *tail(1, ok, None)) == -1
    assert b"dL_dcamera / camera_scratch is NULL" in L.rtg_last_error()
    assert L.rtg_splat_backward_pose(C.byref(view), *tail(1, ok, C.c_void_p(260))) == -1
    assert b"8-byte aligned" in L.rtg_last_error()
    assert L.rtg_splat_backward_pose(C.byref(view), *tail(1, ok, ok, dT=C.c_void_p(258))) == -1
    assert b"dL_dT must be 4-byte aligned" in L.rtg_last_error()
    assert L.rtg_splat_backward_pose(C.byref(view), *tail(1, ok, ok)) == -1   # P > 0 without the forward's buffers
    assert b"NULL pointer" in L.rtg_last_error()


def test_pose_adam_step_validates_before_touching_cuda():
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    assert L.rtg_pose_adam_step(None, None) == -1
    assert b"state is NULL" in L.rtg_last_error()

    def state(**over):
        s = _lib.RtgPoseAdam()
        for k in ("pose", "exp_avg", "exp_avg_sq", "projection", "viewmatrix", "projmatrix", "campos"):
            setattr(s, k, 256)
        s.lr_trans, s.lr_rot, s.beta1, s.beta2, s.eps, s.step = 1e-3, 1e-3, 0.9, 0.999, 1e-8, 1
        for k, v in over.items():
            setattr(s, k, v)
        return s
    for k in ("pose", "exp_avg", "exp_avg_sq"):
        assert L.rtg_pose_adam_step(C.byref(state(**{k: None})), None) == -1, k
        assert b"NULL pose / exp_avg / exp_avg_sq" in L.rtg_last_error()
    for k in ("projection", "viewmatrix", "projmatrix", "campos"):
        assert L.rtg_pose_adam_step(C.byref(state(**{k: None})), None) == -1, k
        assert b"NULL projection / viewmatrix / projmatrix / campos" in L.rtg_last_error()
    assert L.rtg_pose_adam_step(C.byref(state(pose=260)), None) == -1
    assert b"8-byte aligned" in L.rtg_last_error()
    for step in (0, -3):
        assert L.rtg_pose_adam_step(C.byref(state(step=step)), None) == -1
        assert b"step must be >= 1" in L.rtg_last_error()
