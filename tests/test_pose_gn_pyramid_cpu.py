"""CPU tests of coarse-to-fine, robust Gauss-Newton tracking: a float64 statement of the Huber-weighted step (reused by the
GPU tests), pinned against autograd and, below the threshold, against the squared-residual statement; the level camera of
tracking.level_camera on every scene camera; a numpy statement of rtg_frame_downsample (imported by the GPU test); host
validation of rtg_frame_downsample and rtg_splat_pose_gn_step_robust; the RtgPoseRobust layout."""
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

from rtg_slam_b200 import scene
from test_pose_gn_cpu import gn_step, normal_equations, random_problem
from test_pose_refine_cpu import POSES


# ------------------------------------------------------------------------------------------ the Huber step statement
def huber(r, delta):
    """rho(r): r^2 / 2 for |r| <= delta, delta |r| - delta^2 / 2 otherwise."""
    a = r.abs()
    return torch.where(a <= delta, 0.5 * r * r, delta * a - 0.5 * delta * delta)


def huber_weight(r, delta):
    a = r.abs()
    return torch.where(a <= delta, torch.ones_like(r), delta / a)


def huber_normal_equations(Jc, rc, sel_c, Jd, rd, sel_d, color_weight, depth_weight, color_delta, depth_delta):
    """H (6,6), g (6), (E, E_colour, E_depth), N_c, N_d of E = w_c/N_c sum_{S_c} sum_ch rho(r) + w_d/N_d sum_{S_d} rho(r)
    by iteratively reweighted least squares: w = 1 or delta / |r| per residual, H = sum w J^T J, g = sum w J^T r.
    Shapes as in test_pose_gn_cpu.normal_equations. Float64."""
    nc, nd = 3.0 * float(sel_c.sum()), float(sel_d.sum())
    wc = color_weight / nc if nc > 0 else 0.0
    wd = depth_weight / nd if nd > 0 else 0.0
    Jc, rc = Jc[..., sel_c], rc[:, sel_c]
    Jd, rd = Jd[:, sel_d], rd[sel_d]
    uc, ud = huber_weight(rc, color_delta), huber_weight(rd, depth_delta)
    H = wc * torch.einsum("acn,bcn,cn->ab", Jc, Jc, uc) + wd * (Jd * ud) @ Jd.t()
    g = wc * torch.einsum("acn,cn->a", Jc, uc * rc) + wd * Jd @ (ud * rd)
    ec, ed = wc * float(huber(rc, color_delta).sum()), wd * float(huber(rd, depth_delta).sum())
    return H, g, (ec + ed, ec, ed), nc, nd


@pytest.mark.parametrize("seed", [3, 5])
def test_huber_gradient_is_the_autograd_gradient(seed):
    """g is the gradient of sum rho(r + J xi) at xi = 0, with thresholds that down-weight part of both residual sets."""
    Jc, rc, sel_c, Jd, rd, sel_d = random_problem(seed)
    dc = float(rc[:, sel_c].abs().quantile(0.7))
    dd = float(rd[sel_d].abs().quantile(0.7))
    H, g, (E, ec, ed), nc, nd = huber_normal_equations(Jc, rc, sel_c, Jd, rd, sel_d, 0.8, 1.0, dc, dd)
    xi0 = torch.zeros(6, dtype=torch.float64, requires_grad=True)
    rcl = rc[:, sel_c] + torch.einsum("a,acn->cn", xi0, Jc[..., sel_c])
    rdl = rd[sel_d] + xi0 @ Jd[:, sel_d]
    El = 0.8 / nc * huber(rcl, dc).sum() + 1.0 / nd * huber(rdl, dd).sum()
    (gl,) = torch.autograd.grad(El, xi0)
    assert abs(float(El.detach()) - E) <= 1e-12 * abs(E) and abs(ec + ed - E) <= 1e-15 * abs(E)
    assert float((gl - g).abs().max()) <= 1e-12 * float(g.abs().max())
    # both branches ran, and H is symmetric positive definite
    assert 0.2 < float((rc[:, sel_c].abs() > dc).double().mean()) < 0.4 and 0.2 < float((rd[sel_d].abs() > dd).double().mean()) < 0.4
    assert torch.allclose(H, H.t()) and float(torch.linalg.eigvalsh(H).min()) > 0


def test_huber_statement_reduces_to_least_squares_below_the_threshold():
    """With delta >= max |r| the Huber H, g and E are those of test_pose_gn_cpu.normal_equations, and so is the step."""
    Jc, rc, sel_c, Jd, rd, sel_d = random_problem(4)
    big_c, big_d = float(rc.abs().max()), float(rd.abs().max())
    Hh, gh, Eh, nch, ndh = huber_normal_equations(Jc, rc, sel_c, Jd, rd, sel_d, 0.8, 1.0, big_c, big_d)
    H, g, E, nc, nd = normal_equations(Jc, rc, sel_c, Jd, rd, sel_d, 0.8, 1.0)
    assert (nch, ndh) == (nc, nd)
    assert float((Hh - H).abs().max()) <= 1e-12 * float(H.abs().max())
    assert float((gh - g).abs().max()) <= 1e-12 * float(g.abs().max())
    for a, b in zip(Eh, E):
        assert abs(a - b) <= 1e-12 * abs(b)
    w2c = POSES["rotated"]
    (new_h, xi_h), (new, xi) = gn_step(Hh, gh, 1e-4, w2c), gn_step(H, g, 1e-4, w2c)
    assert float((xi_h - xi).abs().max()) <= 1e-12 * float(xi.abs().max())
    assert float((new_h - new).abs().max()) <= 1e-12


# ------------------------------------------------------------------------------------------------------ level camera
def camera_like(cam):
    """The reference-Camera-like object PoseRefiner reads, at the scene camera's pose (float64 torch)."""
    w2c = torch.from_numpy(np.linalg.inv(cam.c2w))
    return types.SimpleNamespace(FoVx=2 * math.atan(cam.tanfovx), FoVy=2 * math.atan(cam.tanfovy), image_height=cam.height,
                                 image_width=cam.width, world_view_transform=w2c.t().contiguous(),
                                 projection_matrix=torch.from_numpy(np.ascontiguousarray(cam.projection)), cx=cam.cx, cy=cam.cy)


def project(camera, Xw):
    """Pixel of world points Xw (n, 3) through projmatrix = viewmatrix @ projection (row-vector storage) and
    ndc * S / 2 + c, as the rasterizer's preprocess maps them. Float64."""
    full = camera.world_view_transform.double() @ camera.projection_matrix.double()
    ph = torch.cat([Xw, torch.ones_like(Xw[:, :1])], 1) @ full
    ndc = ph[:, :2] / ph[:, 3:]
    return torch.stack([ndc[:, 0] * camera.image_width / 2 + camera.cx, ndc[:, 1] * camera.image_height / 2 + camera.cy], 1)


def pixel_ray(px, py, camera):
    """common.cuh pixel_ray with the focal lengths the rasterizer derives from the field of view (fx = W / (2 tanfovx))."""
    fx = camera.image_width / (2 * math.tan(camera.FoVx / 2))
    fy = camera.image_height / (2 * math.tan(camera.FoVy / 2))
    r = torch.stack([(px - camera.cx) / fx, (py - camera.cy) / fy, torch.ones_like(px)], 1)
    return r / r.norm(dim=1, keepdim=True)


@pytest.mark.parametrize("name", sorted(scene.CAMERAS))
@pytest.mark.parametrize("s", [2, 4])
def test_level_camera_looks_along_the_fine_block_centres(name, s):
    from rtg_slam_b200.tracking import level_camera
    cam = scene.make_camera(name, c2w=scene.small_pose())
    fine = camera_like(cam)
    coarse = level_camera(fine, s)
    W, H = cam.width, cam.height
    Ws, Hs = W // s, H // s
    assert (coarse.image_width, coarse.image_height) == (Ws, Hs)
    # every coarse pixel of a sparse grid including the borders
    ii, jj = torch.meshgrid(torch.unique(torch.linspace(0, Ws - 1, 9).round()).double(),
                            torch.unique(torch.linspace(0, Hs - 1, 7).round()).double(), indexing="xy")
    i, j = ii.reshape(-1), jj.reshape(-1)
    u, v = s * i + (s - 1) / 2, s * j + (s - 1) / 2                        # the fine block centres
    # world points on the fine block-centre rays (depths 0.5 .. 4), built through the fine projection
    z = torch.linspace(0.5, 4.0, i.numel(), dtype=torch.float64)
    Pm = fine.projection_matrix.double()
    xc = torch.stack([(u - cam.cx) * 2 / W * z / Pm[0, 0], (v - cam.cy) * 2 / H * z / Pm[1, 1], z], 1)
    c2w = torch.from_numpy(cam.c2w)
    Xw = xc @ c2w[:3, :3].t() + c2w[:3, 3]
    assert float((project(fine, Xw) - torch.stack([u, v], 1)).abs().max()) <= 1e-9
    got = project(coarse, Xw)
    assert float((got - torch.stack([i, j], 1)).abs().max()) <= 1e-6, (got, i, j)
    # the coarse pixel ray is the fine block-centre ray
    assert float((pixel_ray(i, j, coarse) - pixel_ray(u, v, fine)).abs().max()) <= 1e-12
    # the intrinsics of the statement: fx / s, and the field of view unchanged when s divides the size
    assert abs(Ws / (2 * math.tan(coarse.FoVx / 2)) - cam.fx / s) <= 1e-9 * cam.fx
    assert abs(Hs / (2 * math.tan(coarse.FoVy / 2)) - cam.fy / s) <= 1e-9 * cam.fy
    if W % s == 0:
        assert abs(math.tan(coarse.FoVx / 2) - cam.tanfovx) <= 1e-15
    assert torch.equal(coarse.projection_matrix[2:], fine.projection_matrix.double()[2:])
    assert torch.equal(coarse.world_view_transform, fine.world_view_transform)


def test_level_camera_rejects_an_empty_level():
    from rtg_slam_b200.tracking import level_camera
    fine = camera_like(scene.make_camera("tiny"))
    for s in (0, 49):
        with pytest.raises(ValueError):
            level_camera(fine, s)


# ------------------------------------------------------------------------------------------ the downsampling statement
def downsample_statement(color, depth, s, render_mask=None, tile_mask=None, channels_last=False):
    """rtg_frame_downsample in numpy: float32 sums over each s x s block in row order (as the kernel adds them), divided
    by s^2. color (3, H, W) or (H, W, 3) with channels_last; returns (color (3, Hs, Ws), depth, mask or None, tile mask or
    None)."""
    color = np.asarray(color, dtype=np.float32)
    if channels_last:
        color = np.ascontiguousarray(color.transpose(2, 0, 1))
    depth = np.asarray(depth, dtype=np.float32)
    H, W = depth.shape
    Hs, Ws = H // s, W // s
    n = np.float32(s * s)
    c_acc = np.zeros((3, Hs, Ws), np.float32)
    d_acc = np.zeros((Hs, Ws), np.float32)
    d_ok = np.ones((Hs, Ws), bool)
    m_ok = np.ones((Hs, Ws), bool)
    for dy in range(s):
        for dx in range(s):
            blk = (slice(dy, dy + s * Hs, s), slice(dx, dx + s * Ws, s))
            c_acc += color[(slice(None),) + blk]
            d_acc += depth[blk]
            d_ok &= depth[blk] > 0
            if render_mask is not None:
                m_ok &= np.asarray(render_mask)[blk] != 0
    mask = m_ok.astype(np.uint8) if render_mask is not None else None
    tm = None
    if tile_mask is not None:
        tile_mask = np.asarray(tile_mask)
        fty, ftx = tile_mask.shape
        cty, ctx = (Hs + 15) // 16, (Ws + 15) // 16
        tm = np.zeros((cty, ctx), np.int32)
        for ty in range(cty):
            for tx in range(ctx):
                tm[ty, tx] = int(tile_mask[s * ty:min(s * ty + s, fty), s * tx:min(s * tx + s, ftx)].any())
    return c_acc / n, np.where(d_ok, d_acc / n, np.float32(0)).astype(np.float32), mask, tm


def test_downsample_statement_pools_as_documented():
    rng = np.random.default_rng(5)
    H, W, s = 37, 50, 4                                  # a trailing partial row and column
    color = rng.uniform(size=(3, H, W)).astype(np.float32)
    depth = rng.uniform(0.5, 3.0, size=(H, W)).astype(np.float32)
    depth[5, 9] = 0.0                                    # block (i, j) = (2, 1) loses its depth
    mask = np.ones((H, W), np.uint8)
    mask[30, 3] = 0                                      # block (0, 7) leaves the mask
    tiles = np.zeros((3, 4), np.int32)
    tiles[2, 3] = 1                                      # only the last fine tile
    c, d, m, t = downsample_statement(color, depth, s, mask, tiles)
    Hs, Ws = H // s, W // s
    assert c.shape == (3, Hs, Ws) and d.shape == m.shape == (Hs, Ws) and t.shape == (1, 1)
    blocks = color[:, :Hs * s, :Ws * s].reshape(3, Hs, s, Ws, s).astype(np.float64).mean(axis=(2, 4))
    assert np.abs(c - blocks).max() <= 1e-6
    assert d[1, 2] == 0 and (d > 0).sum() == Hs * Ws - 1
    assert m[7, 0] == 0 and m.sum() == Hs * Ws - 1
    assert t[0, 0] == 1                                  # fine tiles [0, 4) x [0, 4) clipped to the 3 x 4 grid
    c2, d2, _, _ = downsample_statement(color.transpose(1, 2, 0), depth, s, channels_last=True)
    assert np.array_equal(c, c2) and np.array_equal(d, d2)


# ------------------------------------------------------------------------------------------------- host validation
def test_robust_struct_layout():
    from rtg_slam_b200 import _lib
    assert C.sizeof(_lib.RtgPoseRobust) == 16
    assert (_lib.RtgPoseRobust.color_delta.offset, _lib.RtgPoseRobust.depth_delta.offset) == (4, 8)
    assert (_lib.RTG_ROBUST_NONE, _lib.RTG_ROBUST_HUBER) == (0, 1)


def test_frame_downsample_validates_before_touching_cuda():
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    ok = C.c_void_p(256)

    def call(color=ok, depth=ok, mask=None, tiles=None, H=48, W=64, s=2, cl=0, c_out=ok, d_out=ok, m_out=None, t_out=None):
        return L.rtg_frame_downsample(color, depth, mask, tiles, H, W, s, cl, c_out, d_out, m_out, t_out, None)
    for s in (1, 0, -2):
        assert call(s=s) == -1 and b"scale must be >= 2" in L.rtg_last_error(), s
    for kw in (dict(H=0), dict(W=-1), dict(H=3, s=4), dict(W=3, s=4)):
        assert call(**kw) == -1 and b"H and W must be >= scale" in L.rtg_last_error(), kw
    assert call(cl=2) == -1 and b"color_channels_last" in L.rtg_last_error()
    for k in ("color", "depth", "c_out", "d_out"):
        assert call(**{k: None}) == -1 and b"NULL pointer" in L.rtg_last_error(), k
    assert call(mask=ok) == -1 and b"mask_out must be given exactly when render_mask is" in L.rtg_last_error()
    assert call(m_out=ok) == -1 and b"mask_out must be given exactly when render_mask is" in L.rtg_last_error()
    assert call(tiles=ok) == -1 and b"tile_mask_out must be given exactly when tile_mask is" in L.rtg_last_error()
    assert call(t_out=ok) == -1 and b"tile_mask_out must be given exactly when tile_mask is" in L.rtg_last_error()


def test_pose_gn_step_robust_validates_before_touching_cuda():
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    ok = C.c_void_p(256)
    view = _lib.RtgSplatView()
    view.image_height, view.image_width, view.sh_degree = 48, 64, 3
    view.viewmatrix = view.projmatrix = view.campos = view.bg = 256  # never dereferenced: validation fails first
    s = _lib.RtgPoseGN()
    for k in ("pose", "projection", "viewmatrix", "projmatrix", "campos", "render", "depth", "hit_depth", "gt_color", "gt_depth",
              "scratch", "report"):
        setattr(s, k, 256)
    s.color_weight, s.depth_weight, s.depth_error_max, s.damping = 0.8, 1.0, 0.1, 1e-4

    def robust(kernel=1, dc=0.1, dd=0.05):
        r = _lib.RtgPoseRobust()
        r.kernel, r.color_delta, r.depth_delta = kernel, dc, dd
        return r

    def call(st=s, r=robust(), P=4):
        return L.rtg_splat_pose_gn_step_robust(C.byref(view), P, 16, ok, ok, None, ok, ok, None, ok, ok, ok, 1024, ok,
                                               None if st is None else C.byref(st), None if r is None else C.byref(r), None)
    assert call(st=None) == -1 and b"state is NULL" in L.rtg_last_error()
    assert call(r=None) == -1 and b"robust is NULL" in L.rtg_last_error()
    for k in (-1, 2, 7):
        assert call(r=robust(kernel=k)) == -1 and b"unknown robust kernel" in L.rtg_last_error(), k
    for dc, dd in ((0.0, 0.05), (-0.1, 0.05), (float("nan"), 0.05), (float("inf"), 0.05), (0.1, 0.0), (0.1, -1.0),
                   (0.1, float("nan")), (0.1, float("inf"))):
        assert call(r=robust(dc=dc, dd=dd)) == -1 and b"positive and finite" in L.rtg_last_error(), (dc, dd)
    # past the robust checks, the arguments of rtg_splat_pose_gn_step are validated as there; NONE ignores the deltas
    assert call(P=0) == -1 and b"P must be >= 1" in L.rtg_last_error()
    assert call(r=robust(kernel=0, dc=float("nan"), dd=-1.0), P=0) == -1 and b"P must be >= 1" in L.rtg_last_error()
    s.damping = -1.0
    assert call() == -1 and b"damping and weights must be >= 0" in L.rtg_last_error()
    assert b"rtg_splat_pose_gn_step_robust" in L.rtg_last_error()


def test_refine_gn_rejects_bad_pyramid_arguments():
    """The new keyword arguments are checked before anything is rendered."""
    from rtg_slam_b200.tracking import PoseRefiner
    ref = PoseRefiner.__new__(PoseRefiner)  # no renderer (it allocates on the GPU): the checks come first
    for kw in (dict(scales=(2,)), dict(scales=(2, 4, 1)), dict(scales=(2, 2, 1)), dict(scales=()),
               dict(scales=(4, 2, 1), iters=(3, 3)), dict(iters=0), dict(scales=(2, 1), iters=(3, 0)), dict(robust="cauchy")):
        kw.setdefault("iters", 3)
        with pytest.raises(ValueError):
            ref.refine_gn(None, None, None, None, **kw)
