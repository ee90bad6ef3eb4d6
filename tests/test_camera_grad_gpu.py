"""GPU tests of the camera gradient: dL/d(viewmatrix, projmatrix, campos) from the rasterizer backward
(rtg_splat_backward_camera through GaussianRasterizer and Renderer.render).

Metric: per block (viewmatrix, projmatrix, campos) max|g - g_ref| / max|g_ref| against the float64 oracle, below
max(1e-3, 10 x the library's own run-to-run difference). The compositing backward accumulates the gradient records with
float atomics in a varying order, and the camera gradient sums the terms of every visible Gaussian, so two runs on the
same inputs differ in the last bits; 1e-3 is the per-Gaussian gradients' oracle tolerance (test_raster_gpu.py) and the
run-to-run term covers scenes (translucent blobs) where that jitter is larger."""
import math
import types

import numpy as np
import pytest
import torch

import helpers
from oracle.camera_oracle import camera_gradient
from oracle.splat_oracle import OracleRender
from rtg_slam_b200 import scene

pytestmark = pytest.mark.gpu
NAMES = ("color", "depth", "hit_color", "hit_depth", "hit_color_weight", "hit_depth_weight", "T_map", "radii")
CAM = ("viewmatrix", "projmatrix", "campos")
KW = {"xyz": "means3D", "opacity": "opacities", "shs": "shs", "colors_precomp": "colors_precomp", "scales": "scales",
      "rotations": "rotations", "cov3D_precomp": "cov3D_precomp"}


def cov3d_f32(scales, rotations, mod=1.0):
    r, x, y, z = rotations.astype(np.float64).T
    R = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
                  np.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
                  np.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], 1)
    Ms = R * (mod * scales.astype(np.float64))[:, None, :]
    S = Ms @ Ms.transpose(0, 2, 1)
    return np.ascontiguousarray(S[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].astype(np.float32))


def scene_case(name):
    """The scenes of test_raster_inputs_gpu.py: surfel room, ragged image size, 50 % tile mask, dense blobs whose tile
    lists exceed 4096 entries (chunked-merge sort)."""
    if name == "small":
        return scene.make_camera("small"), scene.surfel_room(3000, seed=41), None
    if name == "ragged":
        return scene.make_camera("ragged"), scene.random_blobs(1500, seed=42), None
    if name == "masked":
        cam = scene.make_camera("small", c2w=scene.small_pose())
        return cam, scene.surfel_room(3000, seed=43), scene.random_tile_mask(cam, 0.5, seed=143)
    assert name == "dense"
    return scene.make_camera("tiny"), scene.dense_blobs(30_000, seed=44), None


def inputs_for(g, mode):
    base = {k: g[k] for k in ("xyz", "opacity")}
    if mode == "colors_precomp":
        cols = np.random.default_rng(46).uniform(-0.25, 1.25, (len(g["xyz"]), 3)).astype(np.float32)
        return dict(base, scales=g["scales"], rotations=g["rotations"], colors_precomp=cols), {}
    if mode == "cov3D_precomp":
        return dict(base, shs=g["shs"], cov3D_precomp=cov3d_f32(g["scales"], g["rotations"])), {}
    if mode == "M4":
        return dict(base, scales=g["scales"], rotations=g["rotations"], shs=np.ascontiguousarray(g["shs"][:, :4])), {"sh_degree": 1}
    if mode == "modifier":
        return dict(base, scales=g["scales"], rotations=g["rotations"], shs=g["shs"]), {"scale_modifier": 1.7}
    return dict(base, scales=g["scales"], rotations=g["rotations"], shs=g["shs"]), {}


def render(cam, inputs, dev, up, mask=None, camera=CAM, **over):
    """GaussianRasterizer forward + backward of sum(dL/dcolor * color) + sum(dL/ddepth * depth); the settings tensors
    named in `camera` require grad."""
    from rtg_slam_b200.rasterizer import GaussianRasterizer
    rs = helpers.make_settings(cam, dev, **over)
    for k in camera:
        getattr(rs, k).requires_grad_(True)
    leaves = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev).requires_grad_(True) for k, v in inputs.items()}
    tm = None if mask is None else torch.from_numpy(np.ascontiguousarray(mask, dtype=np.int32)).to(dev)
    out = GaussianRasterizer(rs)(**{KW[k]: v for k, v in leaves.items()}, tile_mask=tm)
    res = dict(zip(NAMES, [o.detach().cpu().numpy() for o in out]))
    gc, gd = (torch.from_numpy(x).to(dev) for x in up)
    ((out[0] * gc).sum() + (out[1] * gd).sum()).backward()
    res["grads"] = {KW[k]: v.grad.cpu().numpy() for k, v in leaves.items()}
    res["camera"] = {k: (None if getattr(rs, k).grad is None else getattr(rs, k).grad.cpu().numpy()) for k in CAM}
    return res


def oracle64(cam, inputs, up, mask=None, **over):
    g = {k: (None if inputs.get(k) is None else inputs[k].astype(np.float64)) for k in ("xyz", "opacity", "shs", "scales", "rotations")}
    cp, cv = inputs.get("colors_precomp"), inputs.get("cov3D_precomp")
    o = OracleRender(cam, g, tile_mask=mask, precision="f64", colors_precomp=None if cp is None else cp.astype(np.float64),
                     cov3D_precomp=None if cv is None else cv.astype(np.float64), **over)
    return camera_gradient(o, up[0].astype(np.float64), up[1].astype(np.float64))


CONFIGS = [("small", "sh"), ("ragged", "sh"), ("masked", "sh"), ("dense", "sh"), ("small", "colors_precomp"),
           ("ragged", "cov3D_precomp"), ("masked", "M4"), ("small", "modifier"), ("small", "visible_rows_only")]


@pytest.mark.parametrize("name,mode", CONFIGS)
def test_camera_gradient_matches_f64_oracle(cuda_device, name, mode):
    from rtg_slam_b200.rasterizer import visible_rows_only
    cam, g, mask = scene_case(name)
    inputs, over = inputs_for(g, mode)
    up = scene.upstream_grads(cam, seed=5)
    with visible_rows_only(mode == "visible_rows_only"):
        a = render(cam, inputs, cuda_device, up, mask, **over)
        b = render(cam, inputs, cuda_device, up, mask, **over)
    ref = oracle64(cam, inputs, up, mask, **over)
    assert np.all(a["camera"]["viewmatrix"].reshape(-1)[[3, 7, 11, 15]] == 0)
    for k in CAM:
        if mode == "colors_precomp" and k == "campos":
            assert np.all(a["camera"][k] == 0) and np.all(ref[k] == 0)
            continue
        assert np.abs(ref[k]).max() > 0, k
        jitter = helpers.rel_err(b["camera"][k], a["camera"][k])
        err = helpers.rel_err(a["camera"][k], ref[k])
        print(f"{name}/{mode} d{k}: rel err vs f64 oracle {err:.2e}, run-to-run {jitter:.2e}")
        assert err < max(1e-3, 10 * jitter), (name, mode, k, err, jitter)


def test_camera_gradients_change_nothing_else(cuda_device):
    """Forward bit-identical with camera gradients on and off; the per-Gaussian gradients agree within the run-to-run
    tolerance; a settings tensor that does not require grad gets None."""
    cam, g, mask = scene_case("masked")
    inputs, _ = inputs_for(g, "sh")
    up = scene.upstream_grads(cam, seed=6)
    off = render(cam, inputs, cuda_device, up, mask, camera=())
    off2 = render(cam, inputs, cuda_device, up, mask, camera=())
    on = render(cam, inputs, cuda_device, up, mask)
    for k in NAMES:
        assert np.array_equal(on[k], off[k]), k
    for k in off["grads"]:
        tol = max(1e-5, 10 * helpers.rel_err(off2["grads"][k], off["grads"][k]))
        assert helpers.rel_err(on["grads"][k], off["grads"][k]) < tol, k
    assert all(v is None for v in off["camera"].values())
    only_view = render(cam, inputs, cuda_device, up, mask, camera=("viewmatrix",))
    assert only_view["camera"]["projmatrix"] is None and only_view["camera"]["campos"] is None
    assert helpers.rel_err(only_view["camera"]["viewmatrix"], on["camera"]["viewmatrix"]) < 1e-3


# ---------------------------------------------------------------------------------------------------- invariances
def skew(w):
    z = torch.zeros((), dtype=w.dtype, device=w.device)
    return torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]), torch.stack([-w[1], w[0], z])])


def quat_mul(a, b):
    """Hamilton product of (w, x, y, z) quaternions, broadcast over rows."""
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return torch.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], -1)


def invariance(cam, g, dev, rotation, colors=None):
    """Moves the map and the camera together by a translation (or, `rotation`, a rotation about the origin) and returns
    (sum of the map's and the camera's dL/d(motion), sum of their magnitudes). Every Gaussian gets its own motion
    parameter, so the magnitudes are per Gaussian. The loss cannot change, so the sum must vanish."""
    from rtg_slam_b200.rasterizer import GaussianRasterizer
    t = {k: torch.from_numpy(v).to(dev) for k, v in g.items()}
    P = t["xyz"].shape[0]
    vm = torch.from_numpy(cam.viewmatrix).to(dev)
    proj = torch.from_numpy(np.ascontiguousarray(cam.projection)).to(dev)
    cp = torch.from_numpy(cam.campos).to(dev)
    m_par = torch.zeros((P, 3), device=dev, requires_grad=True)
    c_par = torch.zeros(3, device=dev, requires_grad=True)
    q_par = torch.zeros((P, 3), device=dev, requires_grad=True)
    rots = t["rotations"]
    if rotation:  # R = I + [w]x to first order; the gradient is taken at w = 0
        means = t["xyz"] + torch.cross(m_par, t["xyz"], dim=1)
        one = torch.ones((P, 1), device=dev)
        rots = quat_mul(torch.cat([one, 0.5 * q_par], 1), rots)
        Rc = torch.matrix_exp(skew(c_par))
        vm2 = torch.cat([Rc @ vm[:3], vm[3:]], 0)
        cp2 = Rc @ cp
    else:
        means = t["xyz"] + m_par
        shift = torch.cat([c_par @ vm[:3, :3], torch.zeros(1, device=dev)])
        vm2 = torch.cat([vm[:3], vm[3:] - shift[None]], 0)
        cp2 = cp + c_par
    rs = helpers.make_settings(cam, dev)._replace(viewmatrix=vm2, projmatrix=vm2 @ proj, campos=cp2)
    kw = dict(means3D=means, opacities=t["opacity"], scales=t["scales"], rotations=rots)
    if colors is not None:
        kw["colors_precomp"] = torch.from_numpy(colors).to(dev)
    else:
        kw["shs"] = t["shs"]
    out = GaussianRasterizer(rs)(**kw)
    # positive pixel weights: a coherent loss whose camera term is not itself the residue of a random-sign sum
    gen = torch.Generator(device=dev).manual_seed(9)
    N = cam.width * cam.height
    wc = torch.rand((3, cam.height, cam.width), device=dev, generator=gen) / N + 0.5 / N
    wd = torch.rand((1, cam.height, cam.width), device=dev, generator=gen) / N + 0.5 / N
    loss = (out[0] * wc).sum() + (out[1] * wd).sum()
    pars = [m_par, c_par] + ([q_par] if rotation else [])
    grads = torch.autograd.grad(loss, pars)
    total = sum(gr.double().reshape(-1, 3).sum(0) for gr in grads)
    mag = sum(gr.double().abs().reshape(-1, 3).sum(0) for gr in grads)
    cam_share = grads[1].double().abs()
    total, mag, cam_share = total.cpu().numpy(), mag.cpu().numpy(), cam_share.cpu().numpy()
    print(f"{'rotation' if rotation else 'translation'} {cam.width}x{cam.height}: residue / magnitudes "
          f"{np.abs(total) / mag}, camera share {cam_share / mag}")
    return total, mag, cam_share


@pytest.fixture(scope="module")
def room_1m():
    return scene.surfel_room(1_000_000, seed=2024)


# Each per-Gaussian term carries a float32 rounding error of about 1e-7 of its size and the errors do not add up
# coherently: the residue measured on an H100 is <= 1e-8 of the summed magnitudes at both sizes, both motions. 1e-6 leaves
# a margin of 100. A missing or mis-signed term leaves a residue of the size of the camera term, which is >= 1.4e-3 of
# the magnitudes here and must stay far above the bound for the check to mean anything.
INVARIANCE_TOL = 1e-6


@pytest.mark.parametrize("cam_name", ["replica", "hd"])
def test_translation_invariance_at_timed_sizes(cuda_device, room_1m, cam_name):
    cam = scene.make_camera(cam_name, c2w=scene.small_pose())
    total, mag, cam_share = invariance(cam, room_1m, cuda_device, rotation=False)
    assert np.all(cam_share > 20 * INVARIANCE_TOL * mag), (cam_share, mag)
    assert np.all(np.abs(total) <= INVARIANCE_TOL * mag), (total, mag)


@pytest.mark.parametrize("cam_name", ["replica", "hd"])
def test_rotation_invariance_at_timed_sizes(cuda_device, room_1m, cam_name):
    """With precomputed colours: an SH colour depends on the world-space view direction, which a rotation changes."""
    cam = scene.make_camera(cam_name, c2w=scene.small_pose())
    cols = np.random.default_rng(8).uniform(0, 1, (len(room_1m["xyz"]), 3)).astype(np.float32)
    total, mag, cam_share = invariance(cam, room_1m, cuda_device, rotation=True, colors=cols)
    assert np.all(cam_share > 20 * INVARIANCE_TOL * mag), (cam_share, mag)
    assert np.all(np.abs(total) <= INVARIANCE_TOL * mag), (total, mag)


# ---------------------------------------------------------------------------------------------------- pose refinement
def se3_exp(xi):
    """4x4 exp of the twist xi = (rho, phi) (translation, rotation), built with torch ops."""
    m = torch.zeros((4, 4), dtype=xi.dtype, device=xi.device)
    m = m + torch.nn.functional.pad(skew(xi[3:]), (0, 1, 0, 1)) + torch.nn.functional.pad(xi[:3, None], (3, 0, 0, 1))
    return torch.matrix_exp(m)


def view_camera(cam, w2c):
    """The camera object Renderer.render reads, from a (differentiable) world-to-camera pose."""
    vm = w2c.transpose(0, 1)
    proj = torch.from_numpy(np.ascontiguousarray(cam.projection)).to(w2c.device)
    return types.SimpleNamespace(FoVx=2 * math.atan(cam.tanfovx), FoVy=2 * math.atan(cam.tanfovy), image_height=cam.height,
                                 image_width=cam.width, world_view_transform=vm, full_proj_transform=vm @ proj,
                                 camera_center=torch.linalg.inv(w2c)[:3, 3], cx=cam.cx, cy=cam.cy)


def pose_error(w2c, w2c_true):
    d = (w2c @ torch.linalg.inv(w2c_true)).double().cpu().numpy()
    ang = math.degrees(math.acos(max(-1.0, min(1.0, (np.trace(d[:3, :3]) - 1) / 2))))
    c, c_true = np.linalg.inv(w2c.double().cpu().numpy())[:3, 3], np.linalg.inv(w2c_true.double().cpu().numpy())[:3, 3]
    return ang, float(np.linalg.norm(c - c_true))


def test_pose_refinement_with_adam(cuda_device):
    """Render targets at a pose, start 1 deg / 2 cm away, minimise L1 colour + L1 depth over a twist xi of
    exp(xi) * W2C_start with torch.optim.Adam (150 steps, lr 1e-3). The photometric and depth residuals are smooth in the
    pose at this scale (the surfel room's patches fill the view), so both errors must fall to a tenth of their start."""
    from rtg_slam_b200.render import Renderer
    dev = cuda_device
    cam = scene.make_camera("small")
    g = {k: torch.from_numpy(v).to(dev) for k, v in scene.surfel_room(20_000, seed=7).items()}
    args = types.SimpleNamespace(renderer_opaque_threshold=0.6, renderer_normal_threshold=60, renderer_depth_threshold=1.0,
                                 max_sh_degree=3, color_sigma=3.0, active_sh_degree=3)
    r = Renderer(args)
    w2c_true = torch.from_numpy(np.linalg.inv(scene.small_pose()).astype(np.float32)).to(dev)
    with torch.no_grad():
        tgt = r.render(view_camera(cam, w2c_true), g)
        tgt_c, tgt_d = tgt["render"].clone(), tgt["depth"].clone()
    off = torch.tensor([0.012, -0.010, 0.012, 0.010, -0.012, 0.008], device=dev)  # 2 cm, 1.0 deg
    w2c0 = se3_exp(off) @ w2c_true
    ang0, tr0 = pose_error(w2c0, w2c_true)
    assert 0.8 < ang0 < 1.3 and 0.015 < tr0 < 0.025
    xi = torch.zeros(6, device=dev, requires_grad=True)
    opt = torch.optim.Adam([xi], lr=1e-3)
    valid = tgt_d > 0
    for _ in range(150):
        opt.zero_grad()
        out = r.render(view_camera(cam, se3_exp(xi) @ w2c0), g)
        loss = (out["render"] - tgt_c).abs().mean() + (out["depth"] - tgt_d).abs()[valid].mean()
        loss.backward()
        opt.step()
    with torch.no_grad():
        ang, tr = pose_error(se3_exp(xi) @ w2c0, w2c_true)
    print(f"pose refinement: rotation {ang0:.3f} -> {ang:.3f} deg, translation {100 * tr0:.2f} -> {100 * tr:.2f} cm")
    # measured on an H100: 1.006 -> 0.014..0.020 deg, 1.97 -> 0.01..0.03 cm; Adam's steps of ~lr leave a residual well inside 10 %
    assert ang < 0.1 * ang0 and tr < 0.1 * tr0, (ang0, ang, tr0, tr)


def test_camera_gradients_under_grad_record_hook_raise(cuda_device):
    from rtg_slam_b200.rasterizer import set_grad_record_hook
    cam, g, _ = scene_case("ragged")
    inputs, _ = inputs_for(g, "sh")
    prev = set_grad_record_hook(lambda rec: None)
    try:
        with pytest.raises(RuntimeError, match="camera gradients"):
            render(cam, inputs, cuda_device, scene.upstream_grads(cam, seed=5))
    finally:
        set_grad_record_hook(prev)
