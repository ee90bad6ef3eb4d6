"""GPU tests of pose refinement: the pose-only rasterizer backward (rtg_splat_backward_pose), its dispatch from the
autograd shim, the device pose step (rtg_pose_adam_step) and PoseRefiner.refine.

The pose-only camera gradient is held to the full camera backward on the SAME gradient records. The compositing backward
adds the records with float atomics in a varying order, so two backward calls never see identical records; instead the
records of one real backward are frozen and handed, copy by copy, to both per-Gaussian passes (each call then runs its
compositing backward with zero upstream gradients, which adds nothing). On identical records both reductions have a fixed
order: each path must reproduce itself bit for bit, and the two paths must agree to 1e-5 of each block's largest entry
(they evaluate the same 27 terms, compiled into different kernels)."""
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

import helpers
from rtg_slam_b200 import scene
from test_camera_grad_gpu import CAM, KW, inputs_for, pose_error, scene_case, se3_exp, view_camera
from test_pose_refine_cpu import hat, tangent_grad
from test_transmittance_grad_cpu import t_weights
from test_transmittance_grad_gpu import spy  # noqa: F401 -- fixture: records / replaces backward entry points

pytestmark = pytest.mark.gpu


def forward(cam, inputs, dev, up, mask=None, gaussian_grad=(), **over):
    """GaussianRasterizer forward with the three camera tensors requiring grad (and the named Gaussian inputs, if any);
    returns (settings, leaves, loss) with loss = <dL/dcolor, color> + <dL/ddepth, depth> [+ <dL/dT, T_map>]."""
    from rtg_slam_b200.rasterizer import GaussianRasterizer
    rs = helpers.make_settings(cam, dev, **over)
    for k in CAM:
        getattr(rs, k).requires_grad_(True)
    leaves = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev).requires_grad_(k in gaussian_grad) for k, v in inputs.items()}
    tm = None if mask is None else torch.from_numpy(np.ascontiguousarray(mask, dtype=np.int32)).to(dev)
    out = GaussianRasterizer(rs)(**{KW[k]: v for k, v in leaves.items()}, tile_mask=tm)
    terms = [(out[i] * torch.from_numpy(np.ascontiguousarray(u, dtype=np.float32)).to(dev)).sum()
             for i, u in zip((0, 1, 6), up) if u is not None]
    return rs, leaves, sum(terms)


def frozen_record_runs(dev, H, W, found):
    """A replacement for rtg_splat_backward_pose: fills the gradient records once with the call's real upstream, then runs
    the pose-only and the camera backward twice each (alternating) on copies of those records, with zero upstream
    gradients; stores the four dL_dcamera in `found`. Finally answers the autograd call itself."""
    from rtg_slam_b200 import _lib, rasterizer

    def run(L, *a):
        P, stream = a[1], a[23]
        p = lambda t: C.c_void_p(t.data_ptr())
        scratch = rasterizer._state(dev).scratch[:P * 16]
        outs = [torch.empty(P * 48 + 64, dtype=torch.float32, device=dev) for _ in range(8)]
        _lib.check(L.rtg_splat_backward_render_dt(0, P, *a[:19], a[19], a[20], *(p(o) for o in outs), stream),
                   "rtg_splat_backward_render_dt")
        records = scratch.clone()
        assert float(records.abs().max()) > 0
        zc, zd = torch.zeros((3, H, W), device=dev), torch.zeros((1, H, W), device=dev)
        head = a[:17] + (p(zc), p(zd))
        cam_scratch = torch.empty((int(L.rtg_splat_camera_scratch_bytes(P)),), dtype=torch.uint8, device=dev)
        for path in ("pose", "camera", "pose", "camera"):
            scratch.copy_(records)
            dcam = torch.full((35,), float("nan"), device=dev)
            if path == "pose":
                rc = L.rtg_splat_backward_pose(*head, None, a[20], p(dcam), p(cam_scratch), stream)
            else:
                rc = L.rtg_splat_backward_dt(*head, None, a[20], *(p(o) for o in outs), 0, p(dcam), p(cam_scratch), stream)
            _lib.check(rc, path)
            assert float(scratch.abs().max()) == 0.0, path   # the records are consumed and cleared
            found.setdefault(path, []).append(dcam.cpu().numpy())
        return L.rtg_splat_backward_pose(*a)
    return run


BLOCKS = {"viewmatrix": slice(0, 16), "projmatrix": slice(16, 32), "campos": slice(32, 35)}
CONFIGS = [("small", "sh"), ("ragged", "sh"), ("masked", "sh"), ("dense", "sh"), ("small", "colors_precomp"),
           ("ragged", "cov3D_precomp"), ("masked", "M4"), ("small", "modifier")]


@pytest.mark.parametrize("loss", ["colour_depth", "with_T"])
@pytest.mark.parametrize("name,mode", CONFIGS)
def test_pose_only_gradient_matches_the_camera_path(cuda_device, spy, name, mode, loss):
    from rtg_slam_b200 import rasterizer
    cam, g, mask = scene_case(name)
    inputs, over = inputs_for(g, mode)
    gc, gd = scene.upstream_grads(cam, seed=5)
    up = (gc, gd, t_weights(cam, seed=6).astype(np.float32) if loss == "with_T" else None)
    rs, _, total = forward(cam, inputs, cuda_device, up, mask, **over)
    found = {}
    s = spy({"rtg_splat_backward_pose": frozen_record_runs(cuda_device, cam.height, cam.width, found)})
    total.backward()
    assert s.calls == ["rtg_splat_backward_pose"]
    assert float(rasterizer._state(cuda_device).scratch.abs().max()) == 0.0
    (pose, pose2), (ref, ref2) = found["pose"], found["camera"]
    assert np.array_equal(pose, pose2), "pose-only backward: identical records must give a bit-identical dL_dcamera"
    assert np.array_equal(ref, ref2), "camera backward: identical records must give a bit-identical dL_dcamera"
    assert np.all(pose[[3, 7, 11, 15]] == 0) and np.all(pose[[18, 22, 26, 30]] == 0)
    for k, b in BLOCKS.items():
        if k == "campos" and mode == "colors_precomp":   # campos only enters the SH colour
            assert np.all(pose[b] == 0) and np.all(ref[b] == 0)
            continue
        scale = np.abs(ref[b]).max()
        assert scale > 0, k
        err = np.abs(pose[b] - ref[b]).max()
        print(f"{name}/{mode}/{loss} d{k}: pose-only vs camera path on identical records {err / scale:.2e}"
              f"{' (bit-identical)' if err == 0 else ''}")
        assert err <= 1e-5 * scale, (name, mode, loss, k, err / scale)


def test_entry_point_dispatch(cuda_device, spy):
    """Only the camera requires grad: rtg_splat_backward_pose, no Gaussian gradient, records left zero. Any Gaussian input
    requiring grad, grad_buffers or visible_rows_only: the entry point of before."""
    from rtg_slam_b200 import rasterizer
    from rtg_slam_b200.rasterizer import grad_buffers, visible_rows_only
    cam, g, mask = scene_case("masked")
    inputs, _ = inputs_for(g, "sh")
    gc, gd = scene.upstream_grads(cam, seed=5)
    gT = t_weights(cam, seed=6).astype(np.float32)
    s = spy()

    def calls(up, gaussian_grad=()):
        s.calls.clear()
        rs, leaves, total = forward(cam, inputs, cuda_device, up, mask, gaussian_grad=gaussian_grad)
        total.backward()
        for k, v in leaves.items():
            assert (v.grad is None) == (k not in gaussian_grad), k
        assert all(getattr(rs, k).grad is not None for k in CAM)
        return list(s.calls)
    assert calls((gc, gd, None)) == ["rtg_splat_backward_pose"]
    assert float(rasterizer._state(cuda_device).scratch.abs().max()) == 0.0
    assert calls((gc, gd, gT)) == ["rtg_splat_backward_pose"]
    assert calls((None, None, gT)) == ["rtg_splat_backward_pose"]
    assert float(rasterizer._state(cuda_device).scratch.abs().max()) == 0.0
    assert calls((gc, gd, None), gaussian_grad=("opacity",)) == ["rtg_splat_backward_camera"]
    assert calls((gc, gd, gT), gaussian_grad=("xyz", "shs")) == ["rtg_splat_backward_dt"]
    with visible_rows_only():
        assert calls((gc, gd, None)) == ["rtg_splat_backward_camera"]
    P = len(g["xyz"])
    with grad_buffers({"means3D": torch.empty((P, 3), device=cuda_device)}):
        assert calls((gc, gd, None)) == ["rtg_splat_backward_camera"]


# -------------------------------------------------------------------------------------------------------- pose step
def random_pose(gen):
    xi = torch.randn(6, generator=gen, dtype=torch.float64) * torch.tensor([1.0, 1.0, 1.0, 0.8, 0.8, 0.8], dtype=torch.float64)
    return torch.matrix_exp(hat(xi))


def test_pose_adam_step_matches_torch_adam(cuda_device):
    """Three steps on random gradients, from a random pose: the new pose, the moments and the written viewmatrix /
    projmatrix / campos against torch.optim.Adam (float64) on a zero twist with tangent_grad's gradient, followed by
    W2C <- matrix_exp(xi^) W2C and a reset of xi. The learning rates span both branches of the closed-form exponential."""
    from rtg_slam_b200 import _lib
    dev = cuda_device
    L = _lib.lib()
    gen = torch.Generator().manual_seed(17)
    w2c = random_pose(gen)
    projection = torch.from_numpy(scene.make_camera("small").projection).double()
    d = dict(dtype=torch.float32, device=dev)
    pose = w2c.clone().to(dev)
    m, v = torch.zeros(6, **d), torch.zeros(6, **d)
    proj32 = projection.float().to(dev)
    view, projm, campos = torch.empty(16, **d), torch.empty(16, **d), torch.empty(3, **d)
    st = _lib.RtgPoseAdam()
    st.pose, st.exp_avg, st.exp_avg_sq = pose.data_ptr(), m.data_ptr(), v.data_ptr()
    st.projection, st.viewmatrix, st.projmatrix, st.campos = (t.data_ptr() for t in (proj32, view, projm, campos))
    st.beta1, st.beta2, st.eps = 0.9, 0.999, 1e-8

    rho = torch.zeros(3, dtype=torch.float64, requires_grad=True)
    phi = torch.zeros(3, dtype=torch.float64, requires_grad=True)
    f32 = lambda x: float(np.float32(x))   # the struct carries float32 hyper-parameters; the reference uses the same values
    opt = torch.optim.Adam([{"params": [rho]}, {"params": [phi]}], lr=1.0, betas=(f32(0.9), f32(0.999)), eps=f32(1e-8))
    ref = w2c.clone()
    steps = [(0.1, 0.05, True), (1e-3, 1e-3, False), (0.02, 0.3, True)]   # (lr_trans, lr_rot, with dL/dcampos)
    for i, (lr_t, lr_r, with_cp) in enumerate(steps):
        gv, gp, gcp = (torch.randn(n, generator=gen) for n in (16, 16, 3))
        gcp = gcp if with_cp else torch.zeros(3)
        gv_d, gp_d, gcp_d = gv.to(dev), gp.to(dev), gcp.to(dev)
        st.dL_dviewmatrix, st.dL_dprojmatrix = gv_d.data_ptr(), gp_d.data_ptr()
        st.dL_dcampos = gcp_d.data_ptr() if with_cp else None
        st.lr_trans, st.lr_rot, st.step = lr_t, lr_r, i + 1
        _lib.check(L.rtg_pose_adam_step(C.byref(st), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "rtg_pose_adam_step")

        g6 = tangent_grad(gv.double().view(4, 4), gp.double().view(4, 4), gcp.double(), ref, projection)
        opt.param_groups[0]["lr"], opt.param_groups[1]["lr"] = f32(lr_t), f32(lr_r)
        rho.grad, phi.grad = g6[:3].clone(), g6[3:].clone()
        opt.step()
        with torch.no_grad():
            ref = torch.matrix_exp(hat(torch.cat([rho, phi]))) @ ref
            rho.zero_()
            phi.zero_()
        ref_m = torch.cat([opt.state[rho]["exp_avg"], opt.state[phi]["exp_avg"]])
        ref_v = torch.cat([opt.state[rho]["exp_avg_sq"], opt.state[phi]["exp_avg_sq"]])
        ref_view = ref.t()
        ref_arrays = {"viewmatrix": ref_view.reshape(-1), "projmatrix": (ref_view @ projection).reshape(-1),
                      "campos": -(ref[:3, :3].t() @ ref[:3, 3])}
        got = {"pose": pose.cpu(), "exp_avg": m.cpu().double(), "exp_avg_sq": v.cpu().double(), "viewmatrix": view.cpu().double(),
               "projmatrix": projm.cpu().double(), "campos": campos.cpu().double()}
        want = dict(ref_arrays, pose=ref, exp_avg=ref_m, exp_avg_sq=ref_v)
        for k in want:
            err = float((got[k] - want[k]).abs().max() / max(1.0, float(want[k].abs().max())))
            print(f"step {i + 1} {k}: {err:.2e}")
            assert err <= 1e-6, (i, k, err)
        # rigid to double precision
        R = pose.cpu()[:3, :3]
        assert float((R @ R.t() - torch.eye(3, dtype=torch.float64)).abs().max()) < 1e-12


# -------------------------------------------------------------------------------------------------------- refinement
ARGS = types.SimpleNamespace(renderer_opaque_threshold=0.6, renderer_normal_threshold=60, renderer_depth_threshold=1.0,
                             max_sh_degree=3, color_sigma=3.0, active_sh_degree=3)


def refiner_camera(cam, w2c):
    """A reference-Camera-like object at the pose w2c."""
    return types.SimpleNamespace(FoVx=2 * math.atan(cam.tanfovx), FoVy=2 * math.atan(cam.tanfovy), image_height=cam.height,
                                 image_width=cam.width, world_view_transform=w2c.t().contiguous(),
                                 projection_matrix=torch.from_numpy(np.ascontiguousarray(cam.projection)).to(w2c.device),
                                 cx=cam.cx, cy=cam.cy)


@pytest.mark.parametrize("masks", ["none", "render_mask", "tile_mask"])
def test_pose_refiner_converges(cuda_device, masks):
    """test_camera_grad_gpu.test_pose_refinement_with_adam through PoseRefiner: targets rendered at the true pose, start
    1 deg / 2 cm away, 150 steps at lr 1e-3; both errors must fall to a tenth of their start. render_mask: the refiner sees
    a partial map (the Gaussians at x < 0.5) and the loss only the pixels it covers (T_map != 1 at the start pose);
    tile_mask: half the tiles are rendered."""
    from rtg_slam_b200.render import Renderer
    from rtg_slam_b200.tracking import PoseRefiner
    dev = cuda_device
    cam = scene.make_camera("small")
    g = {k: torch.from_numpy(v).to(dev) for k, v in scene.surfel_room(20_000, seed=7).items()}
    w2c_true = torch.from_numpy(np.linalg.inv(scene.small_pose()).astype(np.float32)).to(dev)
    with torch.no_grad():
        tgt = Renderer(ARGS).render(view_camera(cam, w2c_true), g)
    off = torch.tensor([0.012, -0.010, 0.012, 0.010, -0.012, 0.008], device=dev)  # 2 cm, 1.0 deg
    w2c0 = se3_exp(off) @ w2c_true
    ang0, tr0 = pose_error(w2c0, w2c_true)
    kw, gm = {}, g
    if masks == "render_mask":
        keep = g["xyz"][:, 0] < 0.5
        gm = {k: v[keep] for k, v in g.items()}
        with torch.no_grad():
            kw["render_mask"] = Renderer(ARGS).render(view_camera(cam, w2c0), gm)["T_map"][0] != 1
        frac = float(kw["render_mask"].float().mean())
        assert 0.3 < frac < 0.95, frac
    elif masks == "tile_mask":
        kw["tile_mask"] = torch.from_numpy(scene.random_tile_mask(cam, 0.5, seed=143)).to(dev)
    ref = PoseRefiner(ARGS)
    w2c, parts = ref.refine(refiner_camera(cam, w2c0), gm, tgt["render"], tgt["depth"], iters=150, lr_rot=1e-3, lr_trans=1e-3,
                            color_weight=1.0, depth_weight=1.0, **kw)
    assert w2c.shape == (4, 4) and w2c.dtype == torch.float64 and w2c.is_cuda
    assert parts.is_cuda and parts.shape == (4,)
    ang, tr = pose_error(w2c, w2c_true.double())
    print(f"PoseRefiner ({masks}): rotation {ang0:.3f} -> {ang:.3f} deg, translation {100 * tr0:.2f} -> {100 * tr:.2f} cm, "
          f"last loss {float(parts[0]):.4e}")
    assert ang < 0.1 * ang0 and tr < 0.1 * tr0, (masks, ang0, ang, tr0, tr)


def test_pose_refiner_renders_an_overflowed_iteration_again(cuda_device):
    """With a binning capacity far too small and no waiting forward ('deferred'), the first iteration is rendered empty and
    its backward raises CapacityOverflow with the capacity raised; refine() renders that iteration again and finishes."""
    from rtg_slam_b200 import rasterizer
    from rtg_slam_b200.render import Renderer
    from rtg_slam_b200.tracking import PoseRefiner
    dev = cuda_device
    cam = scene.make_camera("small")
    g = {k: torch.from_numpy(v).to(dev) for k, v in scene.surfel_room(20_000, seed=7).items()}
    w2c_true = torch.from_numpy(np.linalg.inv(scene.small_pose()).astype(np.float32)).to(dev)
    with torch.no_grad():
        tgt = Renderer(ARGS).render(view_camera(cam, w2c_true), g)
    w2c0 = se3_exp(torch.tensor([0.012, -0.010, 0.012, 0.010, -0.012, 0.008], device=dev)) @ w2c_true
    st = rasterizer._state(dev)
    prev_mode, prev_hint = st.mode, st.r_hint
    rasterizer.set_capacity_checks("deferred", dev)
    st.r_hint = 1024
    try:
        w2c, parts = PoseRefiner(ARGS).refine(refiner_camera(cam, w2c0), g, tgt["render"], tgt["depth"], iters=5, lr_rot=1e-3,
                                              lr_trans=1e-3, color_weight=1.0, depth_weight=1.0)
        raised_to = st.r_hint
    finally:
        rasterizer.set_capacity_checks(prev_mode, dev)
        st.r_hint = max(st.r_hint, prev_hint)
    assert raised_to > 1024                                         # the first render did overflow
    assert int(parts[3]) > 0                                        # the last render was not empty: depth pixels counted
    ang0, tr0 = pose_error(w2c0, w2c_true)
    ang, tr = pose_error(w2c, w2c_true.double())
    assert ang < ang0 and tr < tr0, (ang0, ang, tr0, tr)            # five steps towards the true pose
