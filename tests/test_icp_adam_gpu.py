"""GPU parity tests of the ICP kernels and the fused Adam step, through the reference-facing Python classes."""
import os
import types

import numpy as np
import pytest
import torch

import golden
from oracle import icp_oracle as io
from rtg_slam_b200 import scene

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def tracker_args(**over):
    a = dict(icp_downscales=[0.25, 0.5, 1.0], icp_warmup_frames=0, icp_use_model_depth=False, icp_downscale_iters=[5, 5, 5],
             icp_distance_threshold=0.1, icp_normal_threshold=20, icp_damping=1e-4, verbose=False,
             icp_sample_distance_threshold=0.01, icp_sample_normal_threshold=0.01, icp_fail_threshold=0.02)
    a.update(over)
    return types.SimpleNamespace(**a)


@pytest.mark.parametrize("name", ["icp_small", "icp_ragged"])
def test_pyramids_and_levels_match_reference_golden(cuda_device, name):
    from rtg_slam_b200 import icp as ricp
    g = golden.load(name)
    K = tuple(float(k) for k in g["K"])
    d0 = torch.from_numpy(g["depth0"]).to(cuda_device)
    d1 = torch.from_numpy(g["depth1"]).to(cuda_device)
    v0, n0 = ricp.build_pyramids(d0, K, 3)
    v1, n1 = ricp.build_pyramids(d1, K, 3)
    for i in range(3):
        assert np.abs(v0[i].cpu().numpy() - g[f"v0_{i}"]).max() < 1e-6
        assert np.abs(n0[i].cpu().numpy() - g[f"n0_{i}"]).max() < 1e-4
        assert np.abs(n1[i].cpu().numpy() - g[f"n1_{i}"]).max() < 1e-4
    pose = torch.eye(4, device=cuda_device)
    for lvl, s in enumerate((0.25, 0.5, 1.0)):
        tr = ricp.ICP(5, damping=1e-4, distance_threshold=0.1, normal_threshold=20)
        Kl = tuple(float(np.float32(k) * np.float32(s)) for k in K)
        pose, vr = tr.icp(pose, v1[lvl], v0[lvl], n1[lvl], n0[lvl], Kl)
        assert np.linalg.norm(pose.cpu().numpy() - g["poses"][lvl]) < 1e-4, lvl
        assert abs(float(vr) - g["valid_ratios"][lvl]) < 1e-3


@pytest.mark.parametrize("camname", ["tum", "replica"])
def test_tracker_matches_oracle_at_dataset_resolution(cuda_device, camname):
    from rtg_slam_b200 import icp as ricp
    cam0 = scene.make_camera(camname)
    cam1 = scene.make_camera(camname, c2w=scene.small_pose())
    d0 = scene.raycast_room_depth(cam0, noise_sigma=0.002, seed=3)
    d1 = scene.raycast_room_depth(cam1, noise_sigma=0.002, seed=4)
    K = (cam0.fx, cam0.fy, cam0.cx, cam0.cy)
    pose_ref, loss_ref, vr_ref, ok_ref = io.predict_pose(d0, d1, K)
    trk = ricp.IcpTracker(tracker_args())
    Kt = torch.from_numpy(cam0.K)
    trk.update_curr_status(torch.from_numpy(d0).to(cuda_device), Kt)
    trk.move_last_status()
    trk.update_curr_status(torch.from_numpy(d1).to(cuda_device), Kt)
    pose, ok = trk.predict_pose({"K": Kt, "frame_id": 1})
    assert isinstance(pose, np.ndarray) and pose.shape == (4, 4)
    assert np.linalg.norm(pose - pose_ref) < 1e-4
    assert ok == ok_ref and abs(trk.last_p2ploss - loss_ref) < 1e-5 + 1e-3 * loss_ref
    # ground truth: pose maps current-frame points into the previous frame == c2w of the current camera
    assert np.linalg.norm(pose - scene.small_pose()) < 5e-3


def test_fill_model_depth(cuda_device):
    from rtg_slam_b200 import icp as ricp
    g = golden.load("icp_small")
    K = tuple(g["K"])
    v0, n0 = io.build_pyramids(g["depth0"], K)
    trk = ricp.IcpTracker(tracker_args())
    rd = torch.from_numpy(g["fill_render_depth"].copy()).to(cuda_device)[..., None].contiguous()
    trk.update_last_status(None, rd, torch.from_numpy(g["depth0"]).to(cuda_device)[..., None],
                           torch.from_numpy(g["fill_render_normal"]).to(cuda_device), torch.from_numpy(n0[-1]).to(cuda_device))
    got = rd[..., 0].cpu().numpy()
    diff = got != g["fill_out"]
    # the only pixels that may differ from the reference's result are those whose fill decision sits on one of its two
    # thresholds to fp32 rounding (|render - frame depth| vs 0.01 m; 1 - cos(normals) vs 0.01, the golden's frame normals
    # being the reference's own, the test's the oracle's: equal to 1e-5): name them, and require all others to be exact
    rdep, fdep, rn, fn = g["fill_render_depth"], g["depth0"], g["fill_render_normal"], n0[-1]
    cos = (rn * fn).sum(-1) / (np.maximum(np.linalg.norm(rn, axis=-1), 1e-8) * np.maximum(np.linalg.norm(fn, axis=-1), 1e-8))
    borderline = (np.abs(np.abs(rdep - fdep) - 0.01) < 1e-6) | (np.abs((1 - cos) - 0.01) < 2e-4)
    assert not np.any(diff & ~borderline), int((diff & ~borderline).sum())
    assert diff.mean() < 1e-3
    assert trk.last_model_depth is rd


def test_fused_adam_matches_torch(cuda_device):
    from rtg_slam_b200.optim import FusedAdam
    dev = cuda_device
    torch.manual_seed(0)
    P = 5000
    # the six groups of GaussianPointCloud.parametrize with the lrs of configs/base.yaml:82-86
    shapes = [(P, 3), (P, 1, 3), (P, 15, 3), (P, 1), (P, 3), (P, 4)]
    lrs = [1e-3, 5e-4, 5e-4 / 20.0, 0.0, 4e-3, 1e-3]
    pa = [torch.randn(s, device=dev).requires_grad_(True) for s in shapes]
    pb = [p.detach().clone().requires_grad_(True) for p in pa]
    oa = FusedAdam([{"params": [p], "lr": lr} for p, lr in zip(pa, lrs)], lr=0.0, eps=1e-15)
    ob = torch.optim.Adam([{"params": [p], "lr": lr} for p, lr in zip(pb, lrs)], lr=0.0, eps=1e-15)
    rng = np.random.default_rng(1)
    for it in range(10):
        for p, q in zip(pa, pb):
            gr = torch.randn_like(p) * float(10 ** rng.uniform(-5, 0))
            gr[::7] = 0  # exact zeros must stay harmless with eps=1e-15
            p.grad, q.grad = gr.clone(), gr.clone()
        oa.step(); ob.step()
        oa.zero_grad(set_to_none=True); ob.zero_grad(set_to_none=True)
    for p, q, lr in zip(pa, pb, lrs):
        assert float(((p - q).abs().max() / q.abs().max()).detach()) < 1e-5  # SURVEY 8(c)
        if lr == 0.0:
            assert torch.equal(p, q)  # opacity_lr is 0 in every shipped config: parameters must not move
    sa, sb = oa.state[pa[2]], ob.state[pb[2]]
    assert float((sa["exp_avg"] - sb["exp_avg"]).abs().max()) < 1e-6 * float(sb["exp_avg"].abs().max()) + 1e-12
    # a parameter without a gradient is skipped, as in torch
    pa[0].grad = None
    before = pa[0].detach().clone()
    pa[1].grad = torch.ones_like(pa[1])
    oa.step()
    assert torch.equal(before, pa[0])


def test_fused_adam_at_map_size_matches_float64_torch(cuda_device):
    """The six groups at P = 1,000,003 plus a parameter at a storage offset of one float, against torch.optim.Adam in
    float64 from the same float32 start. adam_kernel caps its grid at 2112 x 256 threads of four floats: features_rest
    (45 M elements) takes 21 grid-stride passes; the (P,1), (P,3) and (P,15,3) groups have numel % 4 != 0, so their
    scalar tail runs after the float4 body; the offset view is not 16-byte aligned and takes the scalar path throughout."""
    from rtg_slam_b200.optim import FusedAdam
    dev = cuda_device
    P = 1_000_003
    gen = torch.Generator(device=dev).manual_seed(11)
    shapes = [(P, 3), (P, 1, 3), (P, 15, 3), (P, 1), (P, 3), (P, 4)]
    lrs = [1e-3, 5e-4, 5e-4 / 20.0, 0.0, 4e-3, 1e-3]
    pa = [torch.randn(s, device=dev, generator=gen).requires_grad_(True) for s in shapes]
    base = torch.randn(P * 3 + 1, device=dev, generator=gen)
    before = base[:1].clone()
    pa.append(base[1:].view(P, 3).requires_grad_(True))              # a contiguous view one float into its storage
    lrs.append(2e-3)
    assert pa[-1].is_contiguous() and pa[-1].data_ptr() % 16 == 4
    assert [p.numel() % 4 for p in pa[:6]] == [1, 1, 3, 3, 1, 0]
    pb = [p.detach().double().requires_grad_(True) for p in pa]
    oa = FusedAdam([{"params": [p], "lr": lr} for p, lr in zip(pa, lrs)], lr=0.0, eps=1e-15)
    ob = torch.optim.Adam([{"params": [p], "lr": lr} for p, lr in zip(pb, lrs)], lr=0.0, eps=1e-15)
    start = [p.detach().clone() for p in pa]
    rng = np.random.default_rng(2)
    for it in range(3):
        for p, q in zip(pa, pb):
            gr = torch.randn(p.shape, device=dev, generator=gen) * float(10 ** rng.uniform(-5, 0))
            gr.view(-1)[::7] = 0                                         # exact zeros stay harmless with eps = 1e-15
            p.grad, q.grad = gr, gr.double()
        oa.step(); ob.step()
        oa.zero_grad(set_to_none=True); ob.zero_grad(set_to_none=True)
    for k, (p, q, lr, p0) in enumerate(zip(pa, pb, lrs, start)):
        e = float((p.detach().double() - q.detach()).abs().max() / q.detach().abs().max())
        assert e < 1e-5, (k, e)
        if lr == 0.0:
            assert torch.equal(p.detach(), p0)                          # the lr = 0 group does not move, bit for bit
        else:
            assert not torch.equal(p.detach(), p0), k
    assert torch.equal(base[:1], before)                                 # the float in front of the view is not written


def test_renderer_api(cuda_device):
    """Renderer.render returns the reference's dictionary; the normal map equals normal[depth_index_map]."""
    from rtg_slam_b200.render import Renderer
    import math
    dev = cuda_device
    cam = scene.make_camera("small")
    g = scene.surfel_room(3000, seed=1)
    args = types.SimpleNamespace(renderer_opaque_threshold=0.6, renderer_normal_threshold=60, renderer_depth_threshold=1.0,
                                 max_sh_degree=3, color_sigma=3.0, active_sh_degree=3)
    vc = types.SimpleNamespace(FoVx=2 * math.atan(cam.tanfovx), FoVy=2 * math.atan(cam.tanfovy), image_height=cam.height,
                               image_width=cam.width, world_view_transform=torch.from_numpy(cam.viewmatrix).to(dev),
                               full_proj_transform=torch.from_numpy(cam.projmatrix).to(dev),
                               camera_center=torch.from_numpy(cam.campos).to(dev), cx=cam.cx, cy=cam.cy)
    t = {k: torch.from_numpy(v).to(dev) for k, v in g.items()}
    data = dict(xyz=t["xyz"], opacity=t["opacity"], scales=t["scales"], rotations=t["rotations"], shs=t["shs"], normal=t["normal"])
    out = Renderer(args).render(vc, data)
    # the reference's keys (SLAM/render.py:135-145) plus "radii" (the visibility MapOptimizer.step takes)
    assert set(out) == {"render", "depth", "normal", "color_index_map", "depth_index_map", "color_hit_weight", "depth_hit_weight", "T_map",
                        "radii"}
    idx = out["depth_index_map"][0]
    ref = torch.zeros_like(out["render"])
    ref[:, idx > -1] = t["normal"][idx[idx > -1].long()].permute(1, 0)  # the reference's own expression (render.py:130-133)
    assert torch.equal(ref, out["normal"])
    # the normal map is differentiable w.r.t. the per-Gaussian normals, as the reference's indexing expression is (the
    # cosine normal loss of mapper.py:433-446 back-propagates through it)
    na = t["normal"].clone().requires_grad_(True)
    nb = t["normal"].clone().requires_grad_(True)
    wts = torch.rand_like(out["render"])
    (Renderer(args).render(vc, dict(data, normal=na))["normal"] * wts).sum().backward()
    refn = torch.zeros_like(out["render"])
    refn[:, idx > -1] = nb[idx[idx > -1].long()].permute(1, 0)
    (refn * wts).sum().backward()
    assert float((na.grad - nb.grad).abs().max()) <= 1e-5 * float(nb.grad.abs().max()) and float(nb.grad.abs().max()) > 0


@pytest.mark.parametrize("use_mask", [False, True])
def test_fused_loss_matches_the_reference_expressions(cuda_device, use_mask):
    """rtg_slam_b200.loss.l1_color_depth_loss against the eager expressions of Mapping.loss_update
    (mapper.py:402-431,444-451), values and gradients through the rasterizer outputs."""
    from rtg_slam_b200.loss import l1_color_depth_loss
    dev = cuda_device
    torch.manual_seed(3)
    H, W = 75, 100
    render = torch.rand(3, H, W, device=dev, requires_grad=True)
    depth = (torch.rand(1, H, W, device=dev) * 3).requires_grad_(True)
    depth_index = torch.randint(-1, 50, (1, H, W), device=dev, dtype=torch.int32)
    gt_color = torch.rand(H, W, 3, device=dev)
    gt_depth = torch.rand(H, W, 1, device=dev) * 3
    gt_depth[torch.rand(H, W, 1, device=dev) < 0.1] = 0
    gt_depth = torch.where(torch.rand(H, W, 1, device=dev) < 0.5, depth.detach().permute(1, 2, 0) + 0.05 * torch.randn(H, W, 1, device=dev), gt_depth)
    mask = (torch.rand(H, W, device=dev) < 0.6) if use_mask else None
    loss, parts = l1_color_depth_loss({"render": render, "depth": depth, "depth_index_map": depth_index}, gt_color, gt_depth,
                                      render_mask=mask, color_weight=0.8, depth_weight=1.0, depth_error_max=0.1)
    loss.backward()
    g1, g2 = render.grad.clone(), depth.grad.clone()
    render.grad = None; depth.grad = None
    # the reference's expressions
    image, d, di = render.permute(1, 2, 0), depth.permute(1, 2, 0), depth_index.permute(1, 2, 0)
    rm = torch.ones(H, W, dtype=torch.bool, device=dev) if mask is None else mask.bool()
    color_loss = torch.abs(image[rm] - gt_color[rm]).mean()
    err = d - gt_depth
    valid = (di != -1).squeeze() & (gt_depth > 0).squeeze() & (err < 0.1).squeeze() & rm
    depth_loss = torch.abs(err[valid]).mean()
    ref = 1.0 * depth_loss + 0.8 * color_loss
    ref.backward()
    assert abs(float(loss) - float(ref)) < 1e-6 * max(1.0, abs(float(ref)))
    assert abs(float(parts[1]) - float(color_loss)) < 1e-6 and abs(float(parts[2]) - float(depth_loss)) < 1e-6
    assert int(parts[3]) == int(valid.sum())
    assert float((g1 - render.grad).abs().max()) < 1e-9 + 1e-5 * float(render.grad.abs().max())
    assert float((g2 - depth.grad).abs().max()) < 1e-9 + 1e-5 * float(depth.grad.abs().max())


# ---------------------------------------------------------------- sequence-level tracking (BASELINE configs[3], SURVEY 8(c))
@pytest.mark.parametrize("name", ["icp_sequence_ragged", "icp_sequence_tum"])
def test_tracker_sequence_matches_reference_trajectory(cuda_device, name):
    """IcpTracker driven over a synthetic TUM-like sequence the way SLAM/multiprocess/tracker.py:265-290 drives it, with
    icp_use_model_depth=True (the setting of every shipped dataset config: the frame-to-MODEL association), against the
    trajectory of the UNMODIFIED reference tracker on the same frames (tests/golden/make_icp_sequence_golden.py).
    Tolerances of SURVEY 8(c): per-frame ||dT||_F < 1e-4, ATE within 1 mm of the reference trajectory."""
    from golden.make_icp_sequence_golden import SEQUENCES, sequence_inputs, tracker_args as seq_args
    from rtg_slam_b200 import icp as ricp
    gold = np.load(os.path.join(GOLD, name + ".npz"))
    cfg = SEQUENCES[name]
    cam = scene.make_camera(cfg["cam"])
    Kt = torch.from_numpy(cam.K)
    Kf = (cam.fx, cam.fy, cam.cx, cam.cy)
    trk = ricp.IcpTracker(seq_args(cfg["use_model_depth"], cfg["warmup"]))
    traj = [np.eye(4)]
    for k in range(cfg["frames"]):
        depth, model = sequence_inputs(name, k)
        td = torch.from_numpy(depth).to(cuda_device)
        trk.update_curr_status(td, Kt)
        if k > 0:
            pose, ok = trk.predict_pose({"K": Kt, "frame_id": k})
            assert bool(ok) == bool(gold["success"][k - 1]), k
            err = np.linalg.norm(pose.astype(np.float64) - gold["rel_poses"][k - 1].astype(np.float64))
            assert err < 1e-4, f"frame {k}: ||dT||_F = {err:.2e}"
            traj.append(traj[-1] @ pose.astype(np.float64))  # tracker.py:282
        trk.move_last_status()
        # the mapper's render of this frame becomes the next reference depth (slam.py -> tracker.update_last_status)
        tm = torch.from_numpy(model).to(cuda_device)
        _, rn = ricp.build_pyramids(tm, Kf, 1)
        render_depth = tm[..., None].contiguous().clone()
        trk.update_last_status(None, render_depth, td[..., None], rn[0], trk.normal_pyramid_t1[-1])
        assert trk.last_model_depth is render_depth
    traj = np.stack(traj)
    d = traj[:, :3, 3] - gold["trajectory"][:, :3, 3]
    ate_vs_ref = float(np.sqrt((d * d).sum(-1).mean()))
    assert ate_vs_ref < 1e-3, ate_vs_ref
    d = traj[:, :3, 3] - gold["gt"][:, :3, 3]
    assert abs(float(np.sqrt((d * d).sum(-1).mean())) - float(gold["ate_vs_gt"])) < 1e-3


def test_predict_pose_before_any_frame_raises_like_the_reference(cuda_device):
    """SLAM/icp.py:421-449: with no previous frame the reference sets the identity pose and then evaluates
    point2plane_loss on a None pyramid, i.e. raises TypeError; callers only get here after move_last_status()."""
    from rtg_slam_b200 import icp as ricp
    cam = scene.make_camera("small")
    trk = ricp.IcpTracker(tracker_args())
    Kt = torch.from_numpy(cam.K)
    trk.update_curr_status(torch.from_numpy(scene.raycast_room_depth(cam)).to(cuda_device), Kt)
    with pytest.raises(TypeError):
        trk.predict_pose({"K": Kt, "frame_id": 0})


@pytest.mark.parametrize("use_mask", [False, True])
def test_mapping_loss_with_normal_and_ssim_terms(cuda_device, use_mask):
    """rtg_slam_b200.loss.mapping_loss against the eager expressions of Mapping.loss_update (mapper.py:402-451) including
    the cosine normal term and -- without a render mask, as in the reference -- the SSIM term of utils/loss_utils.py;
    values, gradients, and the single read-back of the reported losses."""
    import torch.nn.functional as F
    from rtg_slam_b200.loss import mapping_loss, report_losses
    dev = cuda_device
    torch.manual_seed(5)
    H, W = 70, 90
    render = torch.rand(3, H, W, device=dev, requires_grad=True)
    depth = (torch.rand(1, H, W, device=dev) * 3).requires_grad_(True)
    normal = F.normalize(torch.randn(3, H, W, device=dev), dim=0).requires_grad_(True)
    depth_index = torch.randint(-1, 50, (1, H, W), device=dev, dtype=torch.int32)
    gt_color = torch.rand(H, W, 3, device=dev)
    gt_depth = depth.detach().permute(1, 2, 0) + 0.05 * torch.randn(H, W, 1, device=dev)
    gt_depth[torch.rand(H, W, 1, device=dev) < 0.1] = 0
    gt_normal = F.normalize(torch.randn(H, W, 3, device=dev), dim=-1)
    gt_normal[torch.rand(H, W, device=dev) < 0.15] = 0
    mask = (torch.rand(H, W, device=dev) < 0.6) if use_mask else None
    w = dict(color_weight=0.8, depth_weight=1.0, normal_weight=0.1, ssim_weight=0.2)
    loss, parts = mapping_loss({"render": render, "depth": depth, "normal": normal, "depth_index_map": depth_index},
                               {"color_map": gt_color, "depth_map": gt_depth, "normal_map": gt_normal}, render_mask=mask,
                               depth_error_max=0.1, **w)
    loss.backward()
    got = [t.grad.clone() for t in (render, depth, normal)]
    for t in (render, depth, normal):
        t.grad = None
    _, parts2 = mapping_loss({"render": render, "depth": depth, "normal": normal, "depth_index_map": depth_index},
                             {"color_map": gt_color, "depth_map": gt_depth, "normal_map": gt_normal}, render_mask=mask,
                             depth_error_max=0.1, **w)
    assert torch.equal(parts, parts2)  # fixed-order sums: the same bits from call to call
    # the reference's expressions
    image, d, n, di = render.permute(1, 2, 0), depth.permute(1, 2, 0), normal.permute(1, 2, 0), depth_index.permute(1, 2, 0)
    ssim_loss = torch.zeros((), device=dev)
    if mask is None:
        rm = torch.ones(H, W, dtype=torch.bool, device=dev)
        from rtg_slam_b200.loss import _ssim_term  # the reference's torch expressions, in float64 (no TF32 convolution in the way)
        ssim_loss = _ssim_term(image.permute(2, 0, 1).double(), gt_color.permute(2, 0, 1).double()).float()
    else:
        rm = mask.bool()
    color_loss = torch.abs(image[rm] - gt_color[rm]).mean()
    err = d - gt_depth
    valid = (di != -1).squeeze() & (gt_depth > 0).squeeze() & (err < 0.1).squeeze() & rm
    depth_loss = torch.abs(err[valid]).mean()
    cos_dist = 1 - F.cosine_similarity(n, gt_normal, dim=-1)
    vn = rm & (di != -1).squeeze() & (~(gt_normal == 0).all(dim=-1))
    normal_loss = cos_dist[vn].mean()
    ref = w["depth_weight"] * depth_loss + w["normal_weight"] * normal_loss + w["color_weight"] * color_loss + w["ssim_weight"] * ssim_loss
    ref.backward()
    assert abs(float(loss.detach()) - float(ref.detach())) < 1e-5 * max(1.0, abs(float(ref.detach())))
    for a, t in zip(got, (render, depth, normal)):
        assert float((a - t.grad).abs().max()) < 1e-9 + 2e-5 * float(t.grad.abs().max())
    rep = report_losses(parts, scale_loss=torch.tensor(0.25, device=dev))
    assert set(rep) == {"total_loss", "depth_loss", "ssim_loss", "normal_loss", "color_loss", "scale_loss"}
    assert abs(rep["normal_loss"] - float(normal_loss)) < 1e-5 and abs(rep["color_loss"] - float(color_loss)) < 1e-6
    assert abs(rep["ssim_loss"] - float(ssim_loss)) < 5e-6 and rep["scale_loss"] == 0.25
    assert int(parts[5]) == int(vn.sum())


@pytest.mark.gpu
@pytest.mark.parametrize("shape,kind", [((3, 70, 90), "noise"), ((1, 16, 16), "noise"), ((3, 5, 7), "noise"), ((2, 33, 130), "noise"),
                                        ((3, 680, 1200), "noise"), ((3, 680, 1200), "smooth")])
def test_fused_ssim_matches_the_reference_formula(cuda_device, shape, kind):
    """rtg_slam_b200.loss.ssim_loss (three kernels: separable tiled SSIM, fixed-order mean, closed-form backward) against the
    reference's expression (utils/loss_utils.py:40-100: grouped 11x11 conv2d, zero padding) differentiated by autograd in
    float64. Tolerance: value 1e-5; gradient 1e-4 of its largest entry, or 4x the error of the same torch expression
    evaluated in float32 where that is larger (smooth images: sigma^2 = E[x^2] - mu^2 cancels and sits next to C2 = 9e-4)."""
    from rtg_slam_b200.loss import ssim_loss, _ssim_term
    dev = cuda_device
    torch.manual_seed(sum(shape))
    C, H, W = shape
    if kind == "noise":
        a = torch.rand(shape, device=dev)
        b = torch.rand(shape, device=dev)
        b[:, : H // 2] = (a[:, : H // 2] + 0.02 * torch.randn(C, H // 2, W, device=dev)).clamp(0, 1)
    else:  # low-frequency images with flat (black) regions, like a render next to its frame
        yy, xx = torch.meshgrid(torch.linspace(0, 1, H, device=dev), torch.linspace(0, 1, W, device=dev), indexing="ij")
        a = torch.stack([0.5 + 0.4 * torch.sin(6 * xx + c) * torch.cos(4 * yy) for c in range(C)])
        b = (a + 0.01 * torch.randn(shape, device=dev)).clamp(0, 1)
        a[:, : H // 4, : W // 3] = 0
        b[:, : H // 5, : W // 4] = 0
    a.requires_grad_(True)
    got = ssim_loss(a, b)
    (3.0 * got).backward()
    g_ours = a.grad.clone() / 3.0
    a.grad = None
    ref64 = _ssim_term(a.double(), b.double())
    ref64.backward()
    g64 = a.grad.clone().double()
    a.grad = None
    ref32 = _ssim_term(a, b)
    ref32.backward()
    g32 = a.grad.clone()
    gmax = float(g64.abs().max())
    err32 = float((g32.double() - g64).abs().max())
    err = float((g_ours.double() - g64).abs().max())
    assert abs(float(got.detach()) - float(ref64.detach())) < 1e-5, (float(got.detach()), float(ref64.detach()))
    assert err <= max(1e-4 * gmax, 4 * err32), (err, err32, gmax)
    # value only (no gradient requested) and reproducibility of the fixed-order mean
    with torch.no_grad():
        v1, v2 = ssim_loss(a.detach(), b), ssim_loss(a.detach(), b)
    assert float(v1) == float(v2) == float(got.detach())


@pytest.mark.gpu
def test_fused_ssim_argument_errors(cuda_device):
    from rtg_slam_b200.loss import ssim_loss
    a = torch.rand(3, 20, 20, device=cuda_device)
    with pytest.raises(ValueError):
        ssim_loss(a, a[:, :10])
    with pytest.raises(ValueError):
        ssim_loss(a[0], a[0])
    with pytest.raises(TypeError):
        ssim_loss(a.double(), a.double())
    with pytest.raises(TypeError):
        ssim_loss(a.cpu(), a.cpu())
