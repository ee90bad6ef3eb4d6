"""GPU tests of the RGB-D ICP tracker: the intensity pyramid and RgbdIcpTracker.predict_pose against the float32 statement
(oracle/icp_rgbd_oracle.py), bit-identity with IcpTracker where the photometric term is off, what the term buys on a
planar wall (single pair and a frame-to-model sequence), and the argument errors."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from oracle import icp_rgbd_oracle as ro
from rtg_slam_b200 import scene

pytestmark = pytest.mark.gpu


def tracker_args(**over):
    a = dict(icp_downscales=[0.25, 0.5, 1.0], icp_warmup_frames=0, icp_use_model_depth=False, icp_downscale_iters=[5, 5, 5],
             icp_distance_threshold=0.1, icp_normal_threshold=20, icp_damping=1e-4, verbose=False,
             icp_sample_distance_threshold=0.01, icp_sample_normal_threshold=0.01, icp_fail_threshold=0.02)
    a.update(over)
    return types.SimpleNamespace(**a)


def _pair(trk, dev, K, d0, d1, c0=None, c1=None):
    Kt = torch.from_numpy(K)
    col = lambda c: None if c is None else torch.from_numpy(np.ascontiguousarray(c)).to(dev)
    if c0 is None:
        trk.update_curr_status(torch.from_numpy(d0).to(dev), Kt)
    else:
        trk.update_curr_status(torch.from_numpy(d0).to(dev), Kt, col(c0))
    trk.move_last_status()
    if c1 is None:
        trk.update_curr_status(torch.from_numpy(d1).to(dev), Kt)
    else:
        trk.update_curr_status(torch.from_numpy(d1).to(dev), Kt, col(c1))
    return trk.predict_pose({"K": Kt, "frame_id": 1})


@pytest.mark.parametrize("camname", ["ragged", "tum"])
def test_intensity_pyramid_matches_the_float32_oracle(cuda_device, camname):
    from rtg_slam_b200 import icp as ricp
    cam = scene.make_camera(camname)
    _, textured = scene.raycast_room_rgbd(cam)
    noise = np.random.default_rng(1).uniform(size=textured.shape).astype(np.float32)
    for color in (textured, noise):
        want = ro.intensity_pyramid(color, 3)
        got = ricp.build_intensity_pyramid(torch.from_numpy(color).to(cuda_device), 3)
        got_cf = ricp.build_intensity_pyramid(torch.from_numpy(np.ascontiguousarray(np.moveaxis(color, -1, 0))).to(cuda_device), 3)
        for i in range(3):
            assert tuple(got[i].shape) == want[i].shape
            assert np.abs(got[i].cpu().numpy() - want[i]).max() < 1e-6
            assert torch.equal(got_cf[i], got[i])


@pytest.mark.parametrize("camname", ["tum", "replica"])
def test_rgbd_tracker_matches_oracle_at_dataset_resolution(cuda_device, camname):
    from rtg_slam_b200 import icp as ricp
    cam0 = scene.make_camera(camname)
    cam1 = scene.make_camera(camname, c2w=scene.small_pose())
    d0, c0 = scene.raycast_room_rgbd(cam0, noise_sigma=0.002, seed=3)
    d1, c1 = scene.raycast_room_rgbd(cam1, noise_sigma=0.002, seed=4)
    K = (cam0.fx, cam0.fy, cam0.cx, cam0.cy)
    pose_ref, loss_ref, vr_ref, ok_ref, pr_ref, prmse_ref = ro.predict_pose_rgbd(d0, d1, c0, c1, K)
    trk = ricp.RgbdIcpTracker(tracker_args())
    if camname == "replica":  # channels-first colour
        c0, c1 = np.moveaxis(c0, -1, 0), np.moveaxis(c1, -1, 0)
    pose, ok = _pair(trk, cuda_device, cam0.K, d0, d1, c0, c1)
    assert isinstance(pose, np.ndarray) and pose.shape == (4, 4)
    assert np.linalg.norm(pose - pose_ref) < 1e-4
    assert ok == ok_ref and abs(trk.last_p2ploss - loss_ref) < 1e-5 + 1e-3 * loss_ref
    assert abs(trk.last_valid_ratio - vr_ref) < 1e-3
    assert abs(trk.last_photometric_ratio - pr_ref) < 1e-3
    assert abs(trk.last_photometric_rmse - prmse_ref) < 1e-3 * max(prmse_ref, 1e-3)
    assert np.linalg.norm(pose - scene.small_pose()) < 5e-3


def test_zero_weight_and_missing_colour_reproduce_icp_tracker_bit_for_bit(cuda_device):
    from rtg_slam_b200 import _lib
    from rtg_slam_b200 import icp as ricp
    cam0 = scene.make_camera("tum")
    cam1 = scene.make_camera("tum", c2w=scene.small_pose())
    d0, c0 = scene.raycast_room_rgbd(cam0, noise_sigma=0.002, seed=3)
    d1, c1 = scene.raycast_room_rgbd(cam1, noise_sigma=0.002, seed=4)
    K = (cam0.fx, cam0.fy, cam0.cx, cam0.cy)
    dev = cuda_device
    # the C level: rtg_icp_predict_pose_rgbd with weight 0 against rtg_icp_predict_pose on the same levels
    L = _lib.lib()
    v0, n0 = ricp.build_pyramids(torch.from_numpy(d0).to(dev), K, 3)
    v1, n1 = ricp.build_pyramids(torch.from_numpy(d1).to(dev), K, 3)
    i0 = ricp.build_intensity_pyramid(torch.from_numpy(c0).to(dev), 3)
    i1 = ricp.build_intensity_pyramid(torch.from_numpy(c1).to(dev), 3)
    lv = (_lib.RtgIcpLevel * 3)()
    for l, s in enumerate((0.25, 0.5, 1.0)):
        e = lv[l]
        # "0" = current frame (frame 1), "1" = previous frame (frame 0)
        e.vertex0, e.normal0, e.vertex1, e.normal1 = v1[l].data_ptr(), n1[l].data_ptr(), v0[l].data_ptr(), n0[l].data_ptr()
        e.H, e.W = v1[l].shape[0], v1[l].shape[1]
        e.fx, e.fy, e.cx, e.cy = (float(np.float32(k) * np.float32(s)) for k in K)
        e.iters = 5
    ws = ricp._workspace(dev)
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())
    cos_thr = float(np.cos(np.deg2rad(20)))
    H, W = d0.shape
    out_geo = torch.full((18,), float("nan"), device=dev)
    out_rgbd = torch.full((20,), float("nan"), device=dev)
    _lib.check(L.rtg_icp_predict_pose(lv, 3, 0.1, cos_thr, 1e-4, None, p(v0[2]), p(v1[2]), p(n0[2]), H, W, p(out_geo), None,
                                      p(ws), stream), "rtg_icp_predict_pose")
    VP = C.c_void_p * 3
    _lib.check(L.rtg_icp_predict_pose_rgbd(lv, VP(*[t.data_ptr() for t in i1]), VP(*[t.data_ptr() for t in i0]), 3, 0.1, cos_thr,
                                           1e-4, 0.0, None, p(v0[2]), p(v1[2]), p(n0[2]), H, W, p(out_rgbd), None, p(ws), stream),
               "rtg_icp_predict_pose_rgbd")
    torch.cuda.synchronize()
    assert torch.equal(out_rgbd[:18].view(torch.int32), out_geo.view(torch.int32))
    assert 0.5 < float(out_rgbd[18]) <= 1.0 and 0.0 < float(out_rgbd[19]) < 0.1
    # the Python level: IcpTracker against RgbdIcpTracker without colour, and with colour at weight 0
    trk_g = ricp.IcpTracker(tracker_args())
    pose_g, ok_g = _pair(trk_g, dev, cam0.K, d0, d1)
    for trk, cols in ((ricp.RgbdIcpTracker(tracker_args()), (None, None)),
                      (ricp.RgbdIcpTracker(tracker_args()), (c0, None)),
                      (ricp.RgbdIcpTracker(tracker_args(), photometric_weight=0.0), (c0, c1))):
        pose, ok = _pair(trk, dev, cam0.K, d0, d1, *cols)
        assert np.array_equal(pose.view(np.int32), pose_g.view(np.int32)) and ok == ok_g
        assert trk.last_p2ploss == trk_g.last_p2ploss and trk.last_valid_ratio == trk_g.last_valid_ratio
        assert trk.last_photometric_ratio == 0.0 and trk.last_photometric_rmse == 0.0


def test_planar_wall_needs_the_photometric_term(cuda_device):
    """640x480, start 2 cm / 1.5 cm in the wall's plane and 1 degree about its normal: IcpTracker keeps the in-plane error,
    RgbdIcpTracker removes at least 90 % of it. Outcomes against the ground truth only (the geometric solve is
    ill-conditioned on this frame)."""
    from rtg_slam_b200 import icp as ricp
    cam0, cam1, gt = scene.wall_cameras(640, 480)
    d0, c0 = scene.raycast_room_rgbd(cam0, spheres=(), noise_sigma=0.002, seed=3)
    d1, c1 = scene.raycast_room_rgbd(cam1, spheres=(), noise_sigma=0.002, seed=4)
    t0, r0 = scene.wall_in_plane_error(cam0, cam1, np.eye(4))
    pose_g, _ = _pair(ricp.IcpTracker(tracker_args()), cuda_device, cam0.K, d0, d1)
    t_g, r_g = scene.wall_in_plane_error(cam0, cam1, pose_g)
    assert t_g > 0.5 * t0 and r_g > 0.5 * r0, (t_g, r_g)
    trk = ricp.RgbdIcpTracker(tracker_args())
    pose, ok = _pair(trk, cuda_device, cam0.K, d0, d1, c0, c1)
    t_c, r_c = scene.wall_in_plane_error(cam0, cam1, pose)
    assert t_c < 0.1 * t0 and r_c < 0.1 * r0, (t_c, r_c)
    assert ok and trk.last_photometric_ratio > 0.3  # 2 mm noise at 640x480 fails the normal test on over half the wall


def test_frame_to_model_sequence_along_a_wall(cuda_device):
    """Ten frames sliding 1 cm per frame along the wall, frame-to-model (icp_use_model_depth=True): the render depth
    handed to update_last_status is the ray-cast depth at each tracked pose. The geometric tracker cannot see the slide;
    the RGB-D tracker's drift stays below a tenth of its drift."""
    from rtg_slam_b200 import icp as ricp
    cam0, _, _ = scene.wall_cameras(640, 480)
    Kt = torch.from_numpy(cam0.K)
    Kf = (cam0.fx, cam0.fy, cam0.cx, cam0.cy)
    dev = cuda_device
    gts = [scene.wall_cameras(640, 480, dx=0.01 * k, dy=0.0, deg=0.0)[1] for k in range(10)]
    frames = [scene.raycast_room_rgbd(c, spheres=(), noise_sigma=0.002, seed=100 + k) for k, c in enumerate(gts)]
    drift = {}
    for name, trk in (("geo", ricp.IcpTracker(tracker_args(icp_use_model_depth=True))),
                      ("rgbd", ricp.RgbdIcpTracker(tracker_args(icp_use_model_depth=True)))):
        c2w = cam0.c2w.copy()
        for k, (depth, color) in enumerate(frames):
            td = torch.from_numpy(depth).to(dev)
            if name == "rgbd":
                trk.update_curr_status(td, Kt, torch.from_numpy(color).to(dev))
            else:
                trk.update_curr_status(td, Kt)
            if k > 0:
                pose, ok = trk.predict_pose({"K": Kt, "frame_id": k})
                c2w = c2w @ pose.astype(np.float64)
            trk.move_last_status()
            cam_t = scene.Camera(cam0.width, cam0.height, cam0.fx, cam0.fy, cam0.cx, cam0.cy, c2w=c2w)
            tm = torch.from_numpy(scene.raycast_room_depth(cam_t, spheres=())).to(dev)
            _, rn = ricp.build_pyramids(tm, Kf, 1)
            render_depth = tm[..., None].contiguous().clone()
            trk.update_last_status(None, render_depth, td[..., None], rn[0], trk.normal_pyramid_t1[-1])
        drift[name] = float(np.linalg.norm(c2w[:3, 3] - gts[-1].c2w[:3, 3]))
    assert drift["geo"] > 0.05, drift
    assert drift["rgbd"] < 0.1 * drift["geo"], drift


def test_argument_errors_are_raised_before_any_cuda_work(cuda_device):
    from rtg_slam_b200 import icp as ricp
    cam = scene.make_camera("tiny")
    d, c = scene.raycast_room_rgbd(cam)
    td = torch.from_numpy(d).to(cuda_device)
    tc = torch.from_numpy(c).to(cuda_device)
    Kt = torch.from_numpy(cam.K)
    for w in (-0.1, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            ricp.RgbdIcpTracker(tracker_args(), photometric_weight=w)
    trk = ricp.RgbdIcpTracker(tracker_args())
    trk.update_curr_status(td, Kt, tc)
    before = (trk.vertex_pyramid_t1, trk.intensity_pyramid_t1, trk.depth_t1)
    bad = [(TypeError, c), (TypeError, tc.cpu()), (TypeError, tc.double()), (ValueError, tc[..., 0]),
           (ValueError, tc[:, :-1]), (ValueError, torch.cat([tc, tc[..., :1]], -1)), (ValueError, tc[1:])]
    for exc, col in bad:
        with pytest.raises(exc):
            trk.update_curr_status(td, Kt, col)
        now = (trk.vertex_pyramid_t1, trk.intensity_pyramid_t1, trk.depth_t1)
        assert all(a is b for a, b in zip(now, before))  # nothing was rebuilt
    with pytest.raises(ValueError):
        ricp.build_intensity_pyramid(tc, 5)
    with pytest.raises(TypeError):
        ricp.build_intensity_pyramid(tc.cpu(), 3)
