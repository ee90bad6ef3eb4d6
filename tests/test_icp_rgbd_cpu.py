"""The RGB-D ICP statement (oracle/icp_rgbd_oracle.py) on the CPU: the intensity pyramid, the photometric Jacobian against
finite differences, w = 0 against the geometric oracle, what the photometric term buys on a planar wall, and the host
validation of the two C entry points (no device needed)."""
import ctypes as C

import numpy as np
import pytest

from oracle import icp_oracle as io
from oracle import icp_rgbd_oracle as ro
from rtg_slam_b200 import _lib, scene


def test_intensity_pyramid_matches_a_direct_loop_at_ragged_sizes():
    rng = np.random.default_rng(0)
    H, W = 70, 90
    color = rng.uniform(size=(H, W, 3))
    levels = ro.intensity_pyramid(color, 3)
    levels_cf = ro.intensity_pyramid(np.ascontiguousarray(np.moveaxis(color, -1, 0)), 3, channels_last=False)
    for i, p in enumerate((4, 2, 1)):
        want = np.zeros((H // p, W // p))
        for y in range(H // p):
            for x in range(W // p):
                s = 0.0
                for a in range(p):
                    for c in range(p):
                        R, G, B = color[y * p + a, x * p + c]
                        s += 0.299 * R + 0.587 * G + 0.114 * B
                want[y, x] = s / (p * p)
        assert levels[i].shape == want.shape
        np.testing.assert_allclose(levels[i], want, rtol=0, atol=1e-14)
        np.testing.assert_array_equal(levels_cf[i], levels[i])


def _textured_pair(camname="tiny"):
    cam0 = scene.make_camera(camname)
    cam1 = scene.make_camera(camname, c2w=scene.small_pose())
    d0, c0 = scene.raycast_room_rgbd(cam0, seed=3)
    d1, c1 = scene.raycast_room_rgbd(cam1, seed=4)
    return cam0, (d0, c0), (d1, c1)


def test_photometric_jacobian_matches_central_differences():
    """J of every row against (r(exp(+eps e_k) T) - r(exp(-eps e_k) T)) / 2 eps in float64, on the pixels whose validity
    and bilinear cell stay the same under both steps (r is smooth there)."""
    cam, (d0, c0), (d1, c1) = _textured_pair("small")
    K = (cam.fx, cam.fy, cam.cx, cam.cy)
    v_prev, n_prev = io.build_pyramids(d0.astype(np.float64), K, 1)
    v_cur, n_cur = io.build_pyramids(d1.astype(np.float64), K, 1)
    I_prev = ro.intensity_pyramid(c0.astype(np.float64), 1)[0]
    I_cur = ro.intensity_pyramid(c1.astype(np.float64), 1)[0]
    T = np.linalg.inv(scene.small_pose(rot_deg=(0.3, 0.2, -0.2), trans=(0.005, 0.004, -0.003))) @ scene.small_pose()
    cos_thr = np.cos(np.deg2rad(20.0))
    args = (v_cur[0], v_prev[0], n_cur[0], n_prev[0], I_cur, I_prev, K, 0.1, cos_thr)
    r, J, valid = ro.photometric_rows(T, *args)
    assert valid.sum() > 0.5 * valid.size

    def cell(P):
        _, u, v = ro.project(P, v_cur[0], K)
        return np.floor(u), np.floor(v)

    eps = 1e-6
    cu0, cv0 = cell(T)
    checked = 0
    for k in range(6):
        e = np.zeros(6)
        e[k] = eps
        Tp, Tm = io.exp_se3(e) @ T, io.exp_se3(-e) @ T
        rp, _, vp = ro.photometric_rows(Tp, *args)
        rm, _, vm = ro.photometric_rows(Tm, *args)
        (cup, cvp), (cum, cvm) = cell(Tp), cell(Tm)
        keep = valid & vp & vm & (cup == cu0) & (cum == cu0) & (cvp == cv0) & (cvm == cv0)
        assert keep.sum() > 0.5 * valid.sum()
        fd = (rp - rm)[keep] / (2 * eps)
        scale = np.abs(J[keep, k]).max()
        rel = np.abs(fd - J[keep, k]).max() / scale
        assert rel < 2e-6, (k, rel)
        checked += int(keep.sum())
    assert checked > 1000


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_zero_weight_reproduces_the_geometric_oracle_exactly(dtype):
    cam, (d0, c0), (d1, c1) = _textured_pair("small")
    K = (cam.fx, cam.fy, cam.cx, cam.cy)
    v_prev, n_prev = io.build_pyramids(d0.astype(dtype), K, 1)
    v_cur, n_cur = io.build_pyramids(d1.astype(dtype), K, 1)
    I_prev = ro.intensity_pyramid(c0.astype(dtype), 1)[0]
    I_cur = ro.intensity_pyramid(c1.astype(dtype), 1)[0]
    pose0 = np.eye(4, dtype=dtype)
    want, vr = io.icp_level(pose0, v_cur[0], v_prev[0], n_cur[0], n_prev[0], K, 5, 0.1, 20.0, 1e-4)
    got, vr2, pr, prmse = ro.icp_level_rgbd(pose0, v_cur[0], v_prev[0], n_cur[0], n_prev[0], I_cur, I_prev, K, 5, 0.1, 20.0,
                                            1e-4, photometric_weight=0.0)
    np.testing.assert_array_equal(got, want)
    assert vr2 == vr and pr == vr and prmse > 0
    full = ro.predict_pose_rgbd(d0.astype(dtype), d1.astype(dtype), c0, c1, K, photometric_weight=0.0)
    geo = io.predict_pose(d0.astype(dtype), d1.astype(dtype), K)
    np.testing.assert_array_equal(full[0], geo[0])
    assert full[1:4] == geo[1:4]


def test_colour_layouts_give_the_same_pose():
    cam, (d0, c0), (d1, c1) = _textured_pair("tiny")
    K = (cam.fx, cam.fy, cam.cx, cam.cy)
    a = ro.predict_pose_rgbd(d0, d1, c0, c1, K)
    b = ro.predict_pose_rgbd(d0, d1, np.moveaxis(c0, -1, 0), np.moveaxis(c1, -1, 0), K, channels_last=False)
    np.testing.assert_array_equal(a[0], b[0])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_planar_wall_is_degenerate_for_geometry_and_tracked_with_colour(dtype):
    """160x120, start 2 cm / 1.5 cm in the wall's plane and 1 degree about its normal: the point-to-plane residual cannot
    see those three directions (the geometric oracle keeps more than half of the error), the photometric term can (the
    RGB-D oracle removes at least 90 % of the in-plane translation and of the rotation error)."""
    cam0, cam1, gt = scene.wall_cameras(160, 120)
    d0, c0 = scene.raycast_room_rgbd(cam0, spheres=())
    d1, c1 = scene.raycast_room_rgbd(cam1, spheres=())
    K = (cam0.fx, cam0.fy, cam0.cx, cam0.cy)
    t_start, r_start = scene.wall_in_plane_error(cam0, cam1, np.eye(4))
    assert abs(t_start - 0.025) < 1e-9 and abs(r_start - 1.0) < 1e-9
    pose_geo = io.predict_pose(d0.astype(dtype), d1.astype(dtype), K)[0]
    t_geo, r_geo = scene.wall_in_plane_error(cam0, cam1, pose_geo)
    assert t_geo > 0.5 * t_start and r_geo > 0.5 * r_start, (t_geo, r_geo)
    pose, loss, vr, ok, pr, prmse = ro.predict_pose_rgbd(d0.astype(dtype), d1.astype(dtype), c0, c1, K)
    t_rgbd, r_rgbd = scene.wall_in_plane_error(cam0, cam1, pose)
    assert t_rgbd < 0.1 * t_start and r_rgbd < 0.1 * r_start, (t_rgbd, r_rgbd)
    assert ok and pr > 0.9 and prmse < 0.01
    assert np.linalg.norm(pose - gt) < 1e-3


def test_c_entry_points_reject_bad_arguments_before_touching_cuda():
    L = _lib.lib()
    dummy = C.c_void_p(16)  # never dereferenced: every call below fails validation first
    pools = (C.c_int32 * 3)(4, 2, 1)
    outs = (C.c_void_p * 3)(16, 16, 16)
    bi = L.rtg_icp_build_intensity_pyramid
    assert bi(None, 48, 64, 1, 3, pools, outs, None) == -1 and b"rtg_icp_build_intensity_pyramid" in L.rtg_last_error()
    assert bi(dummy, 48, 64, 1, 3, None, outs, None) == -1
    assert bi(dummy, 48, 64, 1, 3, pools, None, None) == -1
    assert bi(dummy, 48, 64, 1, 0, pools, outs, None) == -1
    assert bi(dummy, 48, 64, 1, 5, pools, outs, None) == -1
    assert bi(dummy, 0, 64, 1, 3, pools, outs, None) == -1
    assert bi(dummy, 3, 64, 1, 3, pools, outs, None) == -1 and b"bad level" in L.rtg_last_error()   # 3 // 4 == 0 rows
    assert bi(dummy, 48, 64, 1, 3, pools, (C.c_void_p * 3)(16, None, 16), None) == -1 and b"bad level" in L.rtg_last_error()

    lv = (_lib.RtgIcpLevel * 3)()
    for e in lv:
        e.vertex0 = e.normal0 = e.vertex1 = e.normal1 = 16
        e.H, e.W, e.iters = 12, 16, 5
    i0 = (C.c_void_p * 3)(16, 16, 16)
    i1 = (C.c_void_p * 3)(16, 16, 16)
    pp = L.rtg_icp_predict_pose_rgbd

    def call(levels=lv, a=i0, b=i1, n=3, w=0.01, p2p=dummy, out=dummy, ws=dummy):
        return pp(levels, a, b, n, 0.1, 0.94, 1e-4, w, None, p2p, p2p, p2p, 48, 64, out, None, ws, None)

    for kw in (dict(levels=None), dict(a=None), dict(b=None), dict(n=0), dict(n=5), dict(p2p=None), dict(out=None), dict(ws=None)):
        assert call(**kw) == -1, kw
        assert b"rtg_icp_predict_pose_rgbd" in L.rtg_last_error()
    for w in (-1e-3, float("nan"), float("inf")):
        assert call(w=w) == -1 and b"photometric_weight" in L.rtg_last_error(), w
    assert call(a=(C.c_void_p * 3)(16, 16, None)) == -1 and b"bad level" in L.rtg_last_error()
    lv[1].iters = -1
    assert call() == -1 and b"bad level" in L.rtg_last_error()
