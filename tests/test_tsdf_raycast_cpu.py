"""The TSDF ray-cast without a GPU: the float64 statement (tests/tsdf_raycast_oracle.py) against brute-force ray /
triangle intersection with the oracle's own extracted mesh, on analytic grids and on a fused room, with cameras outside
the grid, inside it and behind a wall; the analytic surfaces themselves; and the validation rtg_tsdf_raycast and
TsdfVolume.raycast do before any CUDA work."""
import ctypes as C

import numpy as np
import pytest
import torch

import tsdf_raycast_oracle as RC
from oracle import tsdf_oracle as T
from rtg_slam_b200 import _lib, reconstruct, scene


def _look(eye, at, up=(0.0, 1.0, 0.0)):
    """W2C of a camera at `eye` looking at `at` (+z forward, +y down in the image)."""
    z = np.asarray(at, float) - np.asarray(eye, float)
    z /= np.linalg.norm(z)
    x = np.cross(np.asarray(up, float), z)
    if np.linalg.norm(x) < 1e-6:
        x = np.cross((1.0, 0.0, 0.0), z)
    x /= np.linalg.norm(x)
    c2w = np.eye(4)
    c2w[:3, :3] = np.stack([x, np.cross(z, x), z], 1)
    c2w[:3, 3] = eye
    return np.linalg.inv(c2w)


def _intr(cam):
    return (cam.fx, cam.fy, cam.cx, cam.cy)


def compare_with_mesh(grid, weight, color, origin, s, w2c, cam):
    """Oracle ray-cast against the first triangle of the oracle's mesh along each ray, away from tie pixels."""
    H, W = cam.height, cam.width
    rc = RC.raycast(grid, weight, color, origin, s, w2c, _intr(cam), H, W)
    V, F, Cv = T.extract(grid, weight, color, origin, s)
    o, d = RC.rays(w2c, _intr(cam), H, W)
    rm = RC.ray_mesh(V, F, o, d.T)
    ok = ~rc["tie"].ravel()
    hit = rc["hit"].ravel()
    mesh_hit = (rm["face"] >= 0) & rm["front"]
    assert np.array_equal(hit[ok], mesh_hit[ok]), int((hit[ok] != mesh_hit[ok]).sum())
    extent = s * max(grid.shape)
    h = ok & hit
    assert (rc["depth"].ravel()[~hit] == 0).all() and (rc["normal"].reshape(3, -1)[:, ~hit] == 0).all()
    if not h.any():
        return rc, hit.mean(), rc["tie"].mean()
    assert np.abs(rc["depth"].ravel()[h] - rm["t"][h]).max() <= 1e-9 * extent
    f = F[rm["face"][h]]
    n = np.cross(V[f[:, 1]] - V[f[:, 0]], V[f[:, 2]] - V[f[:, 0]])
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    assert np.abs(rc["normal"].reshape(3, -1)[:, h].T - n).max() < 1e-6
    if color is not None:
        want = np.einsum("rk,rkc->rc", rm["bary"][h], Cv[f])
        assert np.abs(rc["color"].reshape(3, -1)[:, h].T - want).max() < 1e-9
    return rc, hit.mean(), rc["tie"].mean()


def _sphere():
    s, r, c = 0.05, 0.6, np.array([1.01, 0.97, 1.03])
    dims = (42, 41, 40)
    tsdf, w = T.sphere_grid(dims, s, c, r, 5 * s)
    p = T.voxel_centres((0.0, 0.0, 0.0), s, dims)
    col = np.stack([0.5 + 0.4 * np.sin(3 * p[0]), 0.5 + 0.4 * np.cos(2 * p[1]), 0.3 + 0.2 * p[2]])
    return s, r, c, tsdf, w, col


@pytest.mark.parametrize("camname", ["tiny", "ragged"])
@pytest.mark.parametrize("where", ["outside", "inside the grid", "inside the sphere"])
def test_sphere_raycast_is_its_mesh(camname, where):
    s, r, c, tsdf, w, col = _sphere()
    eye = {"outside": (1.31, 0.62, -1.43), "inside the grid": (0.213, 1.79, 0.317), "inside the sphere": (1.113, 1.007, 0.991)}[where]
    w2c = _look(eye, c + (0.05, -0.03, 0.02))
    cam = scene.make_camera(camname)
    rc, frac, ties = compare_with_mesh(tsdf, w, col, (0.0, 0.0, 0.0), s, w2c, cam)
    assert ties < 0.01
    if where == "inside the sphere":
        assert frac == 0                                     # every ray meets the sphere's back faces first
    else:
        assert frac > 0.05
        o, d = RC.rays(w2c, _intr(cam), cam.height, cam.width)
        hit = rc["hit"].ravel()
        p = o[:, None] + rc["depth"].ravel()[hit] * d[:, hit]
        assert np.abs(np.linalg.norm(p - c[:, None], axis=0) - r).max() < s * s / r


@pytest.mark.parametrize("camname", ["tiny", "ragged"])
def test_plane_raycast_is_its_mesh_and_the_plane(camname):
    s, dims = 0.04, (23, 25, 21)
    nrm = np.array([0.3, -0.5, 0.8])
    nrm /= np.linalg.norm(nrm)
    tsdf, w = T.plane_grid(dims, s, nrm, 0.55, 40 * s)     # wide truncation: no corner near the plane is clamped
    cam = scene.make_camera(camname)
    extent = s * max(dims)
    for eye in ((0.603, 0.117, 0.751), (0.91, -0.52, 1.53)):        # on the free side: inside the grid; outside it
        w2c = _look(eye, (0.45, 0.5, 0.6))
        rc, frac, ties = compare_with_mesh(tsdf, w, None, (0.0, 0.0, 0.0), s, w2c, cam)
        assert frac > 0.05 and ties < 0.01
        o, d = RC.rays(w2c, _intr(cam), cam.height, cam.width)
        hit = rc["hit"].ravel()
        p = o[:, None] + rc["depth"].ravel()[hit] * d[:, hit]
        assert np.abs(nrm @ p - 0.55).max() < 1e-9 * extent
        assert np.abs(rc["normal"].reshape(3, -1)[:, hit].T - nrm).max() < 1e-9
    # from the negative side every ray meets the back of the plane: no hit
    rc = RC.raycast(tsdf, w, None, (0.0, 0.0, 0.0), s, _look((0.213, 0.417, 0.109), (0.6, 0.3, 0.7)), _intr(cam), cam.height, cam.width)
    assert not rc["hit"].any()


ROOM_ORIGIN, ROOM_S, ROOM_DIMS, ROOM_TRUNC = (-3.3, -1.8, -3.3), 0.1, (67, 37, 67), 0.3


def _room():
    tsdf, w, col = T.new_volume(ROOM_DIMS, color=True)
    for pose in (scene.small_pose(), scene.small_pose((0.5, 60.0, -1.0), (0.3, 0.1, -0.2)),
                 scene.small_pose((4.0, 180.0, 2.0), (-0.2, -0.1, 0.3))):
        cam = scene.make_camera("small", c2w=pose)
        depth, color = scene.raycast_room_rgbd(cam)
        T.integrate(tsdf, w, col, ROOM_ORIGIN, ROOM_S, ROOM_TRUNC, depth, cam.w2c, _intr(cam), color)
    return tsdf, w, col


@pytest.fixture(scope="module")
def room():
    return _room()


@pytest.mark.parametrize("camname", ["tiny", "ragged"])
@pytest.mark.parametrize("view", ["fusion pose", "novel pose", "behind a wall"])
def test_fused_room_raycast_is_its_mesh(room, camname, view):
    tsdf, w, col = room
    c2w = {"fusion pose": scene.small_pose(), "novel pose": scene.small_pose((3.0, 30.0, 1.0), (0.213, -0.094, 0.127)),
           "behind a wall": np.linalg.inv(_look((0.013, 0.021, 3.157), (0.0, 0.0, 0.0)))}[view]
    cam = scene.make_camera(camname, c2w=c2w)
    rc, frac, ties = compare_with_mesh(tsdf, w, col, ROOM_ORIGIN, ROOM_S, cam.w2c, cam)
    assert ties < 0.01
    if view == "behind a wall":
        assert frac < 0.1        # the wall's back face ends the rays, but where no fusion pose saw the wall
    else:
        assert frac > 0.5


# ------------------------------------------------------------------------------------------------ host validation
def _vol(**over):
    f = dict(nx=4, ny=5, nz=6, voxel_size=0.1, trunc=0.3, origin=(C.c_float * 3)(0, 0, 0), tsdf=8, weight=16, color=None)
    f.update(over)
    return _lib.RtgTsdfVolume(**f)


def test_raycast_rejects_bad_arguments_before_cuda():
    L = _lib.lib()
    v, vc = _vol(), _vol(color=24)

    def call(vol=C.byref(v), w2c=8, H=4, W=4, fx=1.0, fy=1.0, cx=0.0, cy=0.0, depth=8, normal=8, color=None):
        return L.rtg_tsdf_raycast(vol, w2c, 1, H, W, fx, fy, cx, cy, depth, normal, color, None)

    for kw, msg in ((dict(vol=None), b"vol is NULL"), (dict(H=0), b"image size"), (dict(W=-2), b"image size"),
                    (dict(w2c=None), b"NULL pointer"), (dict(depth=None), b"NULL pointer"), (dict(normal=None), b"NULL pointer"),
                    (dict(color=8), b"exactly when the volume has color"), (dict(vol=C.byref(vc)), b"exactly when the volume has color"),
                    (dict(fx=0.0), b"intrinsics"), (dict(fy=float("nan")), b"intrinsics"), (dict(cx=float("inf")), b"intrinsics"),
                    (dict(vol=C.byref(_vol(nx=0))), b"bad dims"), (dict(vol=C.byref(_vol(weight=None))), b"NULL pointer"),
                    (dict(vol=C.byref(_vol(nx=1 << 11, ny=1 << 10, nz=1 << 10))), b"bad dims")):
        assert call(**kw) == -1, kw
        assert msg in L.rtg_last_error() and b"rtg_tsdf_raycast" in L.rtg_last_error(), (kw, L.rtg_last_error())


def test_python_raycast_rejects_bad_inputs_before_cuda():
    vol = reconstruct.TsdfVolume((0, 0, 0), 0.1, (8, 8, 8), 0.3, device="cpu")
    K = (5.0, 5.0, 2.0, 2.5)
    with pytest.raises(TypeError):
        vol.raycast(torch.eye(4, dtype=torch.float64), K, 6, 5)              # not on a CUDA device
    with pytest.raises(TypeError):
        vol.raycast(np.eye(4), K, 6, 5)
    with pytest.raises(TypeError):
        vol.raycast(torch.eye(4, dtype=torch.float16), K, 6, 5)
    with pytest.raises(ValueError):
        vol.raycast(torch.eye(4, dtype=torch.float64), K, 0, 5)
    with pytest.raises(ValueError):
        vol.raycast(torch.eye(4, dtype=torch.float64), K, 6, -1)
