"""The TSDF ray-cast on the device: parity with the float64 statement (tests/tsdf_raycast_oracle.py) on a fused room,
agreement with the device mesh of analytic grids, determinism and the absence of host synchronisation, an end-to-end
ray-cast of fused Gaussian renders, and frame-to-model ICP tracking against the ray-cast (one pair, and a KinectFusion
loop of track, fuse and ray-cast)."""
import math
import types

import numpy as np
import pytest
import torch

import tsdf_raycast_oracle as RC
from oracle import tsdf_oracle as T
from rtg_slam_b200 import _lib, scene
from rtg_slam_b200.reconstruct import TsdfVolume

pytestmark = pytest.mark.gpu

# the 2 cm room grid, shifted by a fraction of a voxel: the fourth fusion pose sits on a voxel of the unshifted grid, and
# rays from a lattice point cross its cells at their corners, so a tenth of its pixels would be ties
ORIGIN, VOXEL, DIMS, TRUNC = (-3.0074, -1.5053, -3.0031), 0.02, (302, 152, 302), 0.08
FUSION_POSES = (scene.small_pose(), scene.small_pose((-2.0, 3.0, 1.0), (0.1, 0.05, -0.2)),
                scene.small_pose((0.5, 25.0, -1.0), (-0.3, 0.1, 0.4)), scene.small_pose((4.0, -40.0, 2.0), (0.2, -0.1, 0.3)))
NOVEL_POSES = (scene.small_pose((2.0, 15.0, -1.5), (0.317, 0.071, -0.233)),     # inside the span the fusion poses saw
               scene.small_pose((-3.0, -20.0, 2.0), (-0.271, 0.113, 0.191)))


def _K(cam):
    return (cam.fx, cam.fy, cam.cx, cam.cy)


def _frames():
    """Four noise-free textured frames: replica and ragged cameras at small_pose offsets from identity."""
    out = []
    for name, pose in zip(("replica", "ragged", "replica", "ragged"), FUSION_POSES):
        cam = scene.make_camera(name, c2w=pose)
        depth, color = scene.raycast_room_rgbd(cam)
        out.append((cam, depth, color))
    return out


@pytest.fixture(scope="module")
def fused(cuda_device):
    vol = TsdfVolume(ORIGIN, VOXEL, DIMS, TRUNC, color=True, device=cuda_device)
    for cam, depth, color in _frames():
        vol.integrate(torch.from_numpy(depth).to(cuda_device), torch.from_numpy(cam.w2c).to(cuda_device), _K(cam),
                      color=torch.from_numpy(color).to(cuda_device), color_channels_last=True)
    return vol


@pytest.fixture(scope="module")
def fused_np(fused):
    return fused.tsdf.cpu().numpy(), fused.weight.cpu().numpy(), fused.color.cpu().numpy()


@pytest.mark.parametrize("pose_dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("camname", ["small", "ragged", "tum"])
def test_raycast_matches_the_oracle(cuda_device, fused, fused_np, camname, pose_dtype):
    tsdf, w, col = fused_np
    npd = np.float64 if pose_dtype == torch.float64 else np.float32
    for n, c2w in enumerate(FUSION_POSES + NOVEL_POSES):
        cam = scene.make_camera(camname, c2w=c2w)
        H, W = cam.height, cam.width
        w2c = np.linalg.inv(c2w).astype(npd)
        out = fused.raycast(torch.from_numpy(w2c).to(cuda_device), _K(cam), H, W)
        ref = RC.raycast(tsdf, w, col, ORIGIN, VOXEL, w2c, _K(cam), H, W)
        ok = ~ref["tie"]
        assert ref["tie"].mean() < 0.01 and ref["hit"].mean() > 0.3, (n, ref["tie"].mean(), ref["hit"].mean())
        depth, normal, color = (out[k].cpu().numpy().astype(np.float64) for k in ("depth", "normal", "color"))
        assert np.array_equal((depth > 0)[ok], ref["hit"][ok]), (n, int(((depth > 0) != ref["hit"])[ok].sum()))
        h = ok & ref["hit"]
        assert np.abs(depth[h] - ref["depth"][h]).max() <= 2e-6 * ref["depth"][h].max(), n
        assert np.abs(normal[:, h] - ref["normal"][:, h]).max() <= 1e-6, n
        assert np.abs(color[:, h] - ref["color"][:, h]).max() <= 1e-6, n
        miss = ~(depth > 0)
        assert (normal[:, miss] == 0).all() and (color[:, miss] == 0).all()


def _analytic(dev, grid, dims, s):
    vol = TsdfVolume((0.0, 0.0, 0.0), s, dims, 1.0, device=dev)
    vol.tsdf.copy_(torch.from_numpy(grid[0]))
    vol.weight.copy_(torch.from_numpy(grid[1]))
    return vol


def _hits_agree_with_device_mesh(vol, s, w2c, cam):
    """Device ray-cast against the first triangle of the device mesh (float32 vertices) along each ray, away from the
    oracle's ties on the same grid; returns the world hit points."""
    dev = vol.device
    H, W = cam.height, cam.width
    out = vol.raycast(torch.from_numpy(w2c).to(dev), _K(cam), H, W)
    depth = out["depth"].cpu().numpy().astype(np.float64).ravel()
    tsdf, wgt = vol.tsdf.cpu().numpy(), vol.weight.cpu().numpy()
    # the mesh's float32 vertices move its triangle edges by ~1e-6 voxels: a wider band of ties at tetrahedron boundaries
    ref = RC.raycast(tsdf, wgt, None, (0.0, 0.0, 0.0), s, w2c, _K(cam), H, W, tie_u=1e-5)
    mesh = vol.extract_mesh()
    o, d = RC.rays(w2c, _K(cam), H, W)
    rm = RC.ray_mesh(mesh["vertices"].cpu().numpy(), mesh["faces"].cpu().numpy(), o, d.T)
    ok = ~ref["tie"].ravel()
    hit = depth > 0
    assert ref["tie"].mean() < 0.01 and hit.mean() > 0.05
    assert np.array_equal(hit[ok], ((rm["face"] >= 0) & rm["front"])[ok])
    extent = s * max(tsdf.shape)
    h = ok & hit
    # float32 rounding moves a mesh vertex by up to ~1e-7 of the extent, the triangle along its normal; a ray meeting it
    # at incidence theta sees that displacement divided by cos(theta) (2.3e-6 of the extent on the sphere's rim)
    V, F = mesh["vertices"].cpu().numpy().astype(np.float64), mesh["faces"].cpu().numpy()
    f = F[rm["face"][h]]
    n = np.cross(V[f[:, 1]] - V[f[:, 0]], V[f[:, 2]] - V[f[:, 0]])
    cos = np.abs((n * d[:, h].T).sum(1)) / (np.linalg.norm(n, axis=1) * np.linalg.norm(d[:, h], axis=0))
    assert (np.abs(depth[h] - rm["t"][h]) * cos).max() <= 1e-6 * extent
    return o[:, None] + depth[hit] * d[:, hit], out["normal"].cpu().numpy().reshape(3, -1)[:, hit]


def _look(eye, at):
    z = np.asarray(at, float) - np.asarray(eye, float)
    z /= np.linalg.norm(z)
    x = np.cross((0.0, 1.0, 0.0), z)
    x /= np.linalg.norm(x)
    c2w = np.eye(4)
    c2w[:3, :3] = np.stack([x, np.cross(z, x), z], 1)
    c2w[:3, 3] = eye
    return c2w


def test_sphere_raycast_on_the_device(cuda_device):
    s, r, c = 0.05, 0.6, np.array([1.01, 0.97, 1.03])
    dims = (42, 41, 40)
    vol = _analytic(cuda_device, T.sphere_grid(dims, s, c, r, 5 * s), dims, s)
    for eye in ((1.31, 0.62, -1.43), (0.213, 1.79, 0.317)):
        cam = scene.make_camera("small")
        p, _ = _hits_agree_with_device_mesh(vol, s, np.linalg.inv(_look(eye, c + (0.05, -0.03, 0.02))), cam)
        assert np.abs(np.linalg.norm(p - c[:, None], axis=0) - r).max() < s * s / r


def test_tilted_plane_raycast_on_the_device(cuda_device):
    s, dims = 0.04, (23, 25, 21)
    nrm = np.array([0.3, -0.5, 0.8])
    nrm /= np.linalg.norm(nrm)
    vol = _analytic(cuda_device, T.plane_grid(dims, s, nrm, 0.55, 40 * s), dims, s)
    extent = s * max(dims)
    for eye in ((0.603, 0.117, 0.751), (0.91, -0.52, 1.53)):
        cam = scene.make_camera("small")
        p, n = _hits_agree_with_device_mesh(vol, s, np.linalg.inv(_look(eye, (0.45, 0.5, 0.6))), cam)
        assert np.abs(nrm @ p - 0.55).max() < 1e-6 * extent      # float32 grid values and outputs
        assert np.abs(n.T - nrm).max() < 1e-6


def test_raycast_is_deterministic_and_does_not_synchronise(cuda_device, fused):
    cam = scene.make_camera("replica", c2w=NOVEL_POSES[0])
    w2c = torch.from_numpy(cam.w2c).to(cuda_device)
    a = fused.raycast(w2c, _K(cam), cam.height, cam.width)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = fused.raycast(w2c, _K(cam), cam.height, cam.width)
        c = fused.raycast(w2c.float(), _K(cam), cam.height, cam.width)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for k in ("depth", "normal", "color"):
        assert torch.equal(a[k], b[k])
    assert float((a["depth"] > 0).float().mean()) > 0.5 and float((c["depth"] > 0).float().mean()) > 0.5


def test_python_raycast_rejects_bad_inputs(cuda_device):
    dev = cuda_device
    vol = TsdfVolume((0, 0, 0), 0.1, (8, 8, 8), 0.3, device=dev)
    w2c = torch.eye(4, dtype=torch.float64, device=dev)
    K = (5.0, 5.0, 2.0, 2.5)
    with pytest.raises(ValueError):
        vol.raycast(w2c[:3], K, 6, 5)
    with pytest.raises(TypeError):
        vol.raycast(w2c.half(), K, 6, 5)
    with pytest.raises(TypeError):
        vol.raycast(w2c.cpu(), K, 6, 5)
    with pytest.raises(ValueError):
        vol.raycast(w2c, K, 0, 5)
    with pytest.raises(_lib.RtgError):
        vol.raycast(w2c, (0.0, 5.0, 2.0, 2.5), 6, 5)
    with pytest.raises(_lib.RtgError):
        vol.raycast(w2c, (5.0, float("nan"), 2.0, 2.5), 6, 5)
    out = vol.raycast(w2c, K, 6, 5)
    assert out["color"] is None and tuple(out["depth"].shape) == (6, 5) and tuple(out["normal"].shape) == (3, 6, 5)


# ------------------------------------------------------------------------------------------------ end to end
ROOM = np.array([6.0, 3.0, 6.0])


def _box_distance(p):
    """Distance of points p (N,3) to the surface of the room's box."""
    q = np.abs(p) - ROOM / 2
    return np.abs(np.linalg.norm(np.maximum(q, 0), axis=1) + np.minimum(q.max(1), 0))


def _look_dir(d, at=(0.1, -0.05, 0.08)):
    z = np.asarray(d, float)
    x = np.array([1.0, 0, 0]) if abs(z[0]) < 0.9 else np.array([0, 0, 1.0])
    x = x - z * (x @ z)
    x /= np.linalg.norm(x)
    c2w = np.eye(4)
    c2w[:3, :3] = np.stack([x, np.cross(z, x), z], 1)
    c2w[:3, 3] = at
    return c2w


def test_raycast_of_fused_renders_lies_on_the_walls(cuda_device):
    """The six renders of surfel_room(n_patches=0) that test_tsdf_gpu fuses at 4 cm, ray-cast from the same six poses.
    The hits lie on the device mesh's triangles, so the mesh's bound carries over: within d_o + sqrt(3) s of the box, d_o
    the farthest vertex of the oracle's mesh of the same frames, and a median distance under s / 4."""
    from rtg_slam_b200.render import Renderer
    dev = cuda_device
    g = scene.surfel_room(400_000, seed=5, n_patches=0)
    data = {k: torch.from_numpy(v).to(dev) for k, v in g.items()}
    args = types.SimpleNamespace(renderer_opaque_threshold=0.6, renderer_normal_threshold=60, renderer_depth_threshold=1.0,
                                 max_sh_degree=3, color_sigma=3.0, active_sh_degree=3)
    s, origin, dims, trunc = 0.04, (-3.12, -1.62, -3.12), (157, 82, 157), 0.12
    vol = TsdfVolume(origin, s, dims, trunc, device=dev)
    otsdf, ow, _ = T.new_volume(dims)
    cams = []
    for d in ((1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)):
        cam = scene.make_camera("tum", c2w=_look_dir(d))
        vc = types.SimpleNamespace(FoVx=2 * math.atan(cam.tanfovx), FoVy=2 * math.atan(cam.tanfovy), image_height=cam.height,
                                   image_width=cam.width, world_view_transform=torch.from_numpy(cam.viewmatrix).to(dev),
                                   full_proj_transform=torch.from_numpy(cam.projmatrix).to(dev),
                                   camera_center=torch.from_numpy(cam.campos).to(dev), cx=cam.cx, cy=cam.cy)
        depth = Renderer(args).render(vc, data)["depth"].detach()
        vol.integrate(depth, torch.from_numpy(cam.w2c).to(dev), _K(cam))
        T.integrate(otsdf, ow, None, origin, s, trunc, depth.cpu().numpy(), cam.w2c, _K(cam))
        cams.append(cam)
    OV, _, _ = T.extract(otsdf, ow, None, origin, s)
    d_o = _box_distance(OV).max()
    pts = []
    for cam in cams:
        out = vol.raycast(torch.from_numpy(cam.w2c).to(dev), _K(cam), cam.height, cam.width)
        depth = out["depth"].cpu().numpy().astype(np.float64).ravel()
        o, d = RC.rays(cam.w2c, _K(cam), cam.height, cam.width)
        hit = depth > 0
        assert hit.mean() > 0.5
        pts.append((o[:, None] + depth[hit] * d[:, hit]).T)
    dist = _box_distance(np.concatenate(pts))
    assert dist.max() <= d_o + math.sqrt(3) * s, (dist.max(), d_o)
    assert np.median(dist) < s / 4, np.median(dist)


# ------------------------------------------------------------------------------------------------ tracking
def _tracker(use_model_depth):
    from rtg_slam_b200 import icp as ricp
    return ricp.IcpTracker(types.SimpleNamespace(
        icp_downscales=[0.25, 0.5, 1.0], icp_warmup_frames=0, icp_use_model_depth=use_model_depth, icp_downscale_iters=[5, 5, 5],
        icp_distance_threshold=0.1, icp_normal_threshold=20, icp_damping=1e-4, verbose=False,
        icp_sample_distance_threshold=0.01, icp_sample_normal_threshold=0.01, icp_fail_threshold=0.02))


def _world(normal_cam, c2w):
    """(H, W, 3) camera-space normals to world space."""
    R = torch.as_tensor(c2w[:3, :3], dtype=torch.float32, device=normal_cam.device)
    return (normal_cam @ R.T).contiguous()


def _pose_error(a, b):
    """(translation m, rotation degrees) of a^-1 b."""
    d = np.linalg.inv(np.asarray(a, np.float64)) @ np.asarray(b, np.float64)
    R = d[:3, :3]
    ang = math.degrees(math.atan2(np.linalg.norm([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]]), np.trace(R) - 1))
    return float(np.linalg.norm(d[:3, 3])), ang


def _track_pair(dev, model_depth, model_normal, frame0, frame0_normal, frame1, cam):
    trk = _tracker(True)
    Kt = torch.from_numpy(cam.K)
    trk.update_curr_status(frame0, Kt)
    trk.move_last_status()
    trk.update_last_status(None, model_depth[..., None].contiguous().clone(), frame0[..., None], model_normal, frame0_normal)
    trk.update_curr_status(frame1, Kt)
    pose, ok = trk.predict_pose({"K": Kt, "frame_id": 1})
    return pose.astype(np.float64)


def test_tracking_against_the_raycast_model(cuda_device, fused):
    """One frame tracked against the ray-cast of the fused room at the previous frame's pose, against the same frame
    tracked against the exact model depth at that pose. Bound: 1 mm and 0.05 degrees."""
    from rtg_slam_b200 import icp as ricp
    dev = cuda_device
    cam0 = scene.make_camera("replica", c2w=FUSION_POSES[0])
    cam1 = scene.make_camera("replica", c2w=FUSION_POSES[0] @ scene.small_pose())
    d0 = torch.from_numpy(scene.raycast_room_depth(cam0)).to(dev)
    d1 = torch.from_numpy(scene.raycast_room_depth(cam1)).to(dev)
    n0 = _world(ricp.build_pyramids(d0, _K(cam0), 1)[1][0], cam0.c2w)
    rc = fused.raycast(torch.from_numpy(cam0.w2c).to(dev), _K(cam0), cam0.height, cam0.width)
    pose_rc = _track_pair(dev, rc["depth"], rc["normal"].permute(1, 2, 0), d0, n0, d1, cam0)
    exact = torch.from_numpy(scene.raycast_room_depth(cam0)).to(dev)
    pose_ex = _track_pair(dev, exact, n0, d0, n0, d1, cam0)
    dt, dr = _pose_error(pose_ex, pose_rc)
    gt_t, gt_r = _pose_error(scene.small_pose(), pose_rc)
    print(f"\n[raycast tracking] pair: vs exact model {dt * 1e3:.4f} mm {dr:.5f} deg; vs ground truth {gt_t * 1e3:.4f} mm {gt_r:.5f} deg")
    assert dt <= 1e-3 and dr <= 0.05


def _loop(dev, mode, cam_name="tum", n=10):
    """Tracks n frames with 2 mm noise from the true first pose; mode "tsdf": against the ray-cast of a volume that fuses
    each frame at its tracked pose; "exact": against the noise-free room depth at the tracked pose; "frame": against the
    previous frame. Returns the final translation drift (m) and the final pose error."""
    from rtg_slam_b200 import icp as ricp
    gt = [scene.small_pose((1.0 * k, -1.5 * k, 0.5 * k), (0.02 * k, -0.01 * k, 0.015 * k)) for k in range(n)]
    cams = [scene.make_camera(cam_name, c2w=p) for p in gt]
    depths = [torch.from_numpy(scene.raycast_room_depth(c, noise_sigma=0.002, seed=20 + k)).to(dev) for k, c in enumerate(cams)]
    K, Kt = _K(cams[0]), torch.from_numpy(cams[0].K)
    H, W = cams[0].height, cams[0].width
    vol = TsdfVolume(ORIGIN, VOXEL, DIMS, TRUNC, device=dev) if mode == "tsdf" else None
    P = gt[0].copy()
    if vol is not None:
        vol.integrate(depths[0], torch.from_numpy(np.linalg.inv(P)).to(dev), K)
    trk = _tracker(mode != "frame")
    trk.update_curr_status(depths[0], Kt)
    for k in range(1, n):
        trk.move_last_status()
        if mode == "tsdf":
            rc = vol.raycast(torch.from_numpy(np.linalg.inv(P)).to(dev), K, H, W)
            trk.update_last_status(None, rc["depth"][..., None].contiguous(), depths[k - 1][..., None], rc["normal"].permute(1, 2, 0),
                                   _world(trk.normal_pyramid_t0[-1], P))
        elif mode == "exact":
            model = torch.from_numpy(scene.raycast_room_depth(scene.make_camera(cam_name, c2w=P))).to(dev)
            nm = ricp.build_pyramids(model, K, 1)[1][0]
            trk.update_last_status(None, model[..., None].contiguous(), depths[k - 1][..., None], nm, trk.normal_pyramid_t0[-1])
        trk.update_curr_status(depths[k], Kt)
        rel, ok = trk.predict_pose({"K": Kt, "frame_id": k})
        P = P @ rel.astype(np.float64)
        if vol is not None:
            vol.integrate(depths[k], torch.from_numpy(np.linalg.inv(P)).to(dev), K)
    return float(np.linalg.norm(P[:3, 3] - gt[-1][:3, 3])), _pose_error(gt[-1], P)[1]


def test_kinectfusion_loop_drift(cuda_device):
    """Ten frames, 2 mm noise: track against the ray-cast, fuse at the tracked pose, ray-cast there as the next model.
    Bound on the final drift: 1 cm. Frame-to-frame tracking and the loop against the exact model are reported beside it."""
    drift, ang = _loop(cuda_device, "tsdf")
    other = {m: _loop(cuda_device, m) for m in ("frame", "exact")}
    print(f"\n[raycast tracking] loop drift after 10 frames: tsdf model {drift * 1e3:.3f} mm {ang:.4f} deg; "
          + "; ".join(f"{m} {d * 1e3:.3f} mm {a:.4f} deg" for m, (d, a) in other.items()))
    assert drift < 0.01
