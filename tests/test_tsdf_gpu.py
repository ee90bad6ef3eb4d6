"""TSDF fusion and marching tetrahedra on the device against the float64 oracle (oracle/tsdf_oracle.py), analytic shapes,
determinism, the absence of host synchronisation, an end-to-end fusion of rendered frames of the surfel room, and the
reconstruction metric against scipy's cKDTree."""
import math
import types

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from oracle import tsdf_oracle as T
from rtg_slam_b200 import scene
from rtg_slam_b200.reconstruct import TsdfVolume, reconstruction_metrics, sample_surface

pytestmark = pytest.mark.gpu

ORIGIN, VOXEL, DIMS, TRUNC = (-3.0, -1.5, -3.0), 0.02, (301, 151, 301), 0.08


def _frames():
    """Four noise-free textured frames: replica and ragged cameras at small_pose offsets from identity."""
    out = []
    for name, pose in (("replica", scene.small_pose()), ("ragged", scene.small_pose((-2.0, 3.0, 1.0), (0.1, 0.05, -0.2))),
                       ("replica", scene.small_pose((0.5, 25.0, -1.0), (-0.3, 0.1, 0.4))),
                       ("ragged", scene.small_pose((4.0, -40.0, 2.0), (0.2, -0.1, 0.3)))):
        cam = scene.make_camera(name, c2w=pose)
        depth, color = scene.raycast_room_rgbd(cam)
        out.append((cam, depth, color))
    return out


def _fuse(dev, frames, pose_dtype, vol=None):
    vol = vol or TsdfVolume(ORIGIN, VOXEL, DIMS, TRUNC, color=True, device=dev)
    for n, (cam, depth, color) in enumerate(frames):
        w2c = torch.from_numpy(np.linalg.inv(cam.c2w)).to(dev, pose_dtype)
        c = torch.from_numpy(color).to(dev)
        cl = n % 2 == 0                                        # both colour layouts
        vol.integrate(torch.from_numpy(depth).to(dev)[None], w2c, (cam.fx, cam.fy, cam.cx, cam.cy),
                      color=c if cl else c.permute(2, 0, 1).contiguous(), color_channels_last=cl)
    return vol


def _oracle(frames, pose_dtype):
    tsdf, w, col = T.new_volume(DIMS, color=True)
    tie = np.zeros(tsdf.shape, bool)
    for cam, depth, color in frames:
        w2c = np.linalg.inv(cam.c2w).astype(np.float32 if pose_dtype == torch.float32 else np.float64)
        tie |= T.integrate(tsdf, w, col, ORIGIN, VOXEL, TRUNC, depth, w2c, (cam.fx, cam.fy, cam.cx, cam.cy), color)
    return tsdf, w, col, tie


@pytest.fixture(scope="module")
def frames():
    return _frames()


@pytest.fixture(scope="module")
def fused(cuda_device, frames):
    return _fuse(cuda_device, frames, torch.float64)


@pytest.mark.parametrize("pose_dtype", [torch.float64, torch.float32])
def test_integration_matches_the_oracle(cuda_device, frames, fused, pose_dtype):
    vol = fused if pose_dtype == torch.float64 else _fuse(cuda_device, frames, pose_dtype)
    tsdf, w, col, tie = _oracle(frames, pose_dtype)
    ok = ~tie
    # a 2e-3 px band per axis and frame flags about 1.6 % of the voxels in view; the rest must match exactly
    assert tie.mean() < 0.02 and (w[ok] > 0).sum() > 1_000_000
    gw, gt, gc = vol.weight.cpu().numpy(), vol.tsdf.cpu().numpy(), vol.color.cpu().numpy()
    assert np.array_equal(gw[ok], w[ok])
    assert np.abs(gt[ok] - tsdf[ok]).max() <= 1e-5
    assert np.abs(gc[:, ok] - col[:, ok]).max() <= 1e-5
    assert gw.max() == 4


def test_extraction_matches_the_oracle(fused):
    mesh = fused.extract_mesh()
    V, F, Cv = (mesh[k].cpu().numpy() for k in ("vertices", "faces", "colors"))
    OV, OF, OC = T.extract(fused.tsdf.cpu().numpy(), fused.weight.cpu().numpy(), fused.color.cpu().numpy(), ORIGIN, VOXEL)
    assert len(OF) > 100_000 and mesh["faces"].dtype == torch.int32
    assert np.array_equal(F, OF)
    assert np.abs(V - OV).max() <= 1e-6 * np.abs(OV).max()
    assert np.abs(Cv - OC).max() <= 1e-6 * np.abs(OC).max()


def test_repeats_are_bit_identical(cuda_device, frames, fused):
    again = _fuse(cuda_device, frames, torch.float64)
    for a, b in ((fused.tsdf, again.tsdf), (fused.weight, again.weight), (fused.color, again.color)):
        assert torch.equal(a, b)
    m1, m2 = fused.extract_mesh(), fused.extract_mesh()
    for k in ("vertices", "faces", "colors"):
        assert torch.equal(m1[k], m2[k])


def test_integrate_does_not_synchronise(cuda_device, frames):
    cam, depth, color = frames[0]
    vol = TsdfVolume(ORIGIN, 0.05, (121, 61, 121), 0.15, color=True, device=cuda_device)
    d = torch.from_numpy(depth).to(cuda_device)
    c = torch.from_numpy(color).to(cuda_device)
    w2c = torch.from_numpy(np.linalg.inv(cam.c2w)).to(cuda_device)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        vol.integrate(d, w2c, (cam.fx, cam.fy, cam.cx, cam.cy), color=c, color_channels_last=True)
        vol.integrate(d, w2c.float(), (cam.fx, cam.fy, cam.cx, cam.cy), color=c, color_channels_last=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert float(vol.weight.max()) == 2


def _analytic(dev, grid, dims, s):
    vol = TsdfVolume((0.0, 0.0, 0.0), s, dims, 1.0, device=dev)
    vol.tsdf.copy_(torch.from_numpy(grid[0]))
    vol.weight.copy_(torch.from_numpy(grid[1]))
    m = vol.extract_mesh()
    return m["vertices"].cpu().numpy().astype(np.float64), m["faces"].cpu().numpy()


def test_sphere_on_the_device(cuda_device):
    s, r, c = 0.05, 0.6, np.array([1.01, 0.97, 1.03])
    dims = (42, 41, 40)
    V, F = _analytic(cuda_device, T.sphere_grid(dims, s, c, r, 5 * s), dims, s)
    e = np.sort(np.concatenate([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]]), axis=1)
    e, cnt = np.unique(e, axis=0, return_counts=True)
    assert len(F) > 1000 and (cnt == 2).all() and len(V) - len(e) + len(F) == 2
    n = np.cross(V[F[:, 1]] - V[F[:, 0]], V[F[:, 2]] - V[F[:, 0]])
    assert (np.einsum("ij,ij->i", n, V[F].mean(1) - c) > 0).all()
    assert np.abs(np.linalg.norm(V - c, axis=1) - r).max() < s * s / r


def test_tilted_plane_on_the_device(cuda_device):
    s, dims = 0.04, (23, 25, 21)
    nrm = np.array([0.3, -0.5, 0.8])
    nrm /= np.linalg.norm(nrm)
    V, F = _analytic(cuda_device, T.plane_grid(dims, s, nrm, 0.55, 4 * s), dims, s)
    extent = s * max(dims)
    assert len(F) > 100 and np.abs(V @ nrm - 0.55).max() < 1e-6 * extent   # float32 rounding of world coordinates
    n = np.cross(V[F[:, 1]] - V[F[:, 0]], V[F[:, 2]] - V[F[:, 0]])
    assert (n @ nrm > 0).all()


# ------------------------------------------------------------------------------------------------ end to end
ROOM = np.array([6.0, 3.0, 6.0])


def _box_distance(p):
    """Distance of points p (N,3) to the surface of the room's box."""
    q = np.abs(p) - ROOM / 2
    return np.abs(np.linalg.norm(np.maximum(q, 0), axis=1) + np.minimum(q.max(1), 0))


def _look(d, at=(0.1, -0.05, 0.08)):
    z = np.asarray(d, float)
    x = np.array([1.0, 0, 0]) if abs(z[0]) < 0.9 else np.array([0, 0, 1.0])
    x = x - z * (x @ z)
    x /= np.linalg.norm(x)
    c2w = np.eye(4)
    c2w[:3, :3] = np.stack([x, np.cross(z, x), z], 1)
    c2w[:3, 3] = at
    return c2w


def test_fused_render_of_the_room_lies_on_its_walls(cuda_device):
    """Six renders of surfel_room(n_patches=0) from inside the room, fused at 4 cm. Bound: the oracle fused from the same
    rendered frames gives a mesh whose farthest vertex lies d_o from the box faces (surfel thickness, normal jitter and the
    room's corners, where the truncation band of two walls meets). The device mesh differs from the oracle's only at tie
    voxels, where one observation more or less moves a zero crossing at most along its edge, up to sqrt(3) s. So the device
    mesh must stay within d_o + sqrt(3) s, and its median distance, which the ties do not move, within s / 4."""
    from rtg_slam_b200.render import Renderer
    dev = cuda_device
    g = scene.surfel_room(400_000, seed=5, n_patches=0)
    data = {k: torch.from_numpy(v).to(dev) for k, v in g.items()}
    args = types.SimpleNamespace(renderer_opaque_threshold=0.6, renderer_normal_threshold=60, renderer_depth_threshold=1.0,
                                 max_sh_degree=3, color_sigma=3.0, active_sh_degree=3)
    s, origin, dims, trunc = 0.04, (-3.12, -1.62, -3.12), (157, 82, 157), 0.12
    vol = TsdfVolume(origin, s, dims, trunc, device=dev)
    otsdf, ow, _ = T.new_volume(dims)
    for d in ((1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)):
        cam = scene.make_camera("tum", c2w=_look(d))
        vc = types.SimpleNamespace(FoVx=2 * math.atan(cam.tanfovx), FoVy=2 * math.atan(cam.tanfovy), image_height=cam.height,
                                   image_width=cam.width, world_view_transform=torch.from_numpy(cam.viewmatrix).to(dev),
                                   full_proj_transform=torch.from_numpy(cam.projmatrix).to(dev),
                                   camera_center=torch.from_numpy(cam.campos).to(dev), cx=cam.cx, cy=cam.cy)
        depth = Renderer(args).render(vc, data)["depth"].detach()
        w2c = torch.from_numpy(cam.w2c).to(dev)
        K = (cam.fx, cam.fy, cam.cx, cam.cy)
        vol.integrate(depth, w2c, K)
        T.integrate(otsdf, ow, None, origin, s, trunc, depth.cpu().numpy(), cam.w2c, K)
    V = vol.extract_mesh()["vertices"].cpu().numpy().astype(np.float64)
    OV, _, _ = T.extract(otsdf, ow, None, origin, s)
    d_o = _box_distance(OV).max()
    dist = _box_distance(V)
    assert len(V) > 50_000
    assert dist.max() <= d_o + math.sqrt(3) * s, (dist.max(), d_o)
    assert np.median(dist) < s / 4, np.median(dist)


# ------------------------------------------------------------------------------------------------ the metric
def test_metrics_match_ckdtree_with_points_outside_the_ground_truth(cuda_device):
    rng = np.random.default_rng(9)
    gt = rng.uniform(-1, 1, (40_000, 3)).astype(np.float32) * np.float32([1.0, 0.5, 1.0])
    rec = np.concatenate([gt[:20_000] + rng.normal(0, 0.02, (20_000, 3)),
                          rng.uniform(-3, 3, (5_000, 3)) * [1, 1, 1] + [0, 2.5, 0]]).astype(np.float32)
    assert (rec[:, 1] > gt[:, 1].max()).sum() > 2000                      # queries the kNN grid has to clamp
    dev = cuda_device
    rt, gtt = torch.from_numpy(rec).to(dev), torch.from_numpy(gt).to(dev)
    from rtg_slam_b200 import mapsurgery
    d2 = mapsurgery.knn(rt, gtt, 1)[0][:, 0].cpu().numpy().astype(np.float64)
    want_acc = cKDTree(gt.astype(np.float64)).query(rec.astype(np.float64))[0]
    assert np.allclose(d2, want_acc ** 2, rtol=1e-5, atol=1e-10)           # exact nearest neighbours, clamped queries included
    want_comp = cKDTree(rec.astype(np.float64)).query(gt.astype(np.float64))[0]
    m = reconstruction_metrics(rt, gtt, thresholds=(0.03, 0.05))
    assert m["accuracy"] == pytest.approx(want_acc.mean() * 100, rel=1e-5)
    assert m["completion"] == pytest.approx(want_comp.mean() * 100, rel=1e-5)
    for t in (0.03, 0.05):
        P, R = (want_acc < t).mean() * 100, (want_comp < t).mean() * 100
        assert m[f"P (< {t})"] == pytest.approx(P, abs=100 / len(rec) + 1e-9)
        assert m[f"R (< {t})"] == pytest.approx(R, abs=100 / len(gt) + 1e-9)
        assert m[f"F1 (< {t})"] == pytest.approx(2 * P * R / (P + R), rel=1e-3)
    assert list(m) == ["accuracy", "completion", "P (< 0.03)", "P (< 0.05)", "R (< 0.03)", "R (< 0.05)", "F1 (< 0.03)",
                       "F1 (< 0.05)"]


def test_sample_surface_follows_the_face_areas(cuda_device):
    rng = np.random.default_rng(3)
    tris = []
    for k in range(5):                                                    # one triangle per plane z = k, areas spread 1..100
        a = rng.uniform(-1, 1, 2)
        e1, e2 = rng.normal(size=2), rng.normal(size=2)
        scale = math.sqrt(10.0 ** (k / 2)) / math.sqrt(abs(e1[0] * e2[1] - e1[1] * e2[0]))
        tris.append([[*a, k], [*(a + scale * e1), k], [*(a + scale * e2), k]])
    V = np.array(tris, np.float32).reshape(-1, 3)
    F = np.arange(15, dtype=np.int32).reshape(5, 3)
    area = np.array([0.5 * abs(np.cross(t[1] - t[0], t[2] - t[0])[2]) for t in V.reshape(5, 3, 3).astype(np.float64)])
    n = 1_000_000
    pts = sample_surface(torch.from_numpy(V).to(cuda_device), torch.from_numpy(F).to(cuda_device), n, seed=1).cpu().numpy()
    face = np.rint(pts[:, 2]).astype(int)
    frac = np.bincount(face, minlength=5) / n
    p = area / area.sum()
    assert np.all(np.abs(frac - p) < 5 * np.sqrt(p * (1 - p) / n))
    for k in range(5):                                                    # every point inside its triangle
        t = V[3 * k: 3 * k + 3].astype(np.float64)
        q = pts[face == k].astype(np.float64)
        M = np.stack([t[1, :2] - t[0, :2], t[2, :2] - t[0, :2]], 1)
        uv = np.linalg.solve(M, (q[:, :2] - t[0, :2]).T).T
        assert uv.min() > -1e-4 and (uv.sum(1)).max() < 1 + 1e-4
    again = sample_surface(torch.from_numpy(V).to(cuda_device), torch.from_numpy(F).to(cuda_device), n, seed=1).cpu().numpy()
    assert np.array_equal(pts, again)


def test_python_argument_errors(cuda_device):
    dev = cuda_device
    vol = TsdfVolume((0, 0, 0), 0.1, (8, 8, 8), 0.3, device=dev)
    d = torch.ones((6, 5), device=dev)
    w2c = torch.eye(4, dtype=torch.float64, device=dev)
    K = (5.0, 5.0, 2.0, 2.5)
    with pytest.raises(TypeError):
        vol.integrate(d.cpu(), w2c, K)
    with pytest.raises(TypeError):
        vol.integrate(d.double(), w2c, K)
    with pytest.raises(TypeError):
        vol.integrate(d, w2c.cpu(), K)
    with pytest.raises(ValueError):
        vol.integrate(torch.ones((2, 6, 5), device=dev), w2c, K)
    with pytest.raises(ValueError):
        vol.integrate(d, w2c[:3], K)
    with pytest.raises(ValueError):
        vol.integrate(d, w2c, K, color=torch.ones((3, 6, 5), device=dev))    # the volume has no colour
    cvol = TsdfVolume((0, 0, 0), 0.1, (8, 8, 8), 0.3, color=True, device=dev)
    with pytest.raises(ValueError):
        cvol.integrate(d, w2c, K)
    with pytest.raises(ValueError):
        cvol.integrate(d, w2c, K, color=torch.ones((3, 6, 5), device=dev), color_channels_last=True)
    with pytest.raises(TypeError):
        cvol.integrate(d, w2c, K, color=torch.ones((3, 6, 5), device=dev, dtype=torch.float16))
    assert float(vol.weight.sum()) == 0 and float(cvol.weight.sum()) == 0
    with pytest.raises(TypeError):
        reconstruction_metrics(torch.zeros((4, 3), device=dev, dtype=torch.float64), torch.zeros((4, 3), device=dev))
    with pytest.raises(ValueError):
        reconstruction_metrics(torch.zeros((4, 2), device=dev), torch.zeros((4, 3), device=dev))
