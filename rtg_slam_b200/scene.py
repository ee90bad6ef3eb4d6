"""Synthetic "surfel room" scenes and cameras for parity tests and benchmarks.

This is workload generation only (numpy, host side). It follows the inputs the
reference's hot path consumes:

* camera matrices as `scene/cameras.py:96-110` builds them (W2C stored
  transposed, `full_proj = view^T-form @ proj^T-form`, symmetric frustum from
  `utils/graphics_utils.py:65-86`, znear .01 / zfar 100) and `cx, cy` passed
  separately to the rasterizer (`SLAM/render.py:68-91`);
* Gaussian parameters in the post-activation form `Renderer.render` hands to
  the rasterizer (`SLAM/render.py:93-120`): xyz (P,3), opacity (P,1) in (0,1),
  scales (P,3) > 0, rotations (P,4) unit quaternions (w,x,y,z), shs (P,16,3);
* surfel shape `r * (1, 1, 0.1)` (`configs/base.yaml:32` xyz_factor), radii in
  [min_radius, max_radius] (`configs/base.yaml:35-36`), opacity 0.99 for
  freshly added and 0.1 for attached Gaussians (`configs/base.yaml:33`,
  `SLAM/multiprocess/mapper.py:829`).

Seed 2024 is the reference's own seed (`utils/general_utils.py:179-181`).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

SH_C0 = 0.28209479177387814

# name -> (W, H, fx, fy, cx, cy); SURVEY.md §8(d)
CAMERAS = {
    "tum": (640, 480, 517.3, 516.5, 318.6, 255.3),
    "replica": (1200, 680, 600.0, 600.0, 599.5, 339.5),
    "hd": (1920, 1080, 960.0, 960.0, 959.5, 539.5),
    "tiny": (64, 48, 60.0, 60.0, 31.5, 23.5),
    "small": (160, 112, 140.0, 140.0, 79.5, 55.5),
    "ragged": (100, 75, 90.0, 85.0, 48.2, 39.1),  # H, W not multiples of 16
}


@dataclass
class Camera:
    """Per-view constants in the layout `GaussianRasterizationSettings` carries
    (`diff_gaussian_rasterization_depth/__init__.py:284-303` in the reference)."""

    width: int
    height: int
    fx: float
    fy: float
    cx: float
    cy: float
    c2w: np.ndarray = field(default_factory=lambda: np.eye(4, dtype=np.float64))
    znear: float = 0.01
    zfar: float = 100.0

    @property
    def tanfovx(self) -> float:
        return self.width / (2.0 * self.fx)

    @property
    def tanfovy(self) -> float:
        return self.height / (2.0 * self.fy)

    @property
    def w2c(self) -> np.ndarray:
        return np.linalg.inv(self.c2w)

    @property
    def viewmatrix(self) -> np.ndarray:
        """world_view_transform: W2C transposed (translation in elements 12..14
        of the flat array), float32 (4,4)."""
        return np.ascontiguousarray(self.w2c.T.astype(np.float32))

    @property
    def projection(self) -> np.ndarray:
        """getProjectionMatrix(...).transpose(0,1) of the reference."""
        ty, tx = self.tanfovy, self.tanfovx
        top, right = ty * self.znear, tx * self.znear
        P = np.zeros((4, 4), dtype=np.float32)
        P[0, 0] = 2.0 * self.znear / (2 * right)
        P[1, 1] = 2.0 * self.znear / (2 * top)
        P[3, 2] = 1.0
        P[2, 2] = self.zfar / (self.zfar - self.znear)
        P[2, 3] = -(self.zfar * self.znear) / (self.zfar - self.znear)
        return np.ascontiguousarray(P.T)

    @property
    def projmatrix(self) -> np.ndarray:
        """full_proj_transform = world_view_transform @ projection (both in the
        transposed storage), float32 (4,4)."""
        return np.ascontiguousarray((self.viewmatrix @ self.projection).astype(np.float32))

    @property
    def campos(self) -> np.ndarray:
        return np.ascontiguousarray(self.c2w[:3, 3].astype(np.float32))

    @property
    def K(self) -> np.ndarray:
        return np.array([[self.fx, 0, self.cx], [0, self.fy, self.cy], [0, 0, 1]], dtype=np.float32)

    @property
    def tile_grid(self):
        return ((self.height + 15) // 16, (self.width + 15) // 16)


def make_camera(name: str = "replica", c2w: np.ndarray | None = None) -> Camera:
    W, H, fx, fy, cx, cy = CAMERAS[name]
    cam = Camera(W, H, fx, fy, cx, cy)
    if c2w is not None:
        cam.c2w = np.asarray(c2w, dtype=np.float64)
    return cam


def small_pose(rot_deg=(1.0, -0.7, 0.4), trans=(0.02, -0.01, 0.015)) -> np.ndarray:
    """A camera-to-world pose a few cm / about a degree from identity."""
    rx, ry, rz = [math.radians(a) for a in rot_deg]
    Rx = np.array([[1, 0, 0], [0, math.cos(rx), -math.sin(rx)], [0, math.sin(rx), math.cos(rx)]])
    Ry = np.array([[math.cos(ry), 0, math.sin(ry)], [0, 1, 0], [-math.sin(ry), 0, math.cos(ry)]])
    Rz = np.array([[math.cos(rz), -math.sin(rz), 0], [math.sin(rz), math.cos(rz), 0], [0, 0, 1]])
    T = np.eye(4)
    T[:3, :3] = Rz @ Ry @ Rx
    T[:3, 3] = trans
    return T


def _quat_mul(a, b):
    aw, ax, ay, az = a[:, 0], a[:, 1], a[:, 2], a[:, 3]
    bw, bx, by, bz = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
    return np.stack(
        [
            aw * bw - ax * bx - ay * by - az * bz,
            aw * bx + ax * bw + ay * bz - az * by,
            aw * by - ax * bz + ay * bw + az * bx,
            aw * bz + ax * by - ay * bx + az * bw,
        ],
        axis=1,
    )


def _quat_z_to(n: np.ndarray) -> np.ndarray:
    """Unit quaternions (w,x,y,z) rotating local +z onto unit vectors n (P,3)."""
    w = 1.0 + n[:, 2]
    q = np.stack([w, -n[:, 1], n[:, 0], np.zeros_like(w)], axis=1)
    flip = w < 1e-6
    q[flip] = np.array([0.0, 1.0, 0.0, 0.0])
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def _perturb_normals(n, rng, sigma_deg):
    d = rng.normal(0.0, math.radians(sigma_deg), size=n.shape)
    m = n + d
    return m / np.linalg.norm(m, axis=1, keepdims=True)


def surfel_room(
    P: int,
    seed: int = 2024,
    box=(6.0, 3.0, 6.0),
    n_patches: int = 20,
    patch_frac: float = 0.3,
    r_min: float = 0.004,
    r_max: float = 0.05,
    sh_coeffs: int = 16,
    low_opacity_frac: float = 0.2,
    normal_sigma_deg: float = 5.0,
    dtype=np.float32,
):
    """Gaussians on the inside faces of a box around the origin plus planar
    patches 1-4 m in front of the identity camera (looking down +z).

    Returns a dict of numpy arrays: xyz (P,3), opacity (P,1), scales (P,3),
    rotations (P,4), shs (P,sh_coeffs,3), normal (P,3).
    """
    rng = np.random.default_rng(seed)
    n_patch = int(P * patch_frac) if n_patches > 0 else 0
    n_box = P - n_patch
    bx, by, bz = box[0] / 2, box[1] / 2, box[2] / 2

    # box faces, sampled by area
    areas = np.array([by * bz, by * bz, bx * bz, bx * bz, bx * by, bx * by]) * 4
    face = rng.choice(6, size=n_box, p=areas / areas.sum())
    u = rng.uniform(-1, 1, size=n_box)
    v = rng.uniform(-1, 1, size=n_box)
    xyz = np.zeros((n_box, 3))
    nrm = np.zeros((n_box, 3))
    for f in range(6):
        m = face == f
        axis, sign = f // 2, (1 if f % 2 == 0 else -1)
        half = [bx, by, bz]
        o = [a for a in range(3) if a != axis]
        xyz[m, axis] = sign * half[axis]
        xyz[m, o[0]] = u[m] * half[o[0]]
        xyz[m, o[1]] = v[m] * half[o[1]]
        nrm[m, axis] = -sign  # facing inwards
    pts, nrms = [xyz], [nrm]

    if n_patch > 0:
        per = np.full(n_patches, n_patch // n_patches)
        per[: n_patch - per.sum()] += 1
        for k in range(n_patches):
            c = np.array([rng.uniform(-2.0, 2.0), rng.uniform(-1.0, 1.0), rng.uniform(1.0, 4.0)])
            nn = -c / np.linalg.norm(c) + rng.normal(0, 0.35, 3)
            nn /= np.linalg.norm(nn)
            a = np.cross(nn, [0.0, 1.0, 0.0])
            a /= np.linalg.norm(a)
            b = np.cross(nn, a)
            ext = rng.uniform(0.15, 0.6, 2)
            s = rng.uniform(-1, 1, (per[k], 2)) * ext
            pts.append(c + s[:, :1] * a + s[:, 1:] * b)
            nrms.append(np.tile(nn, (per[k], 1)))
    xyz = np.concatenate(pts)
    nrm = np.concatenate(nrms)
    perm = rng.permutation(P)  # no spatial order in the Gaussian index
    xyz, nrm = xyz[perm], nrm[perm]

    nrm = _perturb_normals(nrm, rng, normal_sigma_deg)
    q = _quat_z_to(nrm)
    th = rng.uniform(0, 2 * math.pi, P)
    qz = np.stack([np.cos(th / 2), np.zeros(P), np.zeros(P), np.sin(th / 2)], axis=1)
    q = _quat_mul(q, qz)
    q /= np.linalg.norm(q, axis=1, keepdims=True)

    r = np.exp(rng.uniform(math.log(r_min), math.log(r_max), P))
    aniso = rng.uniform(0.7, 1.0, (P, 2))
    scales = np.stack([r * aniso[:, 0], r * aniso[:, 1], r * 0.1], axis=1)

    opacity = np.where(rng.uniform(size=P) < low_opacity_frac, 0.1, 0.99)[:, None]

    rgb = rng.uniform(0, 1, (P, 3))
    shs = np.zeros((P, sh_coeffs, 3))
    shs[:, 0] = (rgb - 0.5) / SH_C0
    if sh_coeffs > 1:
        shs[:, 1:] = rng.normal(0, 0.05, (P, sh_coeffs - 1, 3))

    return {
        "xyz": np.ascontiguousarray(xyz.astype(dtype)),
        "opacity": np.ascontiguousarray(opacity.astype(dtype)),
        "scales": np.ascontiguousarray(scales.astype(dtype)),
        "rotations": np.ascontiguousarray(q.astype(dtype)),
        "shs": np.ascontiguousarray(shs.astype(dtype)),
        "normal": np.ascontiguousarray(nrm.astype(dtype)),
    }


def random_blobs(P: int, seed: int = 7, sh_coeffs: int = 16, depth=(0.4, 5.0), dtype=np.float32):
    """Unstructured Gaussians in front of the identity camera: random
    orientation, anisotropic scales, opacities spanning the alpha cut-offs. Used
    by parity tests to reach branches the surfel room rarely takes (centre-depth
    fallback, no-hit pixels, clamped colours, off-screen and behind-camera
    culls)."""
    rng = np.random.default_rng(seed)
    z = rng.uniform(depth[0] - 0.5, depth[1], P)  # some behind the 0.2 near cut
    xyz = np.stack([rng.uniform(-1.6, 1.6, P) * np.abs(z), rng.uniform(-1.2, 1.2, P) * np.abs(z), z], axis=1)
    q = rng.normal(size=(P, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    scales = np.exp(rng.uniform(math.log(0.003), math.log(0.12), (P, 3)))
    opacity = rng.uniform(0.02, 1.0, (P, 1))
    shs = np.zeros((P, sh_coeffs, 3))
    shs[:, 0] = rng.uniform(-0.4, 1.2, (P, 3)) / SH_C0 - 0.5 / SH_C0
    if sh_coeffs > 1:
        shs[:, 1:] = rng.normal(0, 0.15, (P, sh_coeffs - 1, 3))
    return {
        "xyz": np.ascontiguousarray(xyz.astype(dtype)),
        "opacity": np.ascontiguousarray(opacity.astype(dtype)),
        "scales": np.ascontiguousarray(scales.astype(dtype)),
        "rotations": np.ascontiguousarray(q.astype(dtype)),
        "shs": np.ascontiguousarray(shs.astype(dtype)),
        "normal": np.zeros((P, 3), dtype=dtype),
    }


def dense_blobs(P: int, seed: int = 21, sh_coeffs: int = 16, dtype=np.float32):
    """Translucent Gaussians packed inside a narrow frustum: very long per-tile lists (stress for the per-tile sort
    and for pixels that never reach an opaque hit)."""
    rng = np.random.default_rng(seed)
    z = rng.uniform(1.0, 3.0, P)
    xyz = np.stack([rng.uniform(-0.45, 0.45, P) * z, rng.uniform(-0.35, 0.35, P) * z, z], axis=1)
    q = rng.normal(size=(P, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    scales = np.exp(rng.uniform(math.log(0.01), math.log(0.08), (P, 3)))
    opacity = rng.uniform(0.02, 0.3, (P, 1))
    shs = np.zeros((P, sh_coeffs, 3))
    shs[:, 0] = rng.uniform(0.0, 1.0, (P, 3)) / SH_C0 - 0.5 / SH_C0
    if sh_coeffs > 1:
        shs[:, 1:] = rng.normal(0, 0.1, (P, sh_coeffs - 1, 3))
    return {
        "xyz": np.ascontiguousarray(xyz.astype(dtype)), "opacity": np.ascontiguousarray(opacity.astype(dtype)),
        "scales": np.ascontiguousarray(scales.astype(dtype)), "rotations": np.ascontiguousarray(q.astype(dtype)),
        "shs": np.ascontiguousarray(shs.astype(dtype)), "normal": np.zeros((P, 3), dtype=dtype),
    }


def random_tile_mask(cam: Camera, keep: float = 0.5, seed: int = 11) -> np.ndarray:
    rng = np.random.default_rng(seed)
    th, tw = cam.tile_grid
    return (rng.uniform(size=(th, tw)) < keep).astype(np.int32)


def upstream_grads(cam: Camera, seed: int = 5):
    """dL/dcolor (3,H,W) and dL/ddepth (1,H,W): signs of an L1 loss against a
    random target, scaled 1/N (`SLAM/multiprocess/mapper.py:421-431`)."""
    rng = np.random.default_rng(seed)
    N = cam.width * cam.height
    gc = np.sign(rng.uniform(-1, 1, (3, cam.height, cam.width))) * rng.uniform(0.5, 1.5, (3, cam.height, cam.width))
    gd = np.sign(rng.uniform(-1, 1, (1, cam.height, cam.width))) * rng.uniform(0.5, 1.5, (1, cam.height, cam.width))
    return (gc / N).astype(np.float32), (gd / N).astype(np.float32)


# --------------------------------------------------------------------------
# depth frames for the ICP path
# --------------------------------------------------------------------------

DEFAULT_SPHERES = (((0.3, 0.1, 2.0), 0.6), ((-0.9, -0.3, 2.4), 0.45), ((1.0, 0.5, 2.6), 0.4), ((-0.2, 0.7, 1.6), 0.25),
                   ((0.8, -0.6, 1.8), 0.3))


def raycast_room_depth(cam: Camera, box=(6.0, 3.0, 6.0), noise_sigma: float = 0.0, seed: int = 3,
                       spheres=DEFAULT_SPHERES) -> np.ndarray:
    """z-depth (H,W) float32 of the box room (plus a few spheres, so that all six pose degrees of freedom are
    constrained) seen from `cam.c2w`; optional Gaussian noise; values outside [0.3, 5] m set to 0
    (`configs/base.yaml:38-39` min/max depth)."""
    H, W = cam.height, cam.width
    j, i = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    d_c = np.stack([(i - cam.cx) / cam.fx, (j - cam.cy) / cam.fy, np.ones_like(i, dtype=np.float64)], -1)
    R, t = cam.c2w[:3, :3], cam.c2w[:3, 3]
    d_w = d_c @ R.T
    half = np.array(box) / 2
    with np.errstate(divide="ignore", invalid="ignore"):
        t1 = (half - t) / d_w
        t2 = (-half - t) / d_w
    tfar = np.minimum(np.maximum(t1, t2).min(-1), 1e9)
    depth = tfar.copy()  # ray parameter == z-depth because d_c.z == 1
    for c, rad in (spheres or ()):
        c = np.array(c)
        oc = t - c
        a = (d_w * d_w).sum(-1)
        b = 2 * (d_w * oc).sum(-1)
        cc = (oc * oc).sum() - rad * rad
        disc = b * b - 4 * a * cc
        ts = np.where(disc > 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), np.inf)
        depth = np.where((ts > 0) & (ts < depth), ts, depth)
    if noise_sigma > 0:
        depth = depth + np.random.default_rng(seed).normal(0, noise_sigma, depth.shape)
    depth = np.where((depth < 0.3) | (depth > 5.0), 0.0, depth)
    return depth.astype(np.float32)


def raycast_room_rgbd(cam: Camera, box=(6.0, 3.0, 6.0), noise_sigma: float = 0.0, seed: int = 3, spheres=DEFAULT_SPHERES,
                      color_seed: int = 7, n_waves: int = 4):
    """(depth (H,W) float32, colour (H,W,3) float32 in [0, 1]) of the textured box room seen from `cam.c2w`.

    The depth is `raycast_room_depth`'s (same box, spheres, noise and range mask). The colour is a smooth function of the
    world point the pixel's ray hits, so it moves with the scene, not with the camera: per channel 0.5 plus `n_waves`
    sinusoids of seeded direction, phase, amplitude and wavelength (0.1 - 0.5 m), clipped to [0, 1]. `spheres=()` with the
    camera facing a wall gives a planar view with texture. Pixels without depth take the colour at the camera centre."""
    depth = raycast_room_depth(cam, box, noise_sigma, seed, spheres)
    hit_z = raycast_room_depth(cam, box, 0.0, seed, spheres).astype(np.float64)
    H, W = cam.height, cam.width
    j, i = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    d_c = np.stack([(i - cam.cx) / cam.fx, (j - cam.cy) / cam.fy, np.ones_like(i, dtype=np.float64)], -1)
    p_w = (d_c * hit_z[..., None]) @ cam.c2w[:3, :3].T + cam.c2w[:3, 3]
    rng = np.random.default_rng(color_seed)
    color = np.full((H, W, 3), 0.5)
    for ch in range(3):
        for _ in range(n_waves):
            d = rng.normal(size=3)
            d /= np.linalg.norm(d)
            lam = rng.uniform(0.1, 0.5)
            amp = rng.uniform(0.05, 0.15)
            phase = rng.uniform(0, 2 * np.pi)
            color[..., ch] += amp * np.sin(2 * np.pi * (p_w @ d) / lam + phase)
    return depth, np.clip(color, 0.0, 1.0).astype(np.float32)


def wall_cameras(W: int, H: int, dx: float = 0.02, dy: float = 0.015, deg: float = 1.0):
    """Two cameras (TUM intrinsics scaled to width W) facing the room's far wall (z = 3 m) at 20 degrees, 1.1-2.1 m
    away, with no other surface in view; the second is moved by (dx, dy) in the wall's plane and turned by `deg` about the
    wall normal, the three directions a point-to-plane residual cannot see. Returns (cam0, cam1, ground-truth pose of
    frame 1 in frame 0, i.e. cam0.w2c @ cam1.c2w)."""
    s = W / 640.0
    a, b = math.radians(20.0), math.radians(deg)
    C0 = np.eye(4)
    C0[:3, :3] = [[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]]
    C0[:3, 3] = (-0.5, 0.0, 1.5)
    Rz = np.array([[math.cos(b), -math.sin(b), 0], [math.sin(b), math.cos(b), 0], [0, 0, 1]])
    C1 = C0.copy()
    C1[:3, :3] = Rz @ C0[:3, :3]
    C1[:3, 3] = C0[:3, 3] + (dx, dy, 0.0)
    cams = [Camera(W, H, 517.3 * s, 516.5 * s, 318.6 * s, 255.3 * s, c2w=c) for c in (C0, C1)]
    return cams[0], cams[1], np.linalg.inv(C0) @ C1


def wall_in_plane_error(cam0: Camera, cam1: Camera, pose) -> tuple:
    """(in-plane translation error in m, rotation error about the wall normal in degrees) of a tracked pose of frame 1
    in frame 0 on the views of `wall_cameras`."""
    Ce = cam0.c2w @ np.asarray(pose, dtype=np.float64)
    E = Ce @ np.linalg.inv(cam1.c2w)
    return float(np.linalg.norm(Ce[:2, 3] - cam1.c2w[:2, 3])), abs(math.degrees(math.atan2(E[1, 0], E[0, 0])))
