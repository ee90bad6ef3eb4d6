"""CPU tests of the camera gradient (dL/d viewmatrix, projmatrix, campos) of the float64 oracle against central finite
differences, of the float32 oracle against the float64 one, and host-side validation of rtg_splat_backward_camera.

The reference has no camera gradient, so finite differences are what pin this part of the oracle. A camera perturbation
moves every Gaussian at once, so a discrete decision (cull, tile cut-off, alpha < 1/255, opaque hit, plane test) can flip
inside the step. Every entry is therefore differenced with two step sizes; where the two estimates disagree the entry
straddles a discontinuity and is skipped. The skips are counted and must stay few."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

from oracle.camera_oracle import camera_gradient
from oracle.splat_oracle import OracleRender
from rtg_slam_b200 import scene

import helpers

# entries the forward reads; viewmatrix[3, 7, 11, 15] are never read and get exactly 0
VIEW_READ = [4 * j + k for j in range(4) for k in range(3)]


def make_cam(name="tiny", c2w=None, view=None):
    """Camera with float64 matrices that a test may replace entry by entry (projmatrix = view @ projection unless given)."""
    base = scene.make_camera(name, c2w=c2w)
    vm = base.w2c.T.copy() if view is None else np.asarray(view, np.float64)
    return SimpleNamespace(width=base.width, height=base.height, tanfovx=base.tanfovx, tanfovy=base.tanfovy, cx=base.cx,
                           cy=base.cy, viewmatrix=vm, projmatrix=vm @ base.projection.astype(np.float64),
                           campos=np.linalg.inv(vm.T)[:3, 3].copy())


def compact_scene(P, seed, sh_coeffs=16):
    """P surfels 1.5-3 m in front of the camera, inside the frustum, overlapping: most pixels are covered, many by an
    opaque (alpha >= 0.6) surfel, so both the colour and the depth path carry gradient. Opacity <= 0.95 keeps
    opacity * G below the 0.99 clamp, which the reference's backward does not differentiate."""
    rng = np.random.default_rng(seed)
    z = rng.uniform(1.5, 3.0, P)
    xyz = np.stack([rng.uniform(-0.45, 0.45, P) * z, rng.uniform(-0.32, 0.32, P) * z, z], 1)
    nrm = rng.normal(size=(P, 3)) * [0.3, 0.3, 1.0]
    nrm[:, 2] = np.abs(nrm[:, 2])  # roughly along the optical axis (the plane test uses |n . ray|)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    q = scene._quat_z_to(nrm)
    r = rng.uniform(0.06, 0.2, P)
    scales = np.stack([r, r * rng.uniform(0.6, 1.0, P), 0.1 * r], 1)
    opacity = rng.uniform(0.3, 0.95, (P, 1))
    shs = np.zeros((P, sh_coeffs, 3))
    shs[:, 0] = rng.uniform(0.0, 1.0, (P, 3)) / scene.SH_C0 - 0.5 / scene.SH_C0
    shs[:, 1:] = rng.normal(0, 0.3, (P, sh_coeffs - 1, 3))
    return {"xyz": xyz, "opacity": opacity, "scales": scales, "rotations": q, "shs": shs}


def cov3d(g):
    r, x, y, z = g["rotations"].T
    R = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
                  np.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
                  np.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], 1)
    Ms = R * g["scales"][:, None, :]
    S = Ms @ Ms.transpose(0, 2, 1)
    return S[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]


def nonrigid_view():
    """A pose whose 3x3 block is slightly scaled and sheared (the rasterizer reads the matrices as given)."""
    v = make_cam(c2w=scene.small_pose()).viewmatrix.copy()
    A = np.array([[1.03, 0.02, 0.0], [0.0, 0.97, -0.015], [0.01, 0.0, 1.01]])
    v[:3, :3] = v[:3, :3] @ A.T   # rows of the stored (transposed) matrix are world axes
    return v


def case(name):
    """(camera, gaussians, render kwargs, upstream (dL/dcolor, dL/ddepth))."""
    g = compact_scene(160, seed=11)
    cam = make_cam(c2w=scene.small_pose())
    kw = {}
    gc, gd = scene.upstream_grads(cam, seed=3)
    gc, gd = gc.astype(np.float64), gd.astype(np.float64)
    if name == "colors_precomp":
        kw["colors_precomp"] = np.random.default_rng(12).uniform(-0.2, 1.2, (160, 3))
    elif name == "cov3D_precomp":
        kw["cov3D_precomp"] = cov3d(g)
    elif name == "color_only":
        gd = np.zeros_like(gd)
    elif name == "depth_only":
        gc = np.zeros_like(gc)
    elif name == "nonrigid":
        cam = make_cam(view=nonrigid_view())
    elif name == "masked":  # outside the rendered tiles the hit map keeps its initial 0, which is not a hit
        kw["tile_mask"] = np.array([[1, 0, 1, 1], [0, 1, 0, 1], [1, 1, 0, 0]], np.int32)
    else:
        assert name == "sh3"
    return cam, g, kw, (gc, gd)


CASES = ("sh3", "colors_precomp", "cov3D_precomp", "color_only", "depth_only", "nonrigid", "masked")


def render(cam, g, kw, precision="f64"):
    return OracleRender(cam, g, precision=precision, **kw)


def loss(cam, g, kw, up):
    o = render(cam, g, kw)
    v = float((o.color * up[0]).sum() + (o.depth * up[1]).sum())
    o.close()
    return v


def perturbed(cam, which, idx, h):
    c = SimpleNamespace(**vars(cam))
    arr = getattr(cam, which).copy()
    arr.reshape(-1)[idx] += h
    setattr(c, which, arr)
    return c


def fd(cam, g, kw, up, which, idx, h):
    return (loss(perturbed(cam, which, idx, h), g, kw, up) - loss(perturbed(cam, which, idx, -h), g, kw, up)) / (2 * h)


@pytest.mark.parametrize("name", CASES)
def test_oracle_camera_gradient_matches_finite_differences(name):
    cam, g, kw, up = case(name)
    o = render(cam, g, kw)
    assert (o.radii > 0).sum() > 100
    hit = o.hit_depth[0] >= 0
    assert hit.mean() > 0.3, "the depth path must be exercised"
    if name == "depth_only" or name == "sh3":
        # both branches of the depth hit: plane (surfel) and centre depth
        pv = g["xyz"] @ cam.viewmatrix[:3, :3] + cam.viewmatrix[3, :3]
        centre = np.isclose(o.depth[0][hit], pv[o.hit_depth[0][hit], 2], rtol=0, atol=1e-9)
        assert 0 < centre.sum() < hit.sum(), "need pixels on the plane and on the centre-depth branch"
    an = camera_gradient(o, *up)
    assert np.all(an["viewmatrix"].reshape(-1)[[3, 7, 11, 15]] == 0)
    entries = [("viewmatrix", i) for i in VIEW_READ] + [("projmatrix", i) for i in range(16)] + [("campos", i) for i in range(3)]
    skipped, checked = [], 0
    for which, idx in entries:
        a = float(an[which].reshape(-1)[idx])
        scale = np.abs(an[which]).max()
        h = 1e-6 * max(1.0, abs(float(getattr(cam, which).reshape(-1)[idx])))
        f1, f2 = fd(cam, g, kw, up, which, idx, h), fd(cam, g, kw, up, which, idx, h / 4)
        if abs(f1 - f2) > 1e-6 * scale + 1e-10:  # the two steps disagree: a decision flipped inside the larger one
            skipped.append((which, idx))
            continue
        checked += 1
        assert abs(f2 - a) <= 1e-6 * scale + 1e-10, (name, which, idx, a, f1, f2)  # measured: <= 1e-8
    assert len(skipped) <= 3, (name, skipped)
    if name == "colors_precomp":
        assert np.all(an["campos"] == 0)
    assert checked >= len(entries) - 3


@pytest.mark.parametrize("name", CASES)
def test_oracle_camera_gradient_f32_matches_f64(name):
    cam, g, kw, up = case(name)
    g32 = {k: v.astype(np.float32) for k, v in g.items()}
    kw32 = {k: (v if k == "tile_mask" else v.astype(np.float32)) for k, v in kw.items()}
    c32 = SimpleNamespace(**vars(cam))
    for k in ("viewmatrix", "projmatrix", "campos"):
        setattr(c32, k, getattr(cam, k).astype(np.float32))
    a = camera_gradient(render(c32, g32, kw32, "f32"), up[0].astype(np.float32), up[1].astype(np.float32))
    b = camera_gradient(render(c32, g32, kw32), *up)
    for k in ("viewmatrix", "projmatrix", "campos"):
        if np.abs(b[k]).max() == 0:
            assert np.all(a[k] == 0), (name, k)
            continue
        assert helpers.rel_err(a[k], b[k]) < 1e-4, (name, k, helpers.rel_err(a[k], b[k]))


@pytest.mark.parametrize("name", CASES)
def test_oracle_camera_gradient_cancels_the_mean_gradients_under_translation(name):
    """Moving every mean and the camera by one delta leaves the render unchanged, so the oracle's per-Gaussian dL/dmeans3D
    (splat_oracle.c) and the camera gradient (camera_oracle.py, a separate statement) must cancel: with T' = T - W delta,
    the projection's translation row likewise, and campos' = campos + delta."""
    cam, g, kw, up = case(name)
    o = render(cam, g, kw)
    gr = o.backward(*up)
    cg = camera_gradient(o, *up, grads=gr)
    vm, pm = cam.viewmatrix, cam.projmatrix
    d_cam = -vm[:3, :3] @ cg["viewmatrix"][3, :3] - pm[:3, :] @ cg["projmatrix"][3, :] + cg["campos"]
    d_map = gr["means3D"].sum(0)
    scale = np.abs(gr["means3D"]).sum(0)
    assert np.all(np.abs(d_cam) > 1e-3 * scale), (d_cam, scale)  # the camera carries its half of the cancellation
    assert np.all(np.abs(d_map + d_cam) <= 1e-9 * scale), (d_map, d_cam, scale)


def test_camera_entry_points_validate_before_touching_cuda():
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    nul = [None]
    # rtg_splat_backward's argument list + visible_rows_only, dL_dcamera, camera_scratch (+ stream)
    tail = lambda P, dcam, scratch: (P, 16, *(nul * 6), *(nul * 4), 0, None, *(nul * 4), None, *(nul * 8), 0, dcam, scratch, None)
    assert L.rtg_splat_backward_camera(None, *tail(1, C.c_void_p(256), C.c_void_p(256))) == -1
    assert b"view is NULL" in L.rtg_last_error()
    view = _lib.RtgSplatView()
    view.image_height, view.image_width, view.sh_degree = 48, 64, 3
    view.viewmatrix = view.projmatrix = view.campos = view.bg = 256  # never dereferenced: validation fails first
    assert L.rtg_splat_backward_camera(C.byref(view), *tail(-1, C.c_void_p(256), C.c_void_p(256))) == -1
    assert b"P < 0" in L.rtg_last_error()
    assert L.rtg_splat_backward_camera(C.byref(view), *tail(1, None, C.c_void_p(256))) == -1
    assert b"dL_dcamera / camera_scratch is NULL" in L.rtg_last_error()
    assert L.rtg_splat_backward_camera(C.byref(view), *tail(1, C.c_void_p(256), None)) == -1
    assert b"dL_dcamera / camera_scratch is NULL" in L.rtg_last_error()
    assert L.rtg_splat_backward_camera(C.byref(view), *tail(1, C.c_void_p(256), C.c_void_p(260))) == -1
    assert b"8-byte aligned" in L.rtg_last_error()
    # one double per camera term (27 non-zero entries of the 35) and per 256-thread block of the per-Gaussian pass
    assert L.rtg_splat_camera_scratch_bytes(1) == 27 * 8
    assert L.rtg_splat_camera_scratch_bytes(1_000_000) == ((1_000_000 + 255) // 256) * 27 * 8
    assert L.rtg_splat_camera_scratch_bytes(-1) == 0
