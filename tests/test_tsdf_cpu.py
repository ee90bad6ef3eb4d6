"""TSDF fusion and marching tetrahedra without a GPU: the float64 oracle's case table (against the kernel's), its meshes
of analytic signed distance fields, its integration against a voxel-by-voxel statement of the five rules, the PLY writer,
and the validation rtg_tsdf_* and reconstruct.py do before any CUDA work."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from oracle import tsdf_oracle as T
from rtg_slam_b200 import _lib, reconstruct, scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _edges(F):
    e = np.sort(np.concatenate([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]]), axis=1)
    return np.unique(e, axis=0, return_counts=True)


def test_kernel_case_table_is_the_derived_one():
    src = open(os.path.join(ROOT, "rtg_slam_b200", "csrc", "tsdf.cu")).read()
    body = re.search(r"kTetTriangles\[16\]\[2\]\[3\] = \{(.*?)\};", src, re.S).group(1)
    kernel = np.array([int(x) for x in re.findall(r"-?\d+", body)]).reshape(16, 2, 3)
    assert np.array_equal(kernel, T.tet_table())


def test_case_table_orientation_and_counts():
    """Every case with 1 or 3 negative corners has one triangle, with 2 it has two; each triangle's normal points from
    the negative corners of the unit right tetrahedron to the positive ones."""
    tab = T.tet_table()
    corners = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [1, 1, 1]], float)  # permutation (0,1,2): positively oriented
    assert np.linalg.det(corners[1:] - corners[0]) > 0
    for case in range(16):
        neg = [q for q in range(4) if case >> q & 1]
        n_tri = int((tab[case, :, 0] >= 0).sum())
        assert n_tri == {0: 0, 1: 1, 2: 2, 3: 1, 4: 0}[len(neg)]
        if n_tri == 0:
            continue
        mid = np.array([(corners[a] + corners[b]) / 2 for a, b in T.TET_EDGES])
        dirn = corners[[q for q in range(4) if q not in neg]].mean(0) - corners[neg].mean(0)
        for r in range(n_tri):
            p = mid[tab[case, r]]
            assert np.dot(np.cross(p[1] - p[0], p[2] - p[0]), dirn) > 0, (case, r)


def test_sphere_mesh_is_closed_oriented_and_near():
    s, r, c = 0.05, 0.6, np.array([1.01, 0.97, 1.03])
    tsdf, w = T.sphere_grid((42, 41, 40), s, c, r, 5 * s)
    V, F, _ = T.extract(tsdf, w, None, (0.0, 0.0, 0.0), s)
    assert len(F) > 1000
    e, cnt = _edges(F)
    assert (cnt == 2).all()                                   # every undirected edge is shared by exactly two faces
    assert len(V) - len(e) + len(F) == 2                      # a sphere's Euler characteristic
    n = np.cross(V[F[:, 1]] - V[F[:, 0]], V[F[:, 2]] - V[F[:, 0]])
    assert (np.einsum("ij,ij->i", n, V[F].mean(1) - c) > 0).all()   # outward: from inside (negative) to free space
    assert np.abs(np.linalg.norm(V - c, axis=1) - r).max() < s * s / r


def test_tilted_plane_vertices_lie_on_the_plane():
    s = 0.04
    nrm = np.array([0.3, -0.5, 0.8])
    nrm /= np.linalg.norm(nrm)
    tsdf, w = T.plane_grid((23, 25, 21), s, nrm, 0.55, 4 * s)
    V, F, _ = T.extract(tsdf, w, None, (0.0, 0.0, 0.0), s)
    assert len(F) > 100
    assert np.abs(V @ nrm - 0.55).max() < 1e-6 * s
    n = np.cross(V[F[:, 1]] - V[F[:, 0]], V[F[:, 2]] - V[F[:, 0]])
    assert (n @ nrm > 0).all()


def test_faces_need_four_observed_corners_and_colours_interpolate():
    s = 0.1
    tsdf, w = T.plane_grid((8, 8, 8), s, (0.0, 0.0, 1.0), 0.35, 3 * s)
    col = np.stack([tsdf * 0 + 0.25, tsdf * 0 + 0.5, np.broadcast_to(np.arange(8.0)[:, None, None], tsdf.shape) / 8])
    V, F, Cv = T.extract(tsdf, w, col, (0.0, 0.0, 0.0), s)
    assert np.allclose(Cv[:, 2], V[:, 2] / (8 * s)) and np.allclose(Cv[:, :2], [0.25, 0.5])
    w2 = w.copy()
    w2[:, :, 4:] = 0                                          # the half x >= 4 s unobserved
    V2, F2, _ = T.extract(tsdf, w2, None, (0.0, 0.0, 0.0), s)
    assert 0 < len(F2) < len(F) and V2[F2].max(axis=(0, 1))[0] <= 3 * float(np.float32(s)) + 1e-12


def test_integration_oracle_is_the_five_rules():
    cam = scene.make_camera("small", c2w=scene.small_pose())
    depth = scene.raycast_room_depth(cam)
    rng = np.random.default_rng(4)
    color_img = rng.uniform(0, 1, (cam.height, cam.width, 3)).astype(np.float32)
    origin, s, dims, trunc = (-3.0, -1.5, -3.0), 0.1, (61, 31, 61), 0.3
    tsdf, w, col = T.new_volume(dims, color=True)
    tsdf[:] = rng.uniform(-1, 1, tsdf.shape)                  # a previous state, so that the running mean is exercised
    w[:] = rng.integers(0, 3, w.shape)
    col[:] = rng.uniform(0, 1, col.shape)
    t0, w0, c0 = tsdf.copy(), w.copy(), col.copy()
    w2c = np.linalg.inv(cam.c2w)
    K = (cam.fx, cam.fy, cam.cx, cam.cy)
    tie = T.integrate(tsdf, w, col, origin, s, trunc, depth, w2c, K, color_img)
    assert 0.02 < (w > w0).mean() < 0.5
    fx, fy, cx, cy = (float(np.float32(k)) for k in K)
    o = np.float32(origin).astype(np.float64)
    checked = 0
    for lin in rng.choice(tsdf.size, 6000, replace=False):
        k, j, i = np.unravel_index(lin, tsdf.shape)
        p = o + float(np.float32(s)) * np.array([i, j, k])
        x, y, z = w2c[:3, :3] @ p + w2c[:3, 3]
        want_t, want_w, want_c = t0[k, j, i], w0[k, j, i], c0[:, k, j, i]
        if z > 0:
            u, v = round(fx * x / z + cx), round(fy * y / z + cy)        # Python's round is half to even
            if 0 <= u <= cam.width - 1 and 0 <= v <= cam.height - 1 and depth[v, u] > 0:
                sdf = float(depth[v, u]) - z
                if sdf >= -float(np.float32(trunc)):
                    f = min(1.0, sdf / float(np.float32(trunc)))
                    want_t = (want_t * want_w + f) / (want_w + 1)
                    want_c = (want_c * want_w + color_img[v, u]) / (want_w + 1)
                    want_w = want_w + 1
        assert w[k, j, i] == want_w and tsdf[k, j, i] == pytest.approx(want_t, abs=1e-12), (i, j, k)
        assert np.allclose(col[:, k, j, i], want_c, atol=1e-12)
        checked += want_w > w0[k, j, i]
    assert checked > 150 and tie.mean() < 0.02


def test_write_ply_round_trips(tmp_path):
    rng = np.random.default_rng(2)
    V = rng.normal(size=(57, 3)).astype(np.float32)
    F = rng.integers(0, 57, (91, 3)).astype(np.int32)
    Cv = rng.uniform(-0.1, 1.1, (57, 3)).astype(np.float32)
    for colors in (None, Cv):
        path = str(tmp_path / "m.ply")
        reconstruct.write_ply(path, torch.from_numpy(V), torch.from_numpy(F), None if colors is None else torch.from_numpy(colors))
        V2, F2, C2 = _read_ply(path)
        assert np.array_equal(V2, V) and np.array_equal(F2, F)
        if colors is None:
            assert C2 is None
        else:
            assert np.array_equal(C2, np.rint(np.clip(Cv, 0, 1) * 255).astype(np.uint8))


def _read_ply(path):
    """A minimal binary little-endian PLY reader: vertex x y z [red green blue], face lists of uchar count + int ids."""
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    lines = data[:end].decode("ascii").splitlines()
    assert lines[0] == "ply" and lines[1] == "format binary_little_endian 1.0"
    nv = int(next(ln for ln in lines if ln.startswith("element vertex")).split()[-1])
    nf = int(next(ln for ln in lines if ln.startswith("element face")).split()[-1])
    has_c = "property uchar red" in lines
    vdt = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")] + ([("r", "u1"), ("g", "u1"), ("b", "u1")] if has_c else [])
    vert = np.frombuffer(data, dtype=vdt, count=nv, offset=end)
    face = np.frombuffer(data, dtype=[("n", "u1"), ("i", "<i4", (3,))], count=nf, offset=end + vert.nbytes)
    assert (face["n"] == 3).all() and end + vert.nbytes + face.nbytes == len(data)
    V = np.stack([vert["x"], vert["y"], vert["z"]], 1)
    Cv = np.stack([vert["r"], vert["g"], vert["b"]], 1) if has_c else None
    return V, face["i"], Cv


# ------------------------------------------------------------------------------------------------ host validation
def _vol(**over):
    f = dict(nx=4, ny=5, nz=6, voxel_size=0.1, trunc=0.3, origin=(C.c_float * 3)(0, 0, 0), tsdf=8, weight=16, color=None)
    f.update(over)
    return _lib.RtgTsdfVolume(**f)


def test_volume_struct_layout():
    assert C.sizeof(_lib.RtgTsdfVolume) == 8 * 4 + 3 * 8 and _lib.RtgTsdfVolume.tsdf.offset == 32


@pytest.mark.parametrize("over, msg", [
    (dict(nx=0), b"bad dims"), (dict(nz=-1), b"bad dims"), (dict(nx=1 << 16, ny=1 << 15, nz=1), b"bad dims"),
    (dict(nx=1 << 11, ny=1 << 10, nz=1 << 10), b"bad dims"), (dict(voxel_size=0.0), b"voxel_size"),
    (dict(trunc=-1.0), b"trunc"), (dict(trunc=float("nan")), b"trunc"), (dict(tsdf=None), b"NULL pointer"),
    (dict(weight=None), b"NULL pointer"), (dict(origin=(C.c_float * 3)(0, float("inf"), 0)), b"origin"),
])
def test_integrate_rejects_bad_volumes_before_cuda(over, msg):
    L = _lib.lib()
    v = _vol(**over)
    assert L.rtg_tsdf_integrate(C.byref(v), 8, None, 4, 4, 0, 1.0, 1.0, 0.0, 0.0, 8, 1, None) == -1
    assert msg in L.rtg_last_error()


def test_tsdf_entry_points_reject_bad_arguments_before_cuda():
    L = _lib.lib()
    v = _vol()
    assert L.rtg_tsdf_integrate(None, 8, None, 4, 4, 0, 1.0, 1.0, 0.0, 0.0, 8, 1, None) == -1
    assert b"vol is NULL" in L.rtg_last_error()
    assert L.rtg_tsdf_integrate(C.byref(v), 8, None, 0, 4, 0, 1.0, 1.0, 0.0, 0.0, 8, 1, None) == -1
    assert b"image size" in L.rtg_last_error()
    assert L.rtg_tsdf_integrate(C.byref(v), None, None, 4, 4, 0, 1.0, 1.0, 0.0, 0.0, 8, 1, None) == -1
    assert b"depth or w2c" in L.rtg_last_error()
    assert L.rtg_tsdf_integrate(C.byref(v), 8, None, 4, 4, 0, 1.0, 1.0, 0.0, 0.0, None, 1, None) == -1
    assert L.rtg_tsdf_integrate(C.byref(v), 8, 8, 4, 4, 0, 1.0, 1.0, 0.0, 0.0, 8, 1, None) == -1
    assert b"exactly when the volume has color" in L.rtg_last_error()
    vc = _vol(color=24)
    assert L.rtg_tsdf_integrate(C.byref(vc), 8, None, 4, 4, 0, 1.0, 1.0, 0.0, 0.0, 8, 1, None) == -1
    assert L.rtg_tsdf_integrate(C.byref(v), 8, None, 4, 4, 0, 0.0, 1.0, 0.0, 0.0, 8, 1, None) == -1
    assert b"intrinsics" in L.rtg_last_error()
    assert L.rtg_tsdf_extract_count(None, 8, 8, None) == -1
    assert L.rtg_tsdf_extract_count(C.byref(v), None, 8, None) == -1 and b"ws or counts" in L.rtg_last_error()
    assert L.rtg_tsdf_extract_count(C.byref(v), 8, None, None) == -1
    assert L.rtg_tsdf_extract_emit(C.byref(v), 8, None, None, 8, None) == -1 and b"vertices or faces" in L.rtg_last_error()
    assert L.rtg_tsdf_extract_emit(C.byref(v), 8, 8, None, None, None) == -1
    big = _vol(nx=1024, ny=1024, nz=400)                          # < 2^31 voxels: integrable, too many cells to extract
    assert L.rtg_tsdf_extract_count(C.byref(big), 8, 8, None) == -1 and b"bad dims" in L.rtg_last_error()


def test_extract_workspace_bytes_is_host_only():
    L = _lib.lib()
    n = 301 * 151 * 301
    b = L.rtg_tsdf_extract_workspace_bytes(301, 151, 301)
    assert 9 * n <= b < 9 * n + 4096 + 2 * 4 * (n // 1024 + 1)
    assert L.rtg_tsdf_extract_workspace_bytes(0, 1, 1) == 0
    assert L.rtg_tsdf_extract_workspace_bytes(1024, 1024, 400) == 0


def test_python_rejects_bad_inputs_before_cuda():
    with pytest.raises(ValueError):
        reconstruct.TsdfVolume((0, 0, 0), 0.1, (0, 4, 4), 0.3)
    with pytest.raises(ValueError):
        reconstruct.TsdfVolume((0, 0, 0), 0.1, (2048, 1024, 1024), 0.3)
    with pytest.raises(ValueError):
        reconstruct.TsdfVolume((0, 0, 0), -0.1, (4, 4, 4), 0.3)
    with pytest.raises(ValueError):
        reconstruct.TsdfVolume((0, 0), 0.1, (4, 4, 4), 0.3)
    pts = torch.zeros((10, 3))
    with pytest.raises(TypeError):
        reconstruct.reconstruction_metrics(pts, pts)
    with pytest.raises(TypeError):
        reconstruct.sample_surface(pts, torch.zeros((2, 3), dtype=torch.int32), 5)
    with pytest.raises(ValueError):
        reconstruct.write_ply("/dev/null", np.zeros((3, 2)), np.zeros((1, 3)))
