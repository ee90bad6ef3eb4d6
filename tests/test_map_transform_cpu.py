"""The map transform without a GPU: the float64 oracle's SH rotation (its defining identity and the properties of a
representation), its mean / quaternion / normal formulas against 4x4 matrix products, the C struct's layout, and the
validation that rtg_map_transform and mapsurgery.transform do before any CUDA work."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import maptransform_oracle as mo
from rtg_slam_b200 import _lib, mapsurgery

ROTS = 50
DIRS = 1000


def _rotations(seed):
    rng = np.random.default_rng(seed)
    return [mo.random_rotation(rng, 180.0) for _ in range(ROTS)], rng


@pytest.mark.parametrize("l", [1, 2, 3])
def test_sh_rotation_keeps_the_colour_seen_along_the_rotated_direction(l):
    rots, rng = _rotations(10 + l)
    d = mo.unit_dirs(DIRS, rng)
    b = mo.BANDS[l]
    for R in rots:
        f = np.zeros((DIRS, 16, 3))
        f[:, b] = rng.normal(size=(2 * l + 1, 3))
        g = f.copy()
        g[:, b] = np.einsum("ij,njc->nic", mo.sh_rotation(R, l), f[:, b])
        np.testing.assert_allclose(mo.sh_eval(g, d @ R.T), mo.sh_eval(f, d), rtol=0, atol=1e-12)


@pytest.mark.parametrize("l", [1, 2, 3])
def test_sh_rotation_is_an_orthogonal_representation(l):
    rots, _ = _rotations(20 + l)
    n = 2 * l + 1
    np.testing.assert_allclose(mo.sh_rotation(np.eye(3), l), np.eye(n), rtol=0, atol=1e-12)
    for R1, R2 in zip(rots, rots[1:] + rots[:1]):
        D1, D2 = mo.sh_rotation(R1, l), mo.sh_rotation(R2, l)
        np.testing.assert_allclose(mo.sh_rotation(R1 @ R2, l), D1 @ D2, rtol=0, atol=1e-12)
        np.testing.assert_allclose(D1 @ D1.T, np.eye(n), rtol=0, atol=1e-12)


def test_mean_quaternion_and_normal_follow_the_4x4_correction():
    """x' = (new @ inv(old)) x, R(q') = dR R(q) for a raw (unnormalised) q with |q'| = |q|, n' = dR n, and the anchor's
    camera centre maps onto the new one exactly."""
    rng = np.random.default_rng(3)
    for _ in range(ROTS):
        old = mo.random_pose(rng)
        new = mo.corrected_pose(rng, old)
        q_d, R, t = mo.anchor_transform(old, new)
        T = new @ np.linalg.inv(old)
        np.testing.assert_allclose(R, T[:3, :3], rtol=0, atol=1e-12)
        assert q_d[0] >= 0 and abs(np.linalg.norm(q_d) - 1) < 1e-14
        x = rng.normal(size=(20, 3)) * 3
        np.testing.assert_allclose(x @ R.T + t, (np.c_[x, np.ones(20)] @ T.T)[:, :3], rtol=0, atol=1e-12)
        np.testing.assert_allclose(old[:3, 3] @ R.T + t, new[:3, 3], rtol=0, atol=1e-12)
        q = rng.normal(size=(20, 4)) * rng.uniform(0.3, 3, (20, 1))
        q2 = mo.quat_mul(q_d, q)
        np.testing.assert_allclose(np.linalg.norm(q2, axis=1), np.linalg.norm(q, axis=1), rtol=1e-14)
        from scipy.spatial.transform import Rotation
        Rq = Rotation.from_quat(q[:, [1, 2, 3, 0]]).as_matrix()
        Rq2 = Rotation.from_quat(q2[:, [1, 2, 3, 0]]).as_matrix()
        np.testing.assert_allclose(Rq2, T[:3, :3] @ Rq, rtol=0, atol=1e-12)
        n = mo.unit_dirs(20, rng)
        np.testing.assert_allclose(n @ R.T, (np.c_[n, np.zeros(20)] @ T.T)[:, :3], rtol=0, atol=1e-12)


def test_oracle_leaves_unanchored_unmoved_and_out_of_range_rows_alone():
    rng = np.random.default_rng(4)
    P, K = 64, 5
    params = {"xyz": rng.normal(size=(P, 3)), "rotation": rng.normal(size=(P, 4)), "normal": mo.unit_dirs(P, rng),
              "features_rest": rng.normal(size=(P, 15, 3))}
    old = np.stack([mo.random_pose(rng) for _ in range(K)])
    new = np.stack([mo.corrected_pose(rng, o) for o in old])
    new[2] = old[2]
    anchor = rng.integers(-1, K, P)
    anchor[:4] = [7, -5, K, -1]
    out, moved, n_skipped = mo.transform(params, anchor, old, new)
    assert n_skipped == 3
    keep = ~moved
    assert not moved[(anchor == -1) | (anchor == 2) | (anchor >= K) | (anchor < -1)].any()
    for k in params:
        np.testing.assert_array_equal(out[k][keep], params[k][keep])
        assert not np.allclose(out[k][moved], params[k][moved])


def test_struct_layout_matches_the_header():
    S = _lib.RtgMapTransform
    assert C.sizeof(S) == 4 * 4 + 8 * 8
    offs = {n: getattr(S, n).offset for n in ("P", "K", "sh_rest", "anchor", "old_c2w", "new_c2w", "xyz", "rotation", "normal",
                                              "features_rest", "n_skipped")}
    assert offs == dict(P=0, K=4, sh_rest=8, anchor=16, old_c2w=24, new_c2w=32, xyz=40, rotation=48, normal=56,
                        features_rest=64, n_skipped=72)


def test_c_entry_point_validates_before_touching_cuda():
    L = _lib.lib()
    assert L.rtg_map_transform_workspace_bytes(1000) >= 1000 * (1 + 4 + 9 + 3 + 83) * 4
    assert L.rtg_map_transform_workspace_bytes(0) == 0
    assert L.rtg_map_transform(None, None, None) == -1 and b"xf is NULL" in L.rtg_last_error()
    xf = _lib.RtgMapTransform(P=-1, K=3)
    assert L.rtg_map_transform(C.byref(xf), None, None) == -1 and b"bad sizes" in L.rtg_last_error()
    xf = _lib.RtgMapTransform(P=4, K=-2)
    assert L.rtg_map_transform(C.byref(xf), None, None) == -1 and b"bad sizes" in L.rtg_last_error()
    for bad in (1, 2, 4, 16, -3):
        xf = _lib.RtgMapTransform(P=4, K=3, sh_rest=bad)
        assert L.rtg_map_transform(C.byref(xf), None, None) == -1 and b"sh_rest" in L.rtg_last_error()
    xf = _lib.RtgMapTransform(P=4, K=3, sh_rest=15)
    assert L.rtg_map_transform(C.byref(xf), None, None) == -1 and b"n_skipped" in L.rtg_last_error()
    fake = 1 << 20  # never dereferenced: every case below fails on the host
    xf = _lib.RtgMapTransform(P=4, K=3, sh_rest=15, n_skipped=fake, anchor=fake, old_c2w=fake, new_c2w=fake, xyz=fake)
    assert L.rtg_map_transform(C.byref(xf), C.c_void_p(fake), None) == -1 and b"NULL pointer" in L.rtg_last_error()
    xf.rotation = fake
    assert L.rtg_map_transform(C.byref(xf), C.c_void_p(fake), None) == -1 and b"features_rest" in L.rtg_last_error()
    xf.features_rest, xf.sh_rest = fake, 0
    assert L.rtg_map_transform(C.byref(xf), C.c_void_p(fake), None) == -1 and b"features_rest" in L.rtg_last_error()
    xf.sh_rest = 8
    assert L.rtg_map_transform(C.byref(xf), None, None) == -1 and b"NULL pointer" in L.rtg_last_error()
    assert L.rtg_map_transform(C.byref(xf), C.c_void_p(fake + 4), None) == -1 and b"16-byte" in L.rtg_last_error()
    xf = _lib.RtgMapTransform(P=4, K=0, sh_rest=0, n_skipped=fake, xyz=fake, rotation=fake)   # K == 0 still needs the rows
    assert L.rtg_map_transform(C.byref(xf), None, None) == -1 and b"NULL pointer" in L.rtg_last_error()


def _poses(K, seed=0):
    rng = np.random.default_rng(seed)
    old = np.stack([mo.random_pose(rng) for _ in range(K)])
    return old, np.stack([mo.corrected_pose(rng, o) for o in old])


def test_python_transform_validates_poses_and_tensors_on_the_host():
    old, new = _poses(3)
    xyz = torch.zeros(4, 3)
    params = {"xyz": xyz, "rotation": torch.zeros(4, 4)}
    anchor = torch.zeros(4, dtype=torch.int32)
    for bad in (old[:, :3], old[0], np.zeros((3, 4, 3))):
        with pytest.raises(ValueError, match="shape"):
            mapsurgery.transform(params, anchor, bad, new)
    b = old.copy(); b[1, 0, 0] = np.nan
    with pytest.raises(ValueError, match="non-finite"):
        mapsurgery.transform(params, anchor, b, new)
    b = new.copy(); b[2, 3, 0] = 1e-3
    with pytest.raises(ValueError, match="last row"):
        mapsurgery.transform(params, anchor, old, b)
    b = new.copy(); b[0, :3, :3] *= 1 + 1e-4
    with pytest.raises(ValueError, match="orthonormal"):
        mapsurgery.transform(params, anchor, old, b)
    b = new.copy(); b[0, :3, 0] *= -1
    with pytest.raises(ValueError, match="det > 0"):
        mapsurgery.transform(params, anchor, old, b)
    with pytest.raises(ValueError, match="differ in shape"):
        mapsurgery.transform(params, anchor, old, new[:2])
    ok = old.copy(); ok[0, :3, :3] *= 1 + 1e-6                          # drift inside the tolerance is accepted ...
    with pytest.raises(TypeError, match="CUDA"):                         # ... and the tensor checks follow
        mapsurgery.transform(params, anchor, torch.from_numpy(ok), new)


def test_python_transform_rejects_cpu_tensors_wrong_dtypes_and_shapes():
    """Tensor checks need a CUDA tensor to get past the device test; without a GPU only the CPU / dtype rejections run."""
    old, new = _poses(2)
    params = {"xyz": torch.zeros(4, 3), "rotation": torch.zeros(4, 4)}
    with pytest.raises(TypeError, match="CUDA"):
        mapsurgery.transform(params, torch.zeros(4, dtype=torch.int32), old, new)
    params = {"xyz": torch.zeros(4, 3, dtype=torch.float64), "rotation": torch.zeros(4, 4)}
    with pytest.raises(TypeError, match="float32"):
        mapsurgery.transform(params, torch.zeros(4, dtype=torch.int32), old, new)
    with pytest.raises(TypeError):
        mapsurgery.transform({"xyz": torch.zeros(4), "rotation": torch.zeros(4, 4)}, torch.zeros(4, dtype=torch.int32), old, new)
