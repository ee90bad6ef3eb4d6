"""Rigid per-anchor map transform in float64 numpy -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

States `rtg_map_transform` (include/rtg_splat_b200.h) independently of the kernel: the anchor's rotation comes from
scipy's quaternion conversion, and the band-l SH rotation D^l is the least-squares solution of
    Y_l(R d) D^l = Y_l(d)    over sampled unit directions d,
where Y_l holds the band-l basis functions as `camera_oracle._sh_rgb` (the restatement of computeColorFromSH) evaluates
them. The kernel integrates the same matrix with a quadrature rule over its own copy of the basis, so the two cannot share
a sign or ordering mistake. Only tests/ import it.
"""
from __future__ import annotations

import numpy as np
import torch
from scipy.spatial.transform import Rotation

from oracle.camera_oracle import _sh_rgb

BANDS = {1: slice(1, 4), 2: slice(4, 9), 3: slice(9, 16)}   # coefficient indices of band l in the (M, 3) SH block


def sh_basis(d):
    """(N, 16) float64: the 16 basis functions of the rasterizer's SH colour at the unit directions d (N, 3)."""
    d = torch.as_tensor(np.asarray(d, np.float64))
    n = d.shape[0]
    sh = torch.zeros((16, n, 16, 3), dtype=torch.float64)   # coefficient m set to 1 in block m
    sh[torch.arange(16), :, torch.arange(16), 0] = 1.0
    return _sh_rgb(3, sh.reshape(16 * n, 16, 3), d.repeat(16, 1))[:, 0].reshape(16, n).T.numpy()


def sh_eval(f, d):
    """Colour without the DC offset/clamp: f (N, M, 3) coefficients at directions d (N, 3) -> (N, 3)."""
    Y = sh_basis(d)[:, : f.shape[1]]
    return np.einsum("nm,nmc->nc", Y, f)


def unit_dirs(n, rng):
    d = rng.normal(size=(n, 3))
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def sh_rotation(R, l, n_dirs=100, seed=0):
    """(2l+1, 2l+1) D^l with sh(D f, R d) = sh(f, d) for band l, by least squares over n_dirs random directions."""
    d = unit_dirs(n_dirs, np.random.default_rng(seed))
    b = BANDS[l]
    A = sh_basis(d @ np.asarray(R, np.float64).T)[:, b]
    B = sh_basis(d)[:, b]
    return np.linalg.lstsq(A, B, rcond=None)[0]


def anchor_transform(old_c2w, new_c2w):
    """(q_delta (4,) w >= 0, R (3,3) rebuilt from it, t (3,)) of one anchor, float64."""
    old_c2w, new_c2w = np.asarray(old_c2w, np.float64), np.asarray(new_c2w, np.float64)
    dR = new_c2w[:3, :3] @ old_c2w[:3, :3].T
    x, y, z, w = Rotation.from_matrix(dR).as_quat()
    q = np.array([w, x, y, z])
    q = (q if q[0] >= 0 else -q) / np.linalg.norm(q)
    R = Rotation.from_quat([q[1], q[2], q[3], q[0]]).as_matrix()
    return q, R, new_c2w[:3, 3] - R @ old_c2w[:3, 3]


def quat_mul(a, b):
    """Hamilton product of (w,x,y,z) quaternions, broadcasting over leading dimensions."""
    aw, ax, ay, az = np.moveaxis(a, -1, 0)
    bw, bx, by, bz = np.moveaxis(b, -1, 0)
    return np.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                     aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], -1)


def transform(params, anchor, old_c2w, new_c2w, rows=None):
    """Expected result of rtg_map_transform, float64. params: numpy "xyz", "rotation", optional "normal",
    "features_rest" (P, M-1, 3); anchor (P,) int. rows: indices to evaluate (default all). Returns (dict of the moved
    arrays restricted to `rows`, moved mask over `rows`, number of out-of-range anchors over all rows)."""
    anchor = np.asarray(anchor).reshape(-1)
    K = len(old_c2w)
    rows = np.arange(len(anchor)) if rows is None else np.asarray(rows)
    n_skipped = int(((anchor != -1) & ((anchor < 0) | (anchor >= K))).sum())
    a = anchor[rows]
    valid = (a >= 0) & (a < K)
    changed = np.array([not np.array_equal(o, n) for o, n in zip(old_c2w, new_c2w)], bool)
    moved = np.zeros(len(rows), bool)
    moved[valid] = changed[a[valid]]
    out = {k: np.asarray(v, np.float64)[rows].copy() for k, v in params.items()}
    for k in np.unique(a[moved]):
        sel = moved & (a == k)
        q, R, t = anchor_transform(old_c2w[k], new_c2w[k])
        out["xyz"][sel] = out["xyz"][sel] @ R.T + t
        out["rotation"][sel] = quat_mul(q, out["rotation"][sel])
        if "normal" in out:
            out["normal"][sel] = out["normal"][sel] @ R.T
        if "features_rest" in out:
            M = out["features_rest"].shape[1] + 1
            for l, b in BANDS.items():
                if b.stop <= M:
                    D = sh_rotation(R, l)
                    rb = slice(b.start - 1, b.stop - 1)
                    out["features_rest"][sel, rb] = np.einsum("ij,njc->nic", D, out["features_rest"][sel, rb])
    return out, moved, n_skipped


def random_rotation(rng, max_deg):
    """A rotation about a random axis by an angle uniform in [0, max_deg] degrees."""
    axis = unit_dirs(1, rng)[0]
    return Rotation.from_rotvec(axis * np.deg2rad(rng.uniform(0, max_deg))).as_matrix()


def random_pose(rng, extent=3.0):
    T = np.eye(4)
    T[:3, :3] = Rotation.random(random_state=rng).as_matrix()
    T[:3, 3] = rng.uniform(-extent, extent, 3)
    return T


def corrected_pose(rng, c2w, max_deg=45.0, max_trans=2.0):
    """c2w moved by a rigid correction of at most max_deg degrees and max_trans metres."""
    T = np.eye(4)
    T[:3, :3] = random_rotation(rng, max_deg)
    v = unit_dirs(1, rng)[0]
    T[:3, 3] = v * rng.uniform(0, max_trans)
    return T @ c2w
