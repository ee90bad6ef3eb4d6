"""RGB-D ICP: the point-to-plane ICP of icp_oracle with a photometric term -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only tests/ and tools/ import it. The statement, shared with rtg_icp_predict_pose_rgbd and DESIGN.md:

* Intensity pyramid. Per full-resolution pixel Y = 0.299 R + 0.587 G + 0.114 B; level pixel (y, x) with pool p is the
  mean of Y over the p x p block whose maximum the depth pyramid takes (same grid, same level intrinsics).
* Photometric row. "0" is the current frame, "1" the previous one. For a pixel q whose geometric row is valid
  (icp_oracle.residuals_jacobian), v' = R v0 + t = (x, y, z) projects to u = fx x/z + cx, v = fy y/z + cy (0 < u < W-1,
  0 < v < H-1). With x0 = floor(u), y0 = floor(v), alpha = u - x0, beta = v - y0, I1(u, v) is the bilinear interpolation
  of the previous frame's level intensity over the four taps, r = I1(u, v) - I0[q], and
      gu = (1-beta)(I10 - I00) + beta(I11 - I01),  gv = (1-alpha)(I01 - I00) + alpha(I11 - I10)
  (I10 is the tap at x0+1, I01 the one at y0+1: the exact derivative of the interpolant),
      a = (gu fx/z, gv fy/z, -(gu fx x + gv fy y)/z^2),  J = (v' x a, a).
* Step. H = sum_geo J^T J + w sum_photo J^T J, g = sum_geo J^T r + w sum_photo J^T r; damping, solve and update as in
  icp_oracle.icp_level.

Rows are computed in the input dtype, as icp_oracle computes them, so a float32 run makes the kernel's association
decisions. The geometric sums are icp_oracle's own; the photometric sums are in float64 and are added to them in float64,
so w = 0 reproduces icp_oracle.icp_level exactly.
"""
from __future__ import annotations

import numpy as np

from oracle import icp_oracle as io

LUMA = (0.299, 0.587, 0.114)


def intensity_pyramid(color, n_levels=3, channels_last=True):
    """Index 0 = coarsest (pool 2**(n_levels-1)), in the dtype of `color` ((H,W,3) or, with channels_last=False, (3,H,W))."""
    c = np.asarray(color)
    if not channels_last:
        c = np.moveaxis(c, 0, -1)
    dt = c.dtype
    Y = dt.type(LUMA[0]) * c[..., 0] + dt.type(LUMA[1]) * c[..., 1] + dt.type(LUMA[2]) * c[..., 2]
    H, W = Y.shape
    out = []
    for i in range(n_levels):
        p = 1 << (n_levels - 1 - i)
        Hs, Ws = H // p, W // p
        out.append(Y[: Hs * p, : Ws * p].reshape(Hs, p, Ws, p).astype(np.float64).mean(axis=(1, 3)).astype(dt))
    return out


def project(pose, v0, K):
    dt = v0.dtype
    fx, fy, cx, cy = [dt.type(k) for k in K]
    R, t = pose[:3, :3].astype(dt), pose[:3, 3].astype(dt)
    V = v0.reshape(-1, 3) @ R.T + t
    with np.errstate(divide="ignore", invalid="ignore"):
        u = (V[:, 0] / V[:, 2]) * fx + cx
        v = (V[:, 1] / V[:, 2]) * fy + cy
    return V, u, v


def photometric_rows(pose, v0, v1, n0, n1, I0, I1, K, dist_thr, cos_thr):
    """(r (HW,), J (HW, 6), valid (HW,)): the photometric rows of the pixels whose geometric row is valid, zero elsewhere."""
    H, W, _ = v0.shape
    dt = v0.dtype
    _, _, valid = io.residuals_jacobian(pose, v0, v1, n0, n1, K, dist_thr, cos_thr)
    V, u, v = project(pose, v0, K)
    fx, fy = dt.type(K[0]), dt.type(K[1])
    r = np.zeros(H * W, dtype=dt)
    J = np.zeros((H * W, 6), dtype=dt)
    q = np.nonzero(valid)[0]
    uq, vq = u[q], v[q]
    x0, y0 = np.floor(uq), np.floor(vq)
    al, be = (uq - x0).astype(dt), (vq - y0).astype(dt)
    xi, yi = x0.astype(np.int64), y0.astype(np.int64)
    I1 = np.asarray(I1, dtype=dt)
    i00, i10, i01, i11 = I1[yi, xi], I1[yi, xi + 1], I1[yi + 1, xi], I1[yi + 1, xi + 1]
    one = dt.type(1)
    Iw = (one - be) * ((one - al) * i00 + al * i10) + be * ((one - al) * i01 + al * i11)
    r[q] = Iw - np.asarray(I0, dtype=dt).reshape(-1)[q]
    gu = (one - be) * (i10 - i00) + be * (i11 - i01)
    gv = (one - al) * (i01 - i00) + al * (i11 - i10)
    x, y, z = V[q, 0], V[q, 1], V[q, 2]
    a = np.stack([gu * fx / z, gv * fy / z, -(gu * fx * x + gv * fy * y) / (z * z)], axis=-1).astype(dt)
    J[q, :3] = np.cross(V[q], a)
    J[q, 3:] = a
    return r, J, valid


def icp_level_rgbd(pose, v0, v1, n0, n1, I0, I1, K, iters, dist_thr=0.1, normal_thr_deg=20.0, damping=1e-4,
                   photometric_weight=0.01, solve_dtype=None):
    """`iters` damped Gauss-Newton steps with both terms. Returns (pose, valid_ratio, photometric_ratio, photometric_rmse),
    the ratios and the RMS of the last iteration before its step."""
    dt = v0.dtype
    cos_thr = np.cos(np.deg2rad(normal_thr_deg))
    pose = np.asarray(pose, dtype=dt)
    H, W = v0.shape[:2]
    vr, pr, prmse = 0.0, 0.0, 0.0
    w = float(photometric_weight)
    for _ in range(iters):
        res, J, valid = io.residuals_jacobian(pose, v0, v1, n0, n1, K, dist_thr, cos_thr)
        rp, Jp, _ = photometric_rows(pose, v0, v1, n0, n1, I0, I1, K, dist_thr, cos_thr)
        Jp64, rp64 = Jp.astype(np.float64), rp.astype(np.float64)
        JtJ = ((J.T @ J).astype(dt).astype(np.float64) + w * (Jp64.T @ Jp64)).astype(dt)
        JtR = ((J.T @ res).astype(dt).astype(np.float64) + w * (Jp64.T @ rp64)).astype(dt)
        Hm = JtJ + np.trace(JtJ) * dt.type(damping) * np.eye(6, dtype=dt)
        sd = solve_dtype or dt
        xi = (-(np.linalg.inv(Hm.astype(sd)) @ JtR.astype(sd))).astype(dt)
        pose = (io.exp_se3(xi) @ pose).astype(dt)
        n = int(valid.sum())
        vr, pr = n / H / W, n / H / W
        prmse = float(np.sqrt((rp64 * rp64).sum() / n)) if n else 0.0
    return pose, vr, pr, prmse


def predict_pose_rgbd(depth_prev, depth_curr, color_prev, color_curr, K, iters=(5, 5, 5), downscales=(0.25, 0.5, 1.0),
                      dist_thr=0.1, normal_thr_deg=20.0, damping=1e-4, fail_threshold=0.02, photometric_weight=0.01,
                      channels_last=True):
    """RgbdIcpTracker.predict_pose for two RGB-D frames: (pose 4x4, p2ploss, valid_ratio, success, photometric_ratio,
    photometric_rmse)."""
    dt = np.asarray(depth_curr).dtype
    n = len(downscales)
    v_t0, n_t0 = io.build_pyramids(depth_prev, K, n)
    v_t1, n_t1 = io.build_pyramids(depth_curr, K, n)
    i_t0 = intensity_pyramid(np.asarray(color_prev, dtype=dt), n, channels_last)
    i_t1 = intensity_pyramid(np.asarray(color_curr, dtype=dt), n, channels_last)
    pose = np.eye(4, dtype=dt)
    vr = pr = prmse = 0.0
    for lvl, s in enumerate(downscales):
        Kl = tuple(dt.type(k) * dt.type(s) for k in K)
        pose, vr, pr, prmse = icp_level_rgbd(pose, v_t1[lvl], v_t0[lvl], n_t1[lvl], n_t0[lvl], i_t1[lvl], i_t0[lvl], Kl,
                                             iters[lvl], dist_thr, normal_thr_deg, damping, photometric_weight)
    p = v_t1[-1].reshape(-1, 3) @ pose[:3, :3].T + pose[:3, 3]
    l = ((p - v_t0[-1].reshape(-1, 3)) * n_t0[-1].reshape(-1, 3)).sum(-1)
    loss = float((l * l).mean())
    return pose, loss, float(vr), not (loss > fail_threshold), float(pr), float(prmse)
