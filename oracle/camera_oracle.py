"""Camera gradient of the rasterizer oracle -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The reference has no camera gradient, so there is nothing of it to restate line by line. This module states it
independently of any hand-derived chain: the per-Gaussian quantities that depend on the camera are written as a torch
function of (viewmatrix, projmatrix, campos) and differentiated by autograd, in the oracle's precision, with the
oracle's own per-Gaussian backward intermediates (splat_oracle.c) as the upstream gradient:

    conic (a, b, c) of the EWA splat   <- dL/dconic        (colour path through alpha)
    NDC centre clip.xy / clip.w        <- dL/dmean2D       (W/2, H/2 pixels per NDC unit are inside it)
    SH colour at mean - campos         <- dL/dcolor, 0 where the colour was clamped
    depth of the first opaque surfel   <- dL/ddepth        (plane or centre-depth branch)

The discrete decisions (culling, tile cut-off, alpha < 1/255, opaque hit, plane test) are taken from the oracle's
forward / its backward's rule and held fixed, as the per-Gaussian gradients hold them. The 1.3 tanfov clamp of the EWA
Jacobian is restated as a forward expression; the reference's backward treats a clamped centre differently, but a
Gaussian that survives the cull (|NDC| <= 1.3 of a symmetric frustum) is not clamped. Finite differences of the oracle's
forward pin this module (tests/test_camera_grad_cpu.py). Only tests/ import it.
"""
from __future__ import annotations

import numpy as np
import torch

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435)


def _sh_rgb(deg, sh, d):
    """computeColorFromSH (forward.cu:104-155) before the +0.5 and the clamp; sh (P,M,3), d (P,3) unit directions."""
    x, y, z = (d[:, i:i + 1] for i in range(3))
    r = SH_C0 * sh[:, 0]
    if deg > 0:
        r = r - SH_C1 * y * sh[:, 1] + SH_C1 * z * sh[:, 2] - SH_C1 * x * sh[:, 3]
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        r = (r + SH_C2[0] * xy * sh[:, 4] + SH_C2[1] * yz * sh[:, 5] + SH_C2[2] * (2 * zz - xx - yy) * sh[:, 6]
             + SH_C2[3] * xz * sh[:, 7] + SH_C2[4] * (xx - yy) * sh[:, 8])
    if deg > 2:
        r = (r + SH_C3[0] * y * (3 * xx - yy) * sh[:, 9] + SH_C3[1] * xy * z * sh[:, 10]
             + SH_C3[2] * y * (4 * zz - xx - yy) * sh[:, 11] + SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[:, 12]
             + SH_C3[4] * x * (4 * zz - xx - yy) * sh[:, 13] + SH_C3[5] * z * (xx - yy) * sh[:, 14]
             + SH_C3[6] * x * (xx - 3 * yy) * sh[:, 15])
    return r


def _quat_R(q):
    r, x, y, z = q.unbind(-1)
    return torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
                        torch.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
                        torch.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def camera_gradient(o, dL_dcolor, dL_ddepth, grads=None):
    """dL/d(viewmatrix (4,4), projmatrix (4,4), campos (3,)) of the oracle render `o` (an OracleRender) for the upstream
    (dL/dcolor (3,H,W), dL/ddepth (1,H,W)); `grads` = o.backward(dL_dcolor, dL_ddepth) if already computed. Arrays are in
    the storage the rasterizer reads (viewmatrix = W2C transposed). Computed in the oracle's precision."""
    dt = torch.float32 if o.dt == np.float32 else torch.float64
    t = lambda a: torch.as_tensor(np.asarray(a), dtype=dt)
    V = o.V
    if grads is None:
        grads = o.backward(dL_dcolor, dL_ddepth)
    vm = t(np.array(V.view[:])).reshape(4, 4).requires_grad_(True)
    pm = t(np.array(V.proj[:])).reshape(4, 4).requires_grad_(True)
    cp = t(np.array(V.campos[:])).requires_grad_(True)
    H, W = o.H, o.W
    fx, fy = t(W / (2 * V.tanfovx)), t(H / (2 * V.tanfovy))
    geom = o.geom()
    vis = np.where(o.radii > 0)[0]
    mean = t(o.means[vis])
    mh = torch.cat([mean, torch.ones((len(vis), 1), dtype=dt)], 1)
    loss = torch.zeros((), dtype=dt)

    # EWA splat: t = view-space centre, J = d(pixel)/d(t) with the 1.3 tanfov clamp, A = J W, cov2D = A Sigma A^T + 0.3
    p = (mh @ vm)[:, :3]
    limx, limy = 1.3 * V.tanfovx, 1.3 * V.tanfovy
    tx = torch.clamp(p[:, 0] / p[:, 2], -limx, limx) * p[:, 2]
    ty = torch.clamp(p[:, 1] / p[:, 2], -limy, limy) * p[:, 2]
    tz = p[:, 2]
    zero = torch.zeros_like(tz)
    J = torch.stack([torch.stack([fx / tz, zero, -(fx * tx) / (tz * tz)], -1),
                     torch.stack([zero, fy / tz, -(fy * ty) / (tz * tz)], -1)], 1)
    A = J @ vm[:3, :3].T
    c6 = t(geom["cov3D"][vis])
    S = torch.stack([torch.stack([c6[:, 0], c6[:, 1], c6[:, 2]], -1), torch.stack([c6[:, 1], c6[:, 3], c6[:, 4]], -1),
                     torch.stack([c6[:, 2], c6[:, 4], c6[:, 5]], -1)], 1)
    cov2 = A @ S @ A.transpose(1, 2)
    a, b, c = cov2[:, 0, 0] + 0.3, cov2[:, 0, 1], cov2[:, 1, 1] + 0.3
    det = a * c - b * b
    con = t(grads["conic"][vis])
    # the reference's dL/dconic keeps half the gradient of the off-diagonal entry (backward.cu:985-988; its conic
    # backward, :344-348, doubles it again): the true dL/d(conic.y) is twice the stored value
    loss = loss + (con[:, 0] * c / det + 2 * con[:, 1] * (-b / det) + con[:, 3] * a / det).sum()

    # projection: NDC centre = clip.xy / (clip.w + 1e-7)
    clip = mh @ pm
    ndc = clip[:, :2] / (clip[:, 3:4] + 1e-7)
    loss = loss + (t(grads["means2D"][vis, :2]) * ndc).sum()

    # SH colour (not for precomputed colours): the clamp at 0 passes no gradient
    if o.shs is not None:
        d = mean - cp
        d = d / torch.sqrt((d * d).sum(1, keepdim=True))
        rgb = _sh_rgb(int(V.sh_degree), t(o.shs[vis]), d)
        keep = t(1 - geom["clamped"][vis].astype(np.int64))
        loss = loss + (t(grads["colors"][vis]) * keep * rgb).sum()

    # depth of the first opaque Gaussian of every pixel (backward.cu:997-1065): plane intersection of the surfel, or its
    # view-space centre depth; without a surfel (cov3D_precomp) always the centre depth
    # only pixels of tiles that were rendered: elsewhere (masked-out or empty tiles) the hit map keeps its initial 0
    hid = o.hit_depth[0]
    _, ranges = o.binning()
    rendered = (ranges[:, 1] > ranges[:, 0]).reshape((H + 15) // 16, (W + 15) // 16)
    rendered = np.repeat(np.repeat(rendered, 16, 0), 16, 1)[:H, :W]
    pys, pxs = np.nonzero((hid >= 0) & rendered)
    gid = hid[pys, pxs]
    gd = t(np.asarray(dL_ddepth).reshape(H, W)[pys, pxs])
    ray = torch.stack([(t(pxs) - V.cx) / fx, (t(pys) - V.cy) / fy, torch.ones(len(pxs), dtype=dt)], 1)
    ray = ray / torch.sqrt((ray * ray).sum(1, keepdim=True))
    mg = t(o.means[gid])
    pc = (torch.cat([mg, torch.ones((len(gid), 1), dtype=dt)], 1) @ vm)[:, :3]
    if o.cov3D_precomp is not None or len(gid) == 0:
        depth = pc[:, 2]
    else:
        sc = o.scales[gid]
        axis = np.argmin(sc, 1)  # ties: first index, as arg_min3
        nw = _quat_R(t(o.rots[gid]))[torch.arange(len(gid)), :, torch.as_tensor(axis)]
        nc = nw @ vm[:3, :3]
        num = (pc * nc).sum(1)
        ndotr = (nc * ray).sum(1)
        tt = num / (ndotr + 1e-8)
        with torch.no_grad():  # the backward's plane test: max(scales) without the modifier (backward.cu:1009)
            plane = ((tt * ray[:, 2] - pc[:, 2]).abs() <= V.depth_threshold * t(sc.max(1))) & (ndotr.abs() >= V.normal_threshold)
        depth = torch.where(plane, tt * ray[:, 2], pc[:, 2])
    loss = loss + (gd * depth).sum()

    gv, gp, gc = torch.autograd.grad(loss, [vm, pm, cp], allow_unused=True)
    out = lambda g, n: np.zeros(n, o.dt) if g is None else g.detach().numpy().astype(o.dt)
    return {"viewmatrix": out(gv, (4, 4)), "projmatrix": out(gp, (4, 4)), "campos": out(gc, 3)}
