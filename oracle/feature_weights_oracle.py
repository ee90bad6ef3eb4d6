"""The weight gradient of a feature map -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

rtg_splat_features_backward_geometry differentiates the feature map A F (oracle/features_oracle.py) through its blend
weights w = alpha T, with the features F and the upstream G = dL/dmap held. The weights do not depend on colour, so the map
is linear in F, and three of its channels are the colour image of a forward with colors_precomp = those three columns of
F and a zero background. The gradient of <G, A F> with respect to the Gaussians' geometry and the camera is therefore

    sum over channel triples t of  OracleRender.backward(dL/dcolor = G[t], dL/ddepth = 0)  with colors_precomp = F[:, t], bg = 0

(the last triple padded with zero channels), and likewise of camera_oracle.camera_gradient, and of AntialiasedOracleRender
and its camera_gradient for the antialiased mode. The blended pairs and their weights are the same in every such forward:
the decisions read no colour. Only tests/ and tools/ import it.
"""
from __future__ import annotations

import numpy as np

from oracle import antialias_oracle, camera_oracle
from oracle.antialias_oracle import AntialiasedOracleRender
from oracle.splat_oracle import OracleRender

GEOMETRY = ("means3D", "opacities", "scales", "rotations", "cov3D_precomp")


def weight_gradient(cam, g, F, G, tile_mask=None, cov3D_precomp=None, antialiased=False, camera=False, precision="f64",
                    **settings):
    """(per-Gaussian gradients {means3D, opacities, scales, rotations} or {means3D, opacities, cov3D_precomp}, camera
    gradient {viewmatrix, projmatrix, campos} or None) of <G, A F>. g: the Gaussians as OracleRender takes them (its SH
    colours are not read); F (P, C); G (C, H, W); `settings` as OracleRender takes them (bg is forced to 0)."""
    H, W = cam.height, cam.width
    P = g["xyz"].shape[0]
    dt = np.float64 if precision == "f64" else np.float32
    F = np.asarray(F, np.float64).reshape(P, -1)
    G = np.asarray(G, np.float64).reshape(-1, H, W)
    Cn = F.shape[1]
    pad = (-Cn) % 3
    F = np.concatenate([F, np.zeros((P, pad))], 1)
    G = np.concatenate([G, np.zeros((pad, H, W))], 0)
    cls = AntialiasedOracleRender if antialiased else OracleRender
    cam_grad = antialias_oracle.camera_gradient if antialiased else camera_oracle.camera_gradient
    st = dict(settings, bg=(0.0, 0.0, 0.0))
    zero_depth = np.zeros((1, H, W), dt)
    grads, cams = {}, None
    for t in range(0, Cn + pad, 3):
        o = cls(cam, g, tile_mask=tile_mask, precision=precision, colors_precomp=F[:, t:t + 3],
                cov3D_precomp=cov3D_precomp, **st)
        gc = G[t:t + 3].astype(dt)
        gr = o.backward(gc, zero_depth)
        for k in GEOMETRY:
            if k in gr:
                grads[k] = grads.get(k, 0.0) + gr[k].astype(np.float64)
        if camera:
            c = cam_grad(o, gc, zero_depth, grads=gr)
            cams = {k: v.astype(np.float64) for k, v in c.items()} if cams is None else {k: cams[k] + c[k] for k in cams}
        o.close()
    return grads, cams
