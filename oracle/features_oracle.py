"""Per-Gaussian feature maps of one oracle forward -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The statement of rtg_splat_features and its backward: with A the (pixels x Gaussians) matrix of the forward's colour
weights, A[p, g] = w(p, g) = alpha T for the pairs that add colour (the pairs of oracle/contrib_oracle.py: g at a
position < n_contrib(p) of p's tile list, power <= 0 and alpha = min(0.99, o exp(power)) >= 1/255; T the product of
(1 - alpha) over the pairs in front of it), the feature map is A F and the feature gradient A^T G. It reads an
OracleRender's own geometry, tile lists and n_contrib, in the oracle's precision. For the antialiased mode pass an
AntialiasedOracleRender: its conic_opacity holds o comp. Only tests/ and tools/ import it.
"""
from __future__ import annotations

import numpy as np

CHUNK = 1024  # list entries per step of a tile's walk (bounds the (16, 16, CHUNK) temporaries)


def _weights(o):
    """Yields (ys, xs, ids, w) per tile and list chunk: w (h, w, len(ids)) the colour weights of the tile's pixels
    (ys, xs) with the Gaussians ids (0 where a pair adds no colour)."""
    H, W, dt = o.H, o.W, o.dt
    geo = o.geom()
    xy, co = geo["xy"], geo["conic_opacity"]
    pl, rg = o.binning()
    _, nc = o.image_state()
    tw = (W + 15) // 16
    for t in range(len(rg)):
        r0, r1 = int(rg[t, 0]), int(rg[t, 1])
        if r0 == r1:
            continue
        ty, tx = divmod(t, tw)
        y0, x0 = ty * 16, tx * 16
        ys, xs = np.mgrid[y0:min(y0 + 16, H), x0:min(x0 + 16, W)]
        last = nc[ys, xs].astype(np.int64)
        m = int(last.max())
        pxf, pyf = xs.astype(dt)[..., None], ys.astype(dt)[..., None]
        T = np.ones(ys.shape, dt)
        for k0 in range(0, m, CHUNK):
            ids = pl[r0 + k0:r0 + min(m, k0 + CHUNK)]
            pos = np.arange(k0, k0 + len(ids))
            dx, dy = xy[ids, 0] - pxf, xy[ids, 1] - pyf
            a, b, c, op = co[ids, 0], co[ids, 1], co[ids, 2], co[ids, 3]
            power = dt(-0.5) * (a * dx * dx + c * dy * dy) - b * dx * dy
            with np.errstate(over="ignore"):
                alpha = np.minimum(dt(0.99), op * np.exp(np.minimum(power, 0)))
            ok = (pos[None, None, :] < last[..., None]) & (power <= 0) & (alpha >= dt(1.0 / 255.0))
            alpha = np.where(ok, alpha, dt(0))
            Tin = np.empty(alpha.shape, dt)
            for j in range(len(ids)):  # entry by entry in list order, as the forward multiplies
                Tin[..., j] = T
                T = T * (1 - alpha[..., j])
            yield ys, xs, ids, alpha * Tin


def features(o, F=None, G=None):
    """{"map": A F (C, H, W) when F (P, C) is given, "grad": A^T G (P, C) when G (C, H, W) is given}, in the oracle's
    precision. Pixels outside rendered tiles are 0 in the map and contribute nothing to the gradient."""
    H, W, P, dt = o.H, o.W, o.P, o.dt
    F = None if F is None else np.asarray(F, dt).reshape(P, -1)
    G = None if G is None else np.asarray(G, dt).reshape(-1, H, W)
    out = {}
    if F is not None:
        out["map"] = np.zeros((F.shape[1], H, W), dt)
    if G is not None:
        out["grad"] = np.zeros((P, G.shape[0]), dt)
    for ys, xs, ids, w in _weights(o):
        if F is not None:
            out["map"][:, ys, xs] += np.einsum("yxl,lc->cyx", w, F[ids], optimize=True)
        if G is not None:
            np.add.at(out["grad"], ids, np.einsum("yxl,cyx->lc", w, G[:, ys, xs], optimize=True))
    return out
