"""Per-Gaussian contributions of one oracle forward -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The statement of rtg_splat_contributions: a pair (pixel p, Gaussian g) adds colour when g sits at a position < n_contrib(p)
of p's tile list, power <= 0 and alpha = min(0.99, o exp(power)) >= 1/255; its weight is w = alpha T with T the product of
(1 - alpha) over the pairs in front of it that add colour. It reads an OracleRender's own forward state -- geom()'s xy and
conic_opacity, binning()'s tile lists and image_state()'s n_contrib -- and walks each pixel's prefix as tools/visit_stats.py
does, in the oracle's precision, so the T_threshold and opaque-hit decisions are the oracle's (n_contrib). For the
antialiased mode pass an AntialiasedOracleRender: its conic_opacity holds o comp. Only tests/ and tools/ import it.
"""
from __future__ import annotations

import numpy as np

CHUNK = 1024  # list entries per step of a tile's walk (bounds the (16, 16, CHUNK) temporaries)


def contributions(o, pixel_error=None, pixels=None):
    """{"n_pixels", "weight"[, "error"], "in_prefix"}: (P,) arrays (int64 counts, weights in the oracle's precision).
    `pixel_error`: (H, W) per-pixel error. "in_prefix" counts, per Gaussian, the pixels whose walked prefix (the first
    n_contrib(p) entries of the tile list) contains it, restricted to the boolean (H, W) `pixels` when given."""
    H, W, P, dt = o.H, o.W, o.P, o.dt
    geo = o.geom()
    xy, co = geo["xy"], geo["conic_opacity"]
    pl, rg = o.binning()
    _, nc = o.image_state()
    tw = (W + 15) // 16
    n_pix = np.zeros(P, np.int64)
    in_prefix = np.zeros(P, np.int64)
    weight = np.zeros(P, dt)
    err = None if pixel_error is None else np.zeros(P, dt)
    e_img = None if pixel_error is None else np.asarray(pixel_error, dt).reshape(H, W)
    sel_img = np.ones((H, W), bool) if pixels is None else np.asarray(pixels, bool).reshape(H, W)
    for t in range(len(rg)):
        r0, r1 = int(rg[t, 0]), int(rg[t, 1])
        if r0 == r1:
            continue
        ty, tx = divmod(t, tw)
        y0, x0 = ty * 16, tx * 16
        ys, xs = np.mgrid[y0:min(y0 + 16, H), x0:min(x0 + 16, W)]
        last = nc[ys, xs].astype(np.int64)
        m = int(last.max())
        if m == 0:
            continue
        e = None if e_img is None else e_img[ys, xs]
        sel = sel_img[ys, xs]
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
            pre = pos[None, None, :] < last[..., None]
            ok = pre & (power <= 0) & (alpha >= dt(1.0 / 255.0))
            alpha = np.where(ok, alpha, dt(0))
            # T in front of each entry, multiplied entry by entry in list order as the forward does (a skipped pair
            # multiplies by exactly 1)
            Tin = np.empty(alpha.shape, dt)
            for j in range(len(ids)):
                Tin[..., j] = T
                T = T * (1 - alpha[..., j])
            w = alpha * Tin
            np.add.at(n_pix, ids, ok.sum(axis=(0, 1)))
            np.add.at(in_prefix, ids, (pre & sel[..., None]).sum(axis=(0, 1)))
            np.add.at(weight, ids, w.sum(axis=(0, 1)))
            if err is not None:
                np.add.at(err, ids, (w * e[..., None]).sum(axis=(0, 1)))
    out = {"n_pixels": n_pix, "weight": weight, "in_prefix": in_prefix}
    if err is not None:
        out["error"] = err
    return out
