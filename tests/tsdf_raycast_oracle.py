"""The TSDF ray-cast in float64 numpy -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates `rtg_tsdf_raycast` (include/rtg_splat_b200.h) from its rules: the piecewise-linear field on the Kuhn tetrahedra
of `oracle/tsdf_oracle.extract`, cells walked in ray order, each cut at the planes u_a = u_b into pieces of one
tetrahedron, the first sign change deciding. All rays step through the cell walk in lockstep, so a 640x480 image takes
seconds. `ray_mesh` intersects rays with a triangle list by brute force, so that tests can hold `raycast` to `extract`.
Grids are (nz, ny, nx) arrays, x fastest, as in oracle/tsdf_oracle.py.
"""
from __future__ import annotations

import numpy as np

TIE_F = 1e-6      # |f| at a piece endpoint up to the decision
TIE_U = 1e-7      # local coordinates of the hit from a tetrahedron or cell boundary
TIE_EDGE = 1e-7   # voxel sizes from a cell edge where the ray crosses a cell face before its decision


def rays(w2c, K, H, W):
    """(o (3,), d (3, H*W)) float64: pixel (u, v) has the ray o + t d with o = -R^T t, d = R^T ((u-cx)/fx, (v-cy)/fy, 1),
    w2c as the device reads it and K = (fx, fy, cx, cy) as float32 values. t is camera z."""
    fx, fy, cx, cy = (float(np.float32(k)) for k in K)
    P = np.asarray(w2c).astype(np.float64)
    v, u = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    dcx, dcy = ((u - cx) / fx).ravel(), ((v - cy) / fy).ravel()
    o = np.array([-(P[0, a] * P[0, 3] + P[1, a] * P[1, 3] + P[2, a] * P[2, 3]) for a in range(3)])
    d = np.stack([P[0, a] * dcx + P[1, a] * dcy + P[2, a] for a in range(3)])
    return o, d


def _perm(m0, m1, m2):
    """Axes (p1, p2, p3) ordering (m0, m1, m2) decreasingly, ties to the lower axis."""
    a, b, c = m0 >= m1, m1 >= m2, m0 >= m2
    p1 = np.where(a, np.where(b | c, 0, 2), np.where(c | b, 1, 2))
    p2 = np.where(a, np.where(b, 1, np.where(c, 2, 0)), np.where(c, 0, np.where(b, 2, 1)))
    return p1, p2, 3 - p1 - p2


def raycast(tsdf, weight, color, origin, voxel_size, w2c, K, H, W, tie_u=TIE_U):
    """{"depth": (H, W), "normal": (3, H, W), "color": (3, H, W) or None, "hit": (H, W) bool, "tie": (H, W) bool}, float64.
    `tie` flags pixels whose outcome may differ between this statement and a device evaluation: a piece endpoint at or
    before the decision with |f| < TIE_F, a hit within tie_u (local coordinates) of a tetrahedron or cell boundary, a ray
    crossing a cell face within TIE_EDGE voxels of a cell edge before its decision."""
    nz, ny, nx = tsdf.shape
    n = np.array([nx, ny, nz])
    org = np.asarray(origin, np.float32).astype(np.float64)
    s = float(np.float32(voxel_size))
    o, d = rays(w2c, K, H, W)
    R = H * W
    l = np.repeat(((o - org) / s)[:, None], R, axis=1)
    dg = d / s
    fl = np.asarray(tsdf, np.float64).ravel()
    ob = (np.asarray(weight) > 0).ravel()
    ng = (np.asarray(tsdf) < 0).ravel() & ob
    colf = None if color is None else np.asarray(color, np.float64).reshape(3, -1)
    step = np.array([1, nx, nx * ny])
    offs = np.array([(q & 1) + ((q >> 1) & 1) * nx + ((q >> 2) & 1) * nx * ny for q in range(8)])
    # cells a crossing can happen in: corners 0 and 7 observed, an observed corner of each sign
    cand = np.zeros((nz, ny, nx), bool)
    if min(n) > 1:
        ob3, ng3 = ob.reshape(nz, ny, nx), ng.reshape(nz, ny, nx)
        corner = lambda a, q: a[(q >> 2) & 1:nz - 1 + ((q >> 2) & 1), (q >> 1) & 1:ny - 1 + ((q >> 1) & 1),  # noqa: E731
                                q & 1:nx - 1 + (q & 1)]
        any_neg = np.zeros((nz - 1, ny - 1, nx - 1), bool)
        any_pos = np.zeros((nz - 1, ny - 1, nx - 1), bool)
        for q in range(8):
            any_neg |= corner(ng3, q)
            any_pos |= corner(ob3, q) & ~corner(ng3, q)
        cand[:-1, :-1, :-1] = corner(ob3, 0) & corner(ob3, 7) & any_neg & any_pos
    cand = cand.ravel()

    depth, normal, col = np.zeros(R), np.zeros((3, R)), np.zeros((3, R))
    hit, tie = np.zeros(R, bool), np.zeros(R, bool)
    t_in, t_out = np.zeros(R), np.full(R, np.inf)
    live = np.full(R, bool(min(n) > 1))
    with np.errstate(divide="ignore", invalid="ignore"):
        for a in range(3):
            hi = float(n[a] - 1)
            moving = dg[a] != 0
            ta, tb = -l[a] / dg[a], (hi - l[a]) / dg[a]
            t_in = np.where(moving, np.fmax(t_in, np.fmin(ta, tb)), t_in)
            t_out = np.where(moving, np.fmin(t_out, np.fmax(ta, tb)), t_out)
            live &= moving | ((l[a] >= 0) & (l[a] <= hi))
    live &= t_in < t_out
    idx = np.nonzero(live)[0]
    L, D = l[:, idx], dg[:, idx]
    p_in = L + t_in[idx] * D
    near_int = np.abs(p_in - np.rint(p_in)) < TIE_EDGE
    tie[idx] |= near_int.sum(0) >= 2                                     # entering at a cell edge
    c = np.fmin(np.fmax(np.floor(p_in), 0.0), (n - 2)[:, None]).astype(np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):
        tn = np.where(D > 0, (c + 1 - L) / D, np.where(D < 0, (c - L) / D, np.inf))
    t0, T_out = t_in[idx], t_out[idx]
    sgn = np.where(D > 0, 1, -1)
    base = (c * step[:, None]).sum(0)
    finished = np.zeros(idx.size, bool)
    while idx.size:
        m = idx.size
        ar = np.arange(m)
        ax = np.argmin(tn, axis=0)
        t1 = np.fmin(tn[ax, ar], T_out)
        done = finished.copy()
        sel = np.nonzero(~finished & cand[base] & (t1 > t0))[0]
        if sel.size:
            done[sel] = _cells(sel, L, D, c, base, t0, t1, fl, ob, colf, offs, idx, depth, normal, col, hit, tie, tie_u)
        done |= t1 >= T_out
        # step into the next cell; a face crossing near a cell edge is a tie when a cell around that edge could hold a
        # crossing (elsewhere the walk may take either side of the edge without a decision depending on it)
        pg = L + t1 * D
        fr = np.abs(pg - np.rint(pg)) < TIE_EDGE
        fr[ax, ar] = False
        near = np.nonzero(~done & fr.any(0))[0]
        if near.size:
            lo = c[:, near].copy()
            hi = lo.copy()
            a_ = ax[near]
            hi[a_, np.arange(near.size)] += sgn[a_, near]
            for b_ in range(3):
                k_ = np.rint(pg[b_, near]).astype(np.int64)
                e_ = fr[b_, near]
                lo[b_, e_], hi[b_, e_] = k_[e_] - 1, k_[e_]
            lo = np.clip(np.minimum(lo, hi), 0, (n - 2)[:, None])
            hi = np.clip(np.maximum(lo, hi), 0, (n - 2)[:, None])
            around = np.zeros(near.size, bool)
            for q in range(8):
                cell = np.where(np.array([(q >> a) & 1 for a in range(3)])[:, None] == 1, hi, lo)
                around |= cand[(cell * step[:, None]).sum(0)]
            tie[idx[near[around]]] = True
        t0 = t1
        sa = np.where(done, 0, sgn[ax, ar])
        ca = c[ax, ar] + sa
        out = (ca < 0) | (ca > n[ax] - 2)
        done |= out
        sa = np.where(out, 0, sa)                             # the cell of a finished ray stays in the grid
        ca = c[ax, ar] + sa
        c[ax, ar] = ca
        base = base + sa * step[ax]
        with np.errstate(divide="ignore", invalid="ignore"):
            tn[ax, ar] = np.where(sgn[ax, ar] > 0, (ca + 1) - L[ax, ar], ca - L[ax, ar]) / D[ax, ar]
        finished = done
        if finished.mean() > 0.25 or finished.all():          # drop the finished rays now and then
            keep = ~finished
            idx, L, D, c, tn, t0, T_out, sgn, base = (idx[keep], L[:, keep], D[:, keep], c[:, keep], tn[:, keep], t0[keep],
                                                      T_out[keep], sgn[:, keep], base[keep])
            finished = finished[keep]
    out = {"depth": depth.reshape(H, W), "normal": normal.reshape(3, H, W), "color": None, "hit": hit.reshape(H, W),
           "tie": tie.reshape(H, W)}
    if color is not None:
        out["color"] = col.reshape(3, H, W)
    return out


def _cells(sel, L, D, c, base, t0, t1, fl, ob, colf, offs, idx, depth, normal, col, hit, tie, tie_u):
    """The pieces of the candidate cells of rays `sel` in ray order; writes hits, flags ties, returns the decided rays."""
    k = sel.size
    ar = np.arange(k)
    u = L[:, sel] - c[:, sel]
    dg = D[:, sel]
    ta0, ta4 = t0[sel], t1[sel]
    with np.errstate(divide="ignore", invalid="ignore"):
        s01 = (u[1] - u[0]) / (dg[0] - dg[1])
        s02 = (u[2] - u[0]) / (dg[0] - dg[2])
        s12 = (u[2] - u[1]) / (dg[1] - dg[2])
    s01, s02, s12 = (np.where((x > ta0) & (x < ta4), x, ta4) for x in (s01, s02, s12))
    b = [ta0, np.fmin(np.fmin(s01, s02), s12), np.fmax(np.fmin(s01, s02), np.fmin(np.fmax(s01, s02), s12)),
         np.fmax(np.fmax(s01, s02), s12), ta4]
    cb = base[sel]
    f8 = np.stack([fl[cb + offs[q]] for q in range(8)])
    o8 = np.stack([ob[cb + offs[q]] for q in range(8)])
    state = np.zeros(k, np.int8)
    g_idx = idx[sel]
    for i in range(4):
        ta, tb = b[i], b[i + 1]
        act = (state == 0) & (tb > ta)
        mid = 0.5 * (ta + tb)
        mm = u + mid * dg
        p1, p2, p3 = _perm(mm[0], mm[1], mm[2])
        q1 = 1 << p1
        q2 = q1 | (1 << p2)
        ok = act & o8[q1, ar] & o8[q2, ar]
        f0, f1, f2, f3 = f8[0], f8[q1, ar], f8[q2, ar], f8[7]
        g1, g2, g3 = f1 - f0, f2 - f1, f3 - f2
        ua1, ua2, ua3 = u[p1, ar], u[p2, ar], u[p3, ar]
        d1, d2, d3 = dg[p1, ar], dg[p2, ar], dg[p3, ar]
        fa = f0 + g1 * (ua1 + ta * d1) + g2 * (ua2 + ta * d2) + g3 * (ua3 + ta * d3)
        fb = f0 + g1 * (ua1 + tb * d1) + g2 * (ua2 + tb * d2) + g3 * (ua3 + tb * d3)
        tie[g_idx[ok & ((np.abs(fa) < TIE_F) | (np.abs(fb) < TIE_F))]] = True
        back = ok & (fa < 0) & (fb >= 0)
        front = ok & (fa >= 0) & (fb < 0)
        state[back] = 2
        state[front] = 1
        h = np.nonzero(front)[0]
        if h.size == 0:
            continue
        with np.errstate(divide="ignore", invalid="ignore"):
            ts = ta[h] + (tb[h] - ta[h]) * fa[h] / (fa[h] - fb[h])
        gi = g_idx[h]
        hit[gi] = True
        depth[gi] = ts
        gw = np.zeros((3, h.size))
        for gv, p in ((g1, p1), (g2, p2), (g3, p3)):
            gw[p[h], np.arange(h.size)] = gv[h]
        normal[:, gi] = gw / np.sqrt((gw * gw).sum(0))
        hu = u[:, h] + ts * dg[:, h]
        near = np.minimum(np.minimum(hu, 1 - hu).min(0),
                          np.minimum(np.abs(hu[0] - hu[1]), np.minimum(np.abs(hu[0] - hu[2]), np.abs(hu[1] - hu[2]))))
        tie[gi[near < tie_u]] = True
        if colf is not None:
            h1, h2, h3 = hu[p1[h], np.arange(h.size)], hu[p2[h], np.arange(h.size)], hu[p3[h], np.arange(h.size)]
            w = (1.0 - h1, h1 - h2, h2 - h3, h3)
            cs = cb[h]
            for ch in range(3):
                col[ch, gi] = (w[0] * colf[ch, cs] + w[1] * colf[ch, cs + offs[q1[h]]] + w[2] * colf[ch, cs + offs[q2[h]]]
                               + w[3] * colf[ch, cs + offs[7]])
    return state != 0


def ray_mesh(vertices, faces, origins, dirs, chunk=(4096, 1024)):
    """First intersection with t > 0 of each ray origins + t dirs ((R, 3) or (3,) and (R, 3); t in units of dirs) with the
    triangles `faces` of `vertices`, brute force in float64: a bounding-sphere cull, then Moller-Trumbore on the pairs
    left. {"t": (R,) inf where none, "face": (R,) -1 where none, "front": (R,) bool, the hit triangle's right-handed normal
    against the ray, "bary": (R, 3) weights of its three vertices at the hit}."""
    V = np.asarray(vertices, np.float64)
    F = np.asarray(faces, np.int64)
    Dr = np.asarray(dirs, np.float64)
    R = Dr.shape[0]
    O = np.broadcast_to(np.asarray(origins, np.float64), (R, 3))
    A, B, Cv = V[F[:, 0]], V[F[:, 1]], V[F[:, 2]]
    ctr = (A + B + Cv) / 3
    rad = np.sqrt(np.maximum(np.maximum(((A - ctr) ** 2).sum(1), ((B - ctr) ** 2).sum(1)), ((Cv - ctr) ** 2).sum(1)))
    Dn = Dr / np.linalg.norm(Dr, axis=1, keepdims=True)
    best_t, best_f = np.full(R, np.inf), np.full(R, -1)
    best_uv = np.zeros((R, 2))
    c2 = (ctr * ctr).sum(1)
    for r0 in range(0, R, chunk[1]):
        o, dn, dr = O[r0:r0 + chunk[1]], Dn[r0:r0 + chunk[1]], Dr[r0:r0 + chunk[1]]
        for f0 in range(0, len(F), chunk[0]):
            m, rr = ctr[f0:f0 + chunk[0]], rad[f0:f0 + chunk[0]]
            proj = m @ dn.T - (o * dn).sum(1)[None]
            dist2 = c2[f0:f0 + chunk[0], None] - 2 * m @ o.T + (o * o).sum(1)[None] - proj * proj
            ti, ri = np.nonzero((dist2 <= (rr[:, None] * (1 + 1e-6) + 1e-9) ** 2) & (proj >= -rr[:, None] - 1e-9))
            if ti.size == 0:
                continue
            fi, gi = ti + f0, ri + r0
            a, e1, e2 = A[fi], B[fi] - A[fi], Cv[fi] - A[fi]
            dd = dr[ri]
            pv = np.cross(dd, e2)
            det = (e1 * pv).sum(1)
            with np.errstate(divide="ignore", invalid="ignore"):
                inv = 1.0 / det
                tv = o[ri] - a
                uu = (tv * pv).sum(1) * inv
                qv = np.cross(tv, e1)
                vv = (dd * qv).sum(1) * inv
                t = (e2 * qv).sum(1) * inv
            ok = (det != 0) & (uu >= 0) & (vv >= 0) & (uu + vv <= 1) & (t > 0)
            fi, gi, t, uu, vv = fi[ok], gi[ok], t[ok], uu[ok], vv[ok]
            order = np.lexsort((t, gi))                  # per ray, nearest first
            gi, fi, t, uu, vv = gi[order], fi[order], t[order], uu[order], vv[order]
            first = np.concatenate([[True], gi[1:] != gi[:-1]]) if gi.size else np.zeros(0, bool)
            gi, fi, t, uu, vv = gi[first], fi[first], t[first], uu[first], vv[first]
            better = t < best_t[gi]
            gi, fi, t, uu, vv = gi[better], fi[better], t[better], uu[better], vv[better]
            best_t[gi], best_f[gi] = t, fi
            best_uv[gi] = np.stack([uu, vv], 1)
    nrm = np.cross(B - A, Cv - A)
    hitm = best_f >= 0
    front = np.zeros(R, bool)
    front[hitm] = (nrm[best_f[hitm]] * Dr[hitm]).sum(1) < 0
    bary = np.stack([1 - best_uv[:, 0] - best_uv[:, 1], best_uv[:, 0], best_uv[:, 1]], 1)
    return {"t": best_t, "face": best_f, "front": front, "bary": bary}
