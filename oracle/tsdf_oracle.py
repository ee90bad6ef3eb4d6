"""TSDF fusion and marching-tetrahedra extraction in float64 numpy -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates `rtg_tsdf_integrate` and `rtg_tsdf_extract_count` / `rtg_tsdf_extract_emit` (include/rtg_splat_b200.h) from
their rules, vectorised over the whole grid. Grids are (nz, ny, nx) arrays (x fastest, as the device stores them); voxel
(i, j, k) sits at origin + s * (i, j, k). The triangle table is derived here from the tetrahedron's orientation, not
copied: tests compare it with the kernel's. Only tests/ import it.
"""
from __future__ import annotations

import itertools

import numpy as np

# edge slot -> corner offset (dx, dy, dz): +x, +y, +z, +x+y, +y+z, +x+z, +x+y+z
SLOT_OFFSETS = ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (0, 1, 1), (1, 0, 1), (1, 1, 1))
# the six tetrahedra of a cell, one per axis permutation, in lexicographic order: c, c+e_p0, c+e_p0+e_p1, c+(1,1,1)
PERMUTATIONS = tuple(itertools.permutations(range(3)))
# the six edges of a tetrahedron as pairs of its path corners 0..3
TET_EDGES = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))

TIE_PIXEL = 1e-3     # px from a rounding boundary
TIE_TRUNC = 1e-5     # map units from -trunc
TIE_Z = 1e-6         # map units from the image plane


def _even(p):
    return sum(p[i] > p[j] for i in range(len(p)) for j in range(i + 1, len(p))) % 2 == 0


def _edge(a, b):
    return TET_EDGES.index((min(a, b), max(a, b)))


def tet_table():
    """(16, 2, 3) int: triangles of a positively oriented tetrahedron (det(p1-p0, p2-p0, p3-p0) > 0) per case
    (bit q set = corner q has tsdf < 0), as edge ids into TET_EDGES, -1 = no triangle. Winding is right-handed with the
    normal pointing from the negative corners to the positive ones.

    For an even permutation (a, b, c, d) of the corners, face (b, c, d) has its normal pointing away from a. So one negative
    corner a gives (ab, ac, ad); one positive corner a gives (ab, ad, ac); two negative corners a, b give the quad
    (ac, ad, bd, bc), split along the diagonal ac-bd."""
    table = -np.ones((16, 2, 3), dtype=np.int64)
    for case in range(16):
        neg = [q for q in range(4) if case >> q & 1]
        if len(neg) in (0, 4):
            continue
        for perm in itertools.permutations(range(4)):
            if not _even(perm):
                continue
            a, b, c, d = perm
            if len(neg) == 1 and neg == [a]:
                table[case, 0] = (_edge(a, b), _edge(a, c), _edge(a, d))
                break
            if len(neg) == 3 and a not in neg:
                table[case, 0] = (_edge(a, b), _edge(a, d), _edge(a, c))
                break
            if len(neg) == 2 and sorted(neg) == sorted((a, b)):
                ac, ad, bc, bd = _edge(a, c), _edge(a, d), _edge(b, c), _edge(b, d)
                table[case, 0] = (ac, ad, bd)
                table[case, 1] = (ac, bd, bc)
                break
    return table


def new_volume(dims, color=False):
    nx, ny, nz = dims
    tsdf = np.ones((nz, ny, nx))
    weight = np.zeros((nz, ny, nx))
    col = np.zeros((3, nz, ny, nx)) if color else None
    return tsdf, weight, col


def voxel_centres(origin, voxel_size, dims):
    """(3, nz, ny, nx) float64 world positions of the voxel centres (origin and voxel_size as the device holds them)."""
    nx, ny, nz = dims
    o = np.asarray(origin, np.float32).astype(np.float64)
    s = float(np.float32(voxel_size))
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    return np.stack([o[0] + s * i, o[1] + s * j, o[2] + s * k])


def integrate(tsdf, weight, color, origin, voxel_size, trunc, depth, w2c, K, color_img=None):
    """Folds one frame into (tsdf, weight, color) in place; returns the (nz, ny, nx) bool mask of tie voxels, whose
    outcome may differ between this float64 statement and a float32/float64 device evaluation. depth (H, W); color_img
    (H, W, 3) or None; w2c (4, 4) as the device reads it; K = (fx, fy, cx, cy) as float32 values."""
    fx, fy, cx, cy = (float(np.float32(k)) for k in K)
    tr = float(np.float32(trunc))
    depth = np.asarray(depth, np.float32).reshape(np.asarray(depth).shape[-2:])
    H, W = depth.shape
    P = np.asarray(w2c, np.float64)
    p = voxel_centres(origin, voxel_size, tsdf.shape[::-1])
    pc = np.einsum("ab,bzyx->azyx", P[:3, :3], p) + P[:3, 3, None, None, None]
    x, y, z = pc
    with np.errstate(divide="ignore", invalid="ignore"):
        u = fx * x / z + cx
        v = fy * y / z + cy
    front = z > 0
    ru, rv = np.rint(np.where(front, u, -1.0)), np.rint(np.where(front, v, -1.0))
    inside = front & (ru >= 0) & (ru <= W - 1) & (rv >= 0) & (rv <= H - 1)
    ui, vi = np.where(inside, ru, 0).astype(np.int64), np.where(inside, rv, 0).astype(np.int64)
    d = np.where(inside, depth[vi, ui].astype(np.float64), 0.0)
    seen = inside & (d > 0)
    sdf = d - z
    upd = seen & (sdf >= -tr)
    f = np.minimum(1.0, sdf / tr)
    w = weight
    tsdf[upd] = (tsdf[upd] * w[upd] + f[upd]) / (w[upd] + 1)
    if color is not None:
        c = np.asarray(color_img, np.float32).astype(np.float64)[vi, ui]        # (nz, ny, nx, 3)
        for ch in range(3):
            color[ch][upd] = (color[ch][upd] * w[upd] + c[..., ch][upd]) / (w[upd] + 1)
    weight[upd] += 1
    with np.errstate(invalid="ignore"):
        near_half = lambda t: np.abs(t - np.floor(t) - 0.5) < TIE_PIXEL  # noqa: E731
        tie = np.abs(z) < TIE_Z
        tie |= front & (near_half(u) | near_half(v))
        tie |= seen & (np.abs(sdf + tr) < TIE_TRUNC)
    return tie


def _popc(m):
    m = m.astype(np.int64)
    return sum((m >> b) & 1 for b in range(7))


def extract(tsdf, weight, color, origin, voxel_size):
    """Marching tetrahedra on the Kuhn decomposition: (vertices (V, 3) f64, faces (F, 3) int64, colours (V, 3) or None),
    vertices ordered by (owning voxel, edge slot), faces by (cell, tetrahedron, triangle)."""
    nz, ny, nx = tsdf.shape
    o = np.asarray(origin, np.float32).astype(np.float64)
    s = float(np.float32(voxel_size))
    f = np.asarray(tsdf, np.float64)
    w = np.asarray(weight, np.float64)
    neg = f < 0
    obs = w > 0
    mask = np.zeros((nz, ny, nx), np.int64)
    verts = []   # (lin, slot, position (3,n), colour (3,n) | None)
    lin_all = np.arange(nx * ny * nz).reshape(nz, ny, nx)
    for slot, (dx, dy, dz) in enumerate(SLOT_OFFSETS):
        a = (slice(0, nz - dz), slice(0, ny - dy), slice(0, nx - dx))
        b = (slice(dz, nz), slice(dy, ny), slice(dx, nx))
        has = obs[a] & obs[b] & (neg[a] != neg[b])
        mask[a] |= has.astype(np.int64) << slot
        kk, jj, ii = np.nonzero(has)
        fa, fb = f[a][has], f[b][has]
        tau = fa / (fa - fb)
        pa = np.stack([o[0] + s * ii, o[1] + s * jj, o[2] + s * kk])
        pb = np.stack([o[0] + s * (ii + dx), o[1] + s * (jj + dy), o[2] + s * (kk + dz)])
        pos = pa + tau * (pb - pa)
        col = None
        if color is not None:
            ca = np.stack([color[c][a][has] for c in range(3)])
            cb = np.stack([color[c][b][has] for c in range(3)])
            col = ca + tau * (cb - ca)
        verts.append((lin_all[a][has], np.full(len(tau), slot), pos, col))
    lin = np.concatenate([v[0] for v in verts])
    slot = np.concatenate([v[1] for v in verts])
    order = np.lexsort((slot, lin))
    vertices = np.concatenate([v[2] for v in verts], axis=1).T[order]
    colors = np.concatenate([v[3] for v in verts], axis=1).T[order] if color is not None else None
    counts = _popc(mask).reshape(-1)
    voff = np.concatenate([[0], np.cumsum(counts)[:-1]])
    mflat = mask.reshape(-1)

    table = tet_table()
    cell = (slice(0, nz - 1), slice(0, ny - 1), slice(0, nx - 1))
    clin = lin_all[cell].reshape(-1)
    corner = lambda q: (slice((q >> 2) & 1, nz - 1 + ((q >> 2) & 1)), slice((q >> 1) & 1, ny - 1 + ((q >> 1) & 1)),  # noqa: E731
                        slice(q & 1, nx - 1 + (q & 1)))
    step = {0: 1, 1: nx, 2: nx * ny}
    faces = []   # (cell lin, tet, tri, (n,3) vertex ids)
    for t, perm in enumerate(PERMUTATIONS):
        path = [0, 1 << perm[0], (1 << perm[0]) | (1 << perm[1]), 7]
        case = np.zeros(clin.shape, np.int64)
        allobs = np.ones(clin.shape, bool)
        for q, c in enumerate(path):
            case |= neg[corner(c)].reshape(-1).astype(np.int64) << q
            allobs &= obs[corner(c)].reshape(-1)
        for r in range(2):
            tri = table[case, r]                         # (n, 3) edge ids
            ok = allobs & (tri[:, 0] >= 0)
            ids = np.zeros((int(ok.sum()), 3), np.int64)
            for e in range(3):
                qa = np.array([TET_EDGES[x][0] for x in range(6)])[tri[ok, e]]
                qb = np.array([TET_EDGES[x][1] for x in range(6)])[tri[ok, e]]
                ca, cb = np.array(path)[qa], np.array(path)[qb]
                own = clin[ok] + sum(((ca >> ax) & 1) * step[ax] for ax in range(3))
                sl = np.array([SLOT_OFFSETS.index(((d >> 0) & 1, (d >> 1) & 1, (d >> 2) & 1)) if d else -1 for d in range(8)])[cb ^ ca]
                ids[:, e] = voff[own] + _popc(mflat[own] & ((1 << sl) - 1))
            if not _even(perm):                          # an odd permutation gives a negatively oriented tetrahedron
                ids = ids[:, [0, 2, 1]]
            faces.append((clin[ok], np.full(len(ids), t), np.full(len(ids), r), ids))
    key_c = np.concatenate([x[0] for x in faces])
    key_t = np.concatenate([x[1] for x in faces])
    key_r = np.concatenate([x[2] for x in faces])
    order = np.lexsort((key_r, key_t, key_c))
    tris = np.concatenate([x[3] for x in faces])[order]
    return vertices, tris, colors


def sphere_grid(dims, voxel_size, centre, radius, trunc):
    """Truncated signed distance to a sphere, (tsdf, weight = 1) on a grid at origin 0."""
    p = voxel_centres((0.0, 0.0, 0.0), voxel_size, dims)
    sdf = np.sqrt(((p - np.asarray(centre, np.float64)[:, None, None, None]) ** 2).sum(0)) - radius
    return np.clip(sdf / trunc, -1.0, 1.0), np.ones(sdf.shape)


def plane_grid(dims, voxel_size, normal, offset, trunc):
    """Truncated signed distance to the plane n . p = offset (n unit, pointing to the positive side), at origin 0."""
    p = voxel_centres((0.0, 0.0, 0.0), voxel_size, dims)
    n = np.asarray(normal, np.float64)
    sdf = np.einsum("a,azyx->zyx", n, p) - offset
    return np.clip(sdf / trunc, -1.0, 1.0), np.ones(sdf.shape)
