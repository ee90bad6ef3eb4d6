"""Row-wise comparison of rasterizer gradients with the float64 oracle, and scenes that reach every branch of the
depth-hit path. Shared by test_raster_grad_rows_cpu.py (float32 oracle against float64 oracle: the rehearsal of the
metric) and test_raster_grad_rows_gpu.py (the kernels against the float64 oracle).

Why rows. `helpers.rel_err` divides by the largest entry of a whole tensor, so a Gaussian whose gradient is a thousand
times smaller than the largest one may be wrong by 100 % unseen. Here every visible Gaussian i of every tensor is held to

    e_i = max_j |g_ij - ref_ij|  <=  RTOL * n_i + C * max_i n_i,        n_i = max_j |ref_ij|

(for the gradients behind the 2-D covariance RTOL grows with the square of that covariance's condition number once it
passes 30, see `covariance_condition`).

The absolute term C * max n covers rows that are a cancelling sum of much larger per-pixel terms (an opacity gradient
whose colour terms cancel): their float32 rounding error scales with the terms, not with the sum. `ratio` below is
e_i / (RTOL * n_i + C * max n); a comparison passes when every row's ratio is <= 1.

Two things make a row-wise comparison of a float32 result with a float64 one fair:

* Discrete decisions. A pixel whose alpha, transmittance, opaque-hit or plane test lies within `tie_eps` of its
  threshold may decide differently in the two precisions. `decision_mask` finds those pixels (the oracles' tie maps, plus
  every pixel whose hit / contributor indices differ between the float32 oracle, the float64 oracle and the GPU forward)
  and the upstream gradients are zeroed there before both backwards run. Every term of the backward is linear in the
  pixel's upstream gradient, so a zeroed pixel contributes exactly nothing on either side and both sides replay the same
  decisions.
* Per-Gaussian decisions (`comparable_rows`): a radius that rounds to a different integer, an SH colour channel within
  1e-5 of the clamp at 0, two scales within 1e-6 (argmin / argmax tie). Such rows are left out, counted, and the count is
  bounded."""
from __future__ import annotations

import numpy as np

from oracle.splat_oracle import OracleRender
from rtg_slam_b200 import scene
from test_camera_grad_cpu import compact_scene
from test_camera_grad_gpu import scene_case as _base_scene_case

RTOL = 1e-3
C = 5e-6
LOSSES = ("mixed", "colour", "depth")
SH_SRC = {"means3D": "xyz", "opacities": "opacity"}
# largest share of the image decision_mask may take out: the translucent blobs of `dense` / `oversized` stack hundreds of
# splats per pixel, each a chance to sit within tie_eps of a threshold
MAX_MASKED_SHARE = {"dense": 0.35, "oversized": 0.35}
MAX_EXCLUDED_SHARE = 1e-3


# ----------------------------------------------------------------------------------------------------------- scenes
_CYCLE = {0: (2, 0, 1), 1: (1, 2, 0), 2: (0, 1, 2)}           # new local axis j is old local axis _CYCLE[k][j]
_CYCLE_Q = {0: (0.5, -0.5, -0.5, -0.5), 1: (0.5, 0.5, 0.5, 0.5), 2: (1.0, 0.0, 0.0, 0.0)}   # the same relabelling, R' = R(q) R(c)


def axis_permute(g, seed):
    """Relabels the local axes of every Gaussian by a cyclic permutation chosen per Gaussian, so that the thin axis (2 in
    `g`) becomes 0, 1 or 2 with equal probability. Scales and quaternion change together: the covariance and the surfel
    normal stay what they were. Returns (new dict, thin axis per Gaussian)."""
    P = len(g["xyz"])
    k = np.random.default_rng(seed).integers(0, 3, P)
    out = dict(g)
    sc, q = g["scales"].astype(np.float64), g["rotations"].astype(np.float64)
    sc2, q2 = sc.copy(), q.copy()
    for a in range(3):
        m = k == a
        sc2[m] = sc[m][:, list(_CYCLE[a])]
        q2[m] = scene._quat_mul(q[m], np.tile(np.array(_CYCLE_Q[a]), (int(m.sum()), 1)))
    out["scales"] = np.ascontiguousarray(sc2.astype(g["scales"].dtype))
    out["rotations"] = np.ascontiguousarray(q2.astype(g["rotations"].dtype))
    return out, k


def axis_room(P, seed):
    """`scene.surfel_room` with the thin axis spread over 0, 1, 2 (`axis_permute`) and enough grazing surfels for the
    centre-depth fallback of the plane test: normals scattered by 40 degrees, and every third surfel six times as thick
    (0.6 r instead of 0.1 r: still the thin axis, but an edge-on surfel then covers pixels)."""
    g = scene.surfel_room(P, seed=seed, normal_sigma_deg=40.0)
    thick = np.random.default_rng(seed + 1).uniform(size=P) < 1 / 3
    g["scales"][thick, 2] *= 6.0
    return axis_permute(g, seed + 2)[0]


def axis_compact(P, seed):
    """`compact_scene` (float64, a few hundred overlapping surfels in a 64x48 view) for finite differences: a third of the
    surfels tilted 62-82 degrees away from the optical axis and thickened, then `axis_permute`."""
    g = compact_scene(P, seed)
    rng = np.random.default_rng(seed + 1)
    graze = rng.uniform(size=P) < 0.4
    tilt, az = np.deg2rad(rng.uniform(62, 82, P)), rng.uniform(0, 2 * np.pi, P)
    nrm = np.stack([np.sin(tilt) * np.cos(az), np.sin(tilt) * np.sin(az), np.cos(tilt)], 1)
    g["rotations"][graze] = scene._quat_z_to(nrm[graze])
    g["scales"][graze, 2] *= 5.0
    return axis_permute(g, seed + 2)[0]


def scene_case(name):
    """(camera, gaussians, tile mask): the scenes of test_camera_grad_gpu.scene_case, `axis_room`, and `oversized`
    (30 000 dense blobs in a 64x48 view: tile lists past the on-chip sort capacity)."""
    if name == "axis_room":
        return scene.make_camera("small", c2w=scene.small_pose()), axis_room(3000, seed=51), None
    if name == "oversized":
        return scene.make_camera("tiny"), scene.dense_blobs(30_000, seed=21), None
    return _base_scene_case(name)


def oracle_args(inputs, mask=None, over=None):
    """(g, kw) of OracleRender from a GaussianRasterizer input dict (test_camera_grad_gpu.inputs_for), a tile mask and
    settings overrides; float32 values, which either oracle precision converts exactly."""
    g = {k: inputs.get(k) for k in ("xyz", "opacity", "shs", "scales", "rotations")}
    kw = dict(over or {}, tile_mask=mask)
    for k in ("colors_precomp", "cov3D_precomp"):
        if inputs.get(k) is not None:
            kw[k] = inputs[k]
    return g, kw


def upstream(cam, loss, mask, seed=5):
    """(dL/dcolor, dL/ddepth) float32 of scene.upstream_grads, zero on the pixels of `mask`; `colour` / `depth` zero the
    other map."""
    gc, gd = scene.upstream_grads(cam, seed=seed)
    keep = (~mask).astype(np.float32)
    gc, gd = gc * keep[None], gd * keep[None]
    if loss == "colour":
        gd = np.zeros_like(gd)
    elif loss == "depth":
        gc = np.zeros_like(gc)
    else:
        assert loss == "mixed"
    return gc, gd


# --------------------------------------------------------------------------------------------------- what to compare
def forwards(cam, g, kw, tie_eps=1e-3):
    return tuple(OracleRender(cam, g, precision=p, tie_eps=tie_eps, **kw) for p in ("f32", "f64"))


def decision_mask(cam, g, kw, gpu_forward=None, tie_eps=1e-3, oracles=None):
    """Boolean (H, W): pixels to take out of the loss. `gpu_forward`: dict with the GPU's hit_color / hit_depth maps."""
    o32, o64 = oracles or forwards(cam, g, kw, tie_eps)
    mask = (o32.tie != 0) | (o64.tie != 0)
    mask |= (o32.hit_color[0] != o64.hit_color[0]) | (o32.hit_depth[0] != o64.hit_depth[0])
    mask |= o32.image_state()[1] != o64.image_state()[1]
    if gpu_forward is not None:
        for k in ("hit_color", "hit_depth"):
            mask |= np.asarray(gpu_forward[k]).reshape(mask.shape) != getattr(o64, k)[0]
    return mask


def thin_axis(g):
    return None if g.get("scales") is None else np.argmin(g["scales"], axis=1)


def _near_clamp(cam, g, kw, margin=1e-5):
    """Gaussians with an SH colour channel within `margin` of the clamp at 0: the clamp flags with every colour moved
    down and up by the margin differ. Preprocess only (no tile is rendered)."""
    th, tw = (cam.height + 15) // 16, (cam.width + 15) // 16
    flags = []
    for sgn in (-1.0, 1.0):
        shs = g["shs"].astype(np.float64)
        shs[:, 0] += sgn * margin / scene.SH_C0
        o = OracleRender(cam, dict(g, shs=shs), precision="f64", **dict(kw, tile_mask=np.zeros((th, tw), np.int32)))
        flags.append(o.geom()["clamped"].copy())
        o.close()
    return (flags[0] != flags[1]).any(axis=1)


def comparable_rows(cam, g, kw, o32, o64, gpu_radii=None):
    """(boolean (P,) of the rows to compare, {reason: rows left out}). Raises if more than MAX_EXCLUDED_SHARE of the
    visible rows (at least one row is always allowed) are left out."""
    vis = o64.radii > 0
    out = {"radii": o32.radii != o64.radii}
    if gpu_radii is not None:
        out["radii"] = out["radii"] | (np.asarray(gpu_radii).reshape(-1) != o64.radii)
    if "colors_precomp" not in kw:
        out["clamp"] = _near_clamp(cam, g, kw) | (o32.geom()["clamped"] != o64.geom()["clamped"]).any(axis=1)
    if g.get("scales") is not None:
        s = np.sort(g["scales"].astype(np.float64), axis=1)
        out["scale_tie"] = (np.diff(s, axis=1) <= 1e-6 * s[:, 1:]).any(axis=1)
    bad = np.zeros_like(vis)
    for v in out.values():
        bad |= v
    # a radius mismatch may be a visible / culled disagreement: count against either side's visible rows
    counts = {k: int((v & (vis | (k == "radii"))).sum()) for k, v in out.items()}
    total = int((bad & vis).sum()) + int((out["radii"] & ~vis).sum())
    assert total <= max(1, MAX_EXCLUDED_SHARE * int(vis.sum())), (counts, int(vis.sum()))
    return vis & ~bad, counts


def hit_pixels(o64, pixel_mask=None):
    """Boolean (H, W): pixels with a depth hit, inside the rendered tiles (elsewhere the hit map keeps its initial 0, which
    is not a hit) and outside `pixel_mask`."""
    up = np.kron(o64.tile_mask, np.ones((16, 16), np.int32))[: o64.H, : o64.W].astype(bool)
    return (o64.hit_depth[0] >= 0) & up & (np.ones_like(up) if pixel_mask is None else ~pixel_mask)


def hit_rows(o64, pixel_mask=None):
    """Boolean (P,): Gaussians that are the depth hit of at least one such pixel."""
    rows = np.zeros(len(o64.radii), bool)
    rows[o64.hit_depth[0][hit_pixels(o64, pixel_mask)]] = True
    return rows


def depth_coverage(o64, g, pixel_mask=None):
    """Depth-hit pixels of the float64 forward by (thin axis, branch): {(axis, "plane" | "centre"): (pixel count, sorted
    Gaussian indices)}. A hit pixel took the centre-depth fallback iff its depth is its Gaussian's centre depth. With
    scale_modifier == 1 the backward takes the same branch as the forward. A Gaussian with pixels on both branches is in
    both cells."""
    hit, depth = o64.hit_depth[0], o64.depth[0]
    ok = hit_pixels(o64, pixel_mask)
    ids = hit[ok]
    centre = depth[ok] == o64.geom()["depth"][ids]
    ax = thin_axis(g)[ids]
    cells = {}
    for a in range(3):
        for name, sel in (("plane", ~centre), ("centre", centre)):
            m = (ax == a) & sel
            cells[(a, name)] = (int(m.sum()), np.unique(ids[m]))
    return cells


def assert_coverage(cells, min_pixels=100, min_gaussians=20):
    short = {k: (n, len(ids)) for k, (n, ids) in cells.items() if n < min_pixels or len(ids) < min_gaussians}
    assert not short, f"depth-hit cells below {min_pixels} pixels / {min_gaussians} Gaussians: {short}"


# ------------------------------------------------------------------------------------------------------- the metric
def row_errors(g, ref, rows):
    """{tensor: (e, n)}: per row of `rows` the largest absolute error and the largest reference magnitude."""
    out = {}
    for k in ref:
        if k not in g:
            continue
        a = np.asarray(g[k], np.float64).reshape(len(rows), -1)[rows]
        b = np.asarray(ref[k], np.float64).reshape(len(rows), -1)[rows]
        out[k] = (np.abs(a - b).max(axis=1), np.abs(b).max(axis=1)) if a.shape[1] else (np.zeros(len(a)), np.zeros(len(a)))
    return out


COVARIANCE_CHAIN = ("scales", "rotations", "cov3D_precomp")
KAPPA_0 = 30.0


def covariance_condition(o64):
    """kappa = a c / (a c - b^2) of every Gaussian's 2-D covariance (from its conic; 1 where culled). The backward of the
    conic forms dL/d(a, b, c) as differences of terms of size kappa^2 times the result, so float32 loses kappa^2 * 6e-8 of
    the covariance-chain gradients of a needle seen along its length, in any correct implementation: measured 8e-4 on the
    float32 oracle at kappa = 54."""
    A, B, Cc = o64.geom()["conic_opacity"][:, :3].T
    det = A * Cc - B * B
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where((o64.radii > 0) & (det > 0), A * Cc / det, 1.0)


def row_tolerances(ref, rows, rtol=RTOL, c=C, kappa=None):
    """{tensor: rtol_i * n_i + c * max n}; rtol_i = rtol, times max(1, (kappa_i / KAPPA_0)^2) for the tensors behind the
    2-D covariance when `kappa` (covariance_condition) is given."""
    out = {}
    for k in ref:
        n = np.abs(np.asarray(ref[k], np.float64).reshape(len(rows), -1)[rows]).max(axis=1, initial=0.0)
        wide = np.maximum(1.0, (kappa[rows] / KAPPA_0) ** 2) if (kappa is not None and k in COVARIANCE_CHAIN) else 1.0
        out[k] = rtol * wide * n + c * (n.max() if n.size else 0.0)
    return out


def row_ratios(g, ref, rows, rtol=RTOL, c=C, kappa=None):
    """{tensor: e_i / tolerance_i} (0 where the error is 0, inf where only the tolerance is)."""
    tol = row_tolerances(ref, rows, rtol, c, kappa)
    out = {}
    for k, (e, n) in row_errors(g, ref, rows).items():
        with np.errstate(divide="ignore", invalid="ignore"):
            out[k] = np.where(e == 0, 0.0, e / tol[k])
    return out


def footprint_pixels(o64, i):
    """Pixels where Gaussian i alone reaches alpha >= 1/255 (occlusion and tile masks ignored)."""
    geom = o64.geom()
    (x, y), (a, b, c, op) = geom["xy"][i], geom["conic_opacity"][i]
    yy, xx = np.mgrid[0:o64.H, 0:o64.W]
    dx, dy = x - xx, y - yy
    power = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
    with np.errstate(over="ignore"):
        return int(((power <= 0) & (np.minimum(0.99, op * np.exp(np.minimum(power, 0))) >= 1 / 255)).sum())


def describe_rows(worst, ours, ref, o64, g):
    """Text for failing rows [(ratio, tensor, Gaussian)]: values, footprint, depth-hit pixels, thin axis."""
    P = len(o64.radii)
    hit_count = np.bincount(o64.hit_depth[0][o64.hit_depth[0] >= 0], minlength=P)
    ax = thin_axis(g)
    lines = []
    for ratio, k, i in worst:
        a = np.asarray(ours[k]).reshape(P, -1)[i]
        b = np.asarray(ref[k]).reshape(P, -1)[i]
        j = int(np.abs(a - b).argmax())
        lines.append(f"  Gaussian {i} d{k}[{j}]: ours {a[j]:.9e} reference {b[j]:.9e} (ratio {ratio:.2f}); row max|ref| "
                     f"{np.abs(b).max():.3e}; footprint {footprint_pixels(o64, i)} px, radius {int(o64.radii[i])}; depth-hit "
                     f"pixels {int(hit_count[i])}; thin axis {'n/a' if ax is None else int(ax[i])}")
    return "\n".join(lines)


def check_rows(label, ours, ref, rows, o64, g, again=None, rtol=RTOL, c=C, subset=None):
    """Asserts every row's ratio <= max(1, 10 x the worst ratio between `ours` and `again`, a second run of the same
    computation: its run-to-run jitter in the same units). `subset` (boolean (P,)) restricts the assertion to some of
    `rows`; the tolerance is still scaled by all of them. Returns {tensor: (worst ratio, jitter ratio)}; on failure the
    message lists the five worst rows."""
    kappa = covariance_condition(o64)
    ratios = row_ratios(ours, ref, rows, rtol, c, kappa)
    jit = {k: 0.0 for k in ratios}
    if again is not None:
        # jitter of each row in units of the same row's tolerance
        tol = row_tolerances(ref, rows, rtol, c, kappa)
        for k, (e2, _) in row_errors(again, ours, rows).items():
            with np.errstate(divide="ignore", invalid="ignore"):
                jit[k] = float(np.where(e2 == 0, 0.0, e2 / tol[k]).max(initial=0.0))
    idx = np.where(rows)[0]
    sel = np.ones(len(idx), bool) if subset is None else subset[idx]
    report, worst = {}, []
    for k, r in ratios.items():
        r = np.where(sel, r, 0.0)
        report[k] = (float(r.max()) if r.size else 0.0, jit[k])
        bound = max(1.0, 10 * jit[k])
        worst += [(float(r[t]), k, int(idx[t])) for t in np.where(~(r <= bound))[0]]
    print(f"{label}: " + ", ".join(f"d{k} worst ratio {w:.3f} jitter {j:.3f}" for k, (w, j) in report.items()))
    if worst:
        worst.sort(key=lambda t: -t[0] if np.isfinite(t[0]) else -np.inf)
        raise AssertionError(f"{label}: {len(worst)} rows beyond rtol {rtol:g}, c {c:g}; the worst:\n"
                             + describe_rows(worst[:5], ours, ref, o64, g))
    return report
