"""CPU tests of the row-wise gradient metric (gradcheck.py) and of the oracle's depth-hit path on every surfel axis.

1. The metric passes where it should: the float32 oracle against the float64 oracle, row by row. The float32 oracle has
   the arithmetic of a correct kernel without the atomics, so this is the rehearsal of test_raster_grad_rows_gpu.py.
2. The metric fails where it should: errors planted in a copy of the float32 oracle's gradients. Each is caught by the
   row metric and each passes the per-tensor `helpers.rel_err < 1e-3` every other gradient test uses; both are asserted.
3. The float64 oracle's depth path against central finite differences on each (thin axis, plane / centre-depth) cell,
   with test_transmittance_grad_cpu.fd_check (steps h and h / 4, entries whose decisions flip are skipped and counted)."""
import functools

import numpy as np
import pytest

import gradcheck as gck
import helpers
from oracle.splat_oracle import OracleRender
from rtg_slam_b200 import scene
from test_camera_grad_cpu import make_cam
from test_camera_grad_gpu import inputs_for
from test_transmittance_grad_cpu import fd_check, perturbed_gaussians

SCENES = ("small", "ragged", "masked", "dense", "axis_room")
MODES = ("sh", "colors_precomp", "cov3D_precomp")


@functools.lru_cache(maxsize=None)
def prepared(name, mode):
    """Both oracle forwards of a scene, the decision mask and the comparable rows (shared by the three losses)."""
    cam, g, mask = gck.scene_case(name)
    inputs, over = inputs_for(g, mode)
    g, kw = gck.oracle_args(inputs, mask, over)
    o32, o64 = gck.forwards(cam, g, kw)
    dm = gck.decision_mask(cam, g, kw, oracles=(o32, o64))
    assert dm.mean() <= gck.MAX_MASKED_SHARE.get(name, 0.01), (name, int(dm.sum()), dm.size)
    rows, excluded = gck.comparable_rows(cam, g, kw, o32, o64)
    return cam, g, kw, o32, o64, dm, rows, excluded


def leaf_grads(o, up):
    gr = o.backward(*up)
    return {k: v for k, v in gr.items() if k not in ("means2D", "conic", "colors", "cov3D")}


@pytest.mark.parametrize("loss", gck.LOSSES)
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", SCENES)
def test_f32_oracle_rows_match_f64_oracle(name, mode, loss):
    cam, g, kw, o32, o64, dm, rows, excluded = prepared(name, mode)
    assert rows.sum() > 200
    up = gck.upstream(cam, loss, dm)
    a, b = leaf_grads(o32, up), leaf_grads(o64, up)
    print(f"{name}/{mode}/{loss}: {int(dm.sum())} of {dm.size} pixels masked, rows left out {excluded}")
    gck.check_rows(f"{name}/{mode}/{loss}", a, b, rows, o64, g)
    if loss == "depth":
        hit = gck.hit_rows(o64, dm)
        for k, v in b.items():
            zero = ~hit if k in ("means3D", "rotations") else np.ones_like(hit)
            assert np.all(v[zero] == 0) and np.all(a[k][zero] == 0), k


def test_axis_room_keeps_the_surfels_and_reaches_every_cell():
    """axis_permute changes neither covariance nor normal; axis_room has >= 100 pixels and >= 20 Gaussians on each
    (thin axis, branch) cell, each thin axis on about a third of the surfels."""
    from test_camera_grad_gpu import cov3d_f32
    g0 = scene.surfel_room(500, seed=3)
    g1, k = gck.axis_permute(g0, seed=4)
    assert np.array_equal(gck.thin_axis(g1), k) and min(np.bincount(k, minlength=3)) > 120
    assert np.abs(cov3d_f32(g1["scales"], g1["rotations"]) - cov3d_f32(g0["scales"], g0["rotations"])).max() < 1e-7
    cam, g, kw, o32, o64, dm, rows, _ = prepared("axis_room", "sh")
    cells = gck.depth_coverage(o64, g, dm)
    print({k: (n, len(ids)) for k, (n, ids) in cells.items()})
    gck.assert_coverage(cells)
    # the scenes every other gradient test uses reach one thin axis (surfel room) or few pixels per cell (blobs)
    small = gck.depth_coverage(prepared("small", "sh")[4], prepared("small", "sh")[1])
    assert all(small[(a, b)][0] == 0 for a in (0, 1) for b in ("plane", "centre"))


# ------------------------------------------------------------------------------------------------ planted errors
def old_metric_passes(planted, ref):
    return all(helpers.rel_err(planted[k], ref[k]) < 1e-3 for k in ref)


def assert_caught_by_rows_only(label, planted, ref, rows, o64, g):
    assert old_metric_passes(planted, ref), f"{label}: the per-tensor metric sees this error too"
    with pytest.raises(AssertionError, match="rows beyond"):
        gck.check_rows(label, planted, ref, rows, o64, g)


def mixed_case(name):
    cam, g, kw, o32, o64, dm, rows, _ = prepared(name, "sh")
    up = gck.upstream(cam, "mixed", dm)
    a, b = leaf_grads(o32, up), leaf_grads(o64, up)
    gck.check_rows(f"{name} unplanted", a, b, rows, o64, g)
    assert old_metric_passes(a, b)
    return cam, g, kw, o32, o64, dm, rows, a, b


def small_row(ref, rows, k, share):
    """The visible row of tensor k whose magnitude is closest to `share` of the largest row's, if within a factor 3 of
    it (else None); it is below the median."""
    n = np.abs(ref[k].reshape(len(rows), -1)).max(axis=1)
    idx = np.where(rows & (n > 0))[0]
    i = int(idx[np.abs(np.log(n[idx] / (share * n.max()))).argmin()])
    if not share / 3 < n[i] / n.max() < 3 * share:
        return None
    assert n[i] < np.median(n[idx]), (k, n[i], np.median(n[idx]))
    return i


# An error of relative size d on a row of magnitude n is invisible to the per-tensor metric while d * n < 1e-3 * max n, and
# visible to the row metric once d * n > RTOL * n + C * max n: the rows are picked in the middle of that window.
@pytest.mark.parametrize("name", ["small", "ragged"])
@pytest.mark.parametrize("factor,share", [(1.05, 1.5e-3), (-1.0, 5e-5)], ids=["scaled_5_percent", "sign_flipped"])
def test_planted_error_in_one_small_row(name, factor, share):
    cam, g, kw, o32, o64, dm, rows, a, b = mixed_case(name)
    done = 0
    for k in a:
        i = small_row(b, rows, k, share)
        if i is None:   # this tensor has no row that small
            continue
        planted = {t: v.copy() for t, v in a.items()}
        planted[k][i] *= factor
        assert_caught_by_rows_only(f"{name} d{k} x {factor}", planted, b, rows, o64, g)
        done += 1
    assert done >= 2


def rotation_matrix(q):
    r, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)],
                     [2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)],
                     [2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]])


def dcolumn_dq(q, axis):
    """(4, 3): d(column `axis` of R(q)) / dq_k. R is quadratic in q, so the central difference with step 1 is exact."""
    q = np.asarray(q, np.float64)
    return np.stack([(rotation_matrix(q + e)[:, axis] - rotation_matrix(q - e)[:, axis]) / 2 for e in np.eye(4)])


def test_planted_wrong_axis_table_for_thin_axis_0():
    """The depth path's dL/drotation of thin-axis-0 Gaussians recomputed with the d(normal)/dq table of axis 1. dL/dnormal
    is recovered from the depth-only rotation gradient (dL/dq = D_0(q) dL/dnormal, D_0 of full column rank). Planted on
    the rows where the per-tensor metric cannot see it: the change is below half of 1e-3 of the largest rotation gradient."""
    cam, g, kw, o32, o64, dm, rows, a, b = mixed_case("axis_room")
    depth_only = leaf_grads(o32, gck.upstream(cam, "depth", dm))["rotations"]
    cells = gck.depth_coverage(o64, g, dm)
    planted = {k: v.copy() for k, v in a.items()}
    changed = 0
    for i in cells[(0, "plane")][1]:
        q = g["rotations"][i].astype(np.float64)
        D0, D1 = dcolumn_dq(q, 0), dcolumn_dq(q, 1)
        w, res, rank, _ = np.linalg.lstsq(D0, depth_only[i].astype(np.float64), rcond=None)
        assert rank == 3 and np.abs(D0 @ w - depth_only[i]).max() <= 1e-5 * np.abs(depth_only[i]).max()
        delta = D1 @ w - depth_only[i]
        if rows[i] and np.abs(delta).max() < 0.5e-3 * np.abs(b["rotations"]).max():
            planted["rotations"][i] += delta.astype(np.float32)
            changed += 1
    print(f"wrong table planted on {changed} of {len(cells[(0, 'plane')][1])} thin-axis-0 plane-branch Gaussians")
    assert changed >= 20
    assert_caught_by_rows_only("axis 1 table on axis 0 rows", planted, b, rows, o64, g)


def test_planted_dropped_hit_pixel():
    """The dL/dnormal of one plane-branch hit pixel missing from its Gaussian's rotation gradient (the backward is linear in
    the upstream gradient: the pixel's share is the backward of that pixel's dL/ddepth alone). dL/dmeans3D is left whole: one
    pixel's share of it, about dL/ddepth itself, is above 1e-3 of the largest row at this image size."""
    cam, g, kw, o32, o64, dm, rows, a, b = mixed_case("axis_room")
    gc, gd = gck.upstream(cam, "mixed", dm)
    hit = o64.hit_depth[0]
    counts = np.bincount(hit[(hit >= 0) & ~dm], minlength=len(rows))
    caught = 0
    for i in np.where(rows & (counts >= 2))[0]:
        py, px = np.argwhere((hit == i) & ~dm)[0]
        one = np.zeros_like(gd)
        one[0, py, px] = gd[0, py, px]
        share = leaf_grads(o32, (np.zeros_like(gc), one))
        assert np.abs(share["means3D"][i]).max() > 0 and all(np.all(np.delete(v, i, axis=0) == 0) for v in share.values())
        lost = np.abs(share["rotations"]).max()
        if lost == 0 or lost >= 0.5e-3 * np.abs(b["rotations"]).max():
            continue   # a centre-depth pixel, or one heavy enough to show in the per-tensor metric as well
        planted = dict(a, rotations=a["rotations"] - share["rotations"])
        assert_caught_by_rows_only(f"hit pixel ({px}, {py}) of Gaussian {i} dropped", planted, b, rows, o64, g)
        caught += 1
        if caught == 8:
            break
    assert caught == 8


def test_planted_opacity_error_on_rows_with_a_clamped_alpha():
    """dL/dopacity of Gaussians that reach the min(0.99, .) clamp of alpha at some pixel, off by 1 %."""
    cam, g0, mask = gck.scene_case("ragged")
    g0 = dict(g0, opacity=g0["opacity"].copy())
    g0["opacity"][::5] = 1.0
    inputs, over = inputs_for(g0, "sh")
    g, kw = gck.oracle_args(inputs, mask, over)
    o32, o64 = gck.forwards(cam, g, kw)
    dm = gck.decision_mask(cam, g, kw, oracles=(o32, o64))
    rows, _ = gck.comparable_rows(cam, g, kw, o32, o64)
    up = gck.upstream(cam, "mixed", dm)
    a, b = leaf_grads(o32, up), leaf_grads(o64, up)
    gck.check_rows("clamped unplanted", a, b, rows, o64, g)
    geom = o64.geom()
    yy, xx = np.mgrid[0:cam.height, 0:cam.width]
    n = np.abs(b["opacities"]).reshape(-1)
    clamped = []
    for i in np.where(rows & (g["opacity"].reshape(-1) > 0.99))[0]:
        (x, y), (ca, cb, cc, op) = geom["xy"][i], geom["conic_opacity"][i]
        dx, dy = x - xx, y - yy
        power = -0.5 * (ca * dx * dx + cc * dy * dy) - cb * dx * dy
        if (op * np.exp(np.minimum(power, 0)) > 0.99).any() and 1e3 * gck.C * n.max() < n[i] < 0.05 * n.max():
            clamped.append(i)
    assert len(clamped) >= 3, clamped
    planted = {k: v.copy() for k, v in a.items()}
    planted["opacities"][clamped] *= 1.01
    assert_caught_by_rows_only("1 % on clamped-alpha opacity rows", planted, b, rows, o64, g)


# ------------------------------------------------------------------------- the oracle's depth path, finite differences
@pytest.mark.parametrize("loss", ["depth", "mixed"])
def test_oracle_depth_path_matches_finite_differences_on_every_axis(loss):
    """xyz, rotations and scales of eight hit Gaussians per (thin axis, branch) cell. The tolerance of each entry is scaled
    by its own row (not by the tensor's largest entry) wherever the row is above 1 % of the largest one. The reference
    does not differentiate the depth with respect to the scales: the analytic depth-only gradient is exactly zero and so
    is the finite difference, away from argmin / threshold flips."""
    P = 240
    g = gck.axis_compact(P, seed=17)
    cam = make_cam(c2w=scene.small_pose())
    gc, gd = (x.astype(np.float64) for x in scene.upstream_grads(cam, seed=3))
    if loss == "depth":
        gc = np.zeros_like(gc)
    up = (gc, gd, np.zeros_like(gd))
    o = OracleRender(cam, g, precision="f64")
    cells = gck.depth_coverage(o, g)
    gr = o.backward(gc, gd, nthreads=1)
    o.close()
    picked = []
    for cell, (n, ids) in sorted(cells.items()):
        assert len(ids) >= 8, (cell, n, len(ids))
        picked += [int(i) for i in ids[:8]]
    picked = sorted(set(picked))
    if loss == "depth":
        assert np.all(gr["scales"] == 0) and np.all(gr["opacities"] == 0) and np.all(gr["shs"] == 0)
    values = []
    for k, src in (("means3D", "xyz"), ("rotations", "rotations"), ("scales", "scales")):
        a = gr[k].reshape(P, -1)
        block = float(np.abs(gr[k if a.any() else "means3D"]).max())
        for i in picked:
            scale = max(float(np.abs(a[i]).max()), 1e-2 * block)
            values += [((k, i * a.shape[1] + j), float(a[i, j]), scale, float(g[src][i, j])) for j in range(a.shape[1])]

    def loss_of(gm):
        r = OracleRender(cam, gm, precision="f64")
        v = float((r.color * up[0]).sum() + (r.depth * up[1]).sum())
        r.close()
        return v

    def estimate(entry, h):
        k, idx = entry
        return (loss_of(perturbed_gaussians(g, {}, k, idx, h)[0]) - loss_of(perturbed_gaussians(g, {}, k, idx, -h)[0])) / (2 * h)
    checked, skipped = fd_check(values, estimate, f"axis_compact/{loss}", max_skip=len(values) // 25)
    print(f"axis_compact/{loss}: {len(picked)} Gaussians, {checked} entries checked, {len(skipped)} skipped; cells "
          f"{ {c: (n, len(i)) for c, (n, i) in cells.items()} }")
    assert checked >= 0.9 * len(values)
