"""CPU tests of the rasterizer oracle (oracle/splat_oracle.c): internal consistency (f32 vs f64, analytic vs
finite-difference gradients), the reference's documented quirks, and -- the pin -- agreement with the golden
outputs of the reference's own CUDA code (tests/golden/raster_*.npz, see make_raster_golden.py)."""
import glob
import os

import numpy as np
import pytest

from oracle.splat_oracle import OracleRender
from rtg_slam_b200 import scene

import helpers
from golden.make_raster_golden import CASES, build_case
from golden.make_raster_inputs_golden import CASES as INPUT_CASES, build_case as build_input_case

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = ("color", "depth", "hit_color", "hit_depth", "hit_color_weight", "hit_depth_weight", "T_map", "radii")


def outputs(o):
    return dict(zip(NAMES, o.outputs()))


@pytest.fixture(scope="module")
def room():
    cam = scene.make_camera("small")
    return cam, scene.surfel_room(3000, seed=1)


def test_f32_matches_f64(room):
    cam, g = room
    a = OracleRender(cam, g, precision="f32", tie_eps=1e-4)
    b = OracleRender(cam, g, precision="f64")
    st = helpers.compare_outputs(outputs(a), outputs(b), tie=a.tie, tol=1e-4)
    assert st["radii_mismatch"] == 0
    gc, gd = scene.upstream_grads(cam)
    ga, gb = a.backward(gc, gd), b.backward(gc, gd)
    for k in ("means3D", "shs", "opacities", "scales", "rotations"):
        assert helpers.rel_err(ga[k], gb[k]) < 1e-4, k


def test_analytic_gradient_matches_finite_differences(room):
    cam, g = room
    g64 = {k: v.astype(np.float64) for k, v in g.items()}
    gc, gd = scene.upstream_grads(cam)
    base = OracleRender(cam, g64, precision="f64")
    an = base.backward(gc, gd)
    vis = np.where(base.radii > 0)[0]
    rng = np.random.default_rng(0)

    def loss(gm):
        o = OracleRender(cam, gm, precision="f64")
        val = float((o.color * gc).sum() + (o.depth * gd).sum())
        o.close()
        return val

    for name, key in (("xyz", "means3D"), ("scales", "scales"), ("rotations", "rotations"), ("opacity", "opacities"), ("shs", "shs")):
        for _ in range(4):
            i = int(rng.choice(vis))
            idx = (i,) + tuple(int(rng.integers(0, s)) for s in g64[name].shape[1:])
            h = 1e-6 * max(1e-2, abs(g64[name][idx]))
            gp = dict(g64); gp[name] = g64[name].copy(); gp[name][idx] += h
            gm = dict(g64); gm[name] = g64[name].copy(); gm[name][idx] -= h
            fd = (loss(gp) - loss(gm)) / (2 * h)
            assert abs(fd - an[key][idx]) <= 1e-4 * max(abs(fd), abs(an[key][idx])) + 1e-9, (name, idx, fd, an[key][idx])


def test_quirks_initial_values_and_mask(room):
    """SURVEY appendix: masked-out / empty tiles keep colour 0, depth 0, hit maps 0 (not -1), T 1; gradients of
    Gaussians that only touch masked-out tiles are exactly zero."""
    cam, g = room
    th, tw = cam.tile_grid
    mask = np.zeros((th, tw), np.int32)
    mask[:, : tw // 2] = 1
    o = OracleRender(cam, g, tile_mask=mask)
    out = outputs(o)
    px = (tw // 2) * 16
    assert np.all(out["color"][:, :, px:] == 0) and np.all(out["depth"][:, :, px:] == 0)
    assert np.all(out["hit_color"][:, :, px:] == 0) and np.all(out["hit_depth"][:, :, px:] == 0)
    assert np.all(out["T_map"][:, :, px:] == 1)
    assert out["hit_depth"][:, :, :px].min() == -1  # -1 only inside rendered tiles
    gc, gd = scene.upstream_grads(cam)
    gr = o.backward(gc, gd)
    geom = o.geom()
    right_only = (geom["xy"][:, 0] - o.radii > px + 16) & (o.radii > 0)
    assert right_only.any()
    assert np.all(gr["opacities"][right_only] == 0) and np.all(gr["shs"][right_only] == 0)


def test_invariants(room):
    cam, g = room
    o = OracleRender(cam, g)
    out = outputs(o)
    assert (out["T_map"] > 0).all() and (out["T_map"] <= 1).all()
    hit = out["hit_depth"][0] >= 0
    assert (out["hit_depth_weight"][0][hit] > 0).all()
    assert (out["depth"][0][~hit] == 0).all()
    # first opaque Gaussian has alpha >= threshold => weight / T_before >= thr; weight <= 0.99
    assert (out["hit_depth_weight"] <= 0.99 + 1e-6).all()
    pl, rg = o.binning()
    geom = o.geom()
    for t in np.where(rg[:, 0] != rg[:, 1])[0][:50]:
        d = geom["depth"][pl[rg[t, 0]:rg[t, 1]]]
        assert (np.diff(d) >= 0).all(), "tile list must be sorted front to back"


def test_empty_and_fully_culled():
    cam = scene.make_camera("tiny")
    g = scene.random_blobs(50, seed=3)
    g["xyz"][:, 2] = -1.0  # behind the camera
    o = OracleRender(cam, g)
    assert o.num_rendered == 0 and (o.radii == 0).all() and (o.T_map == 1).all()


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_cuda_golden(name):
    path = os.path.join(GOLD, name + ".npz")
    if not os.path.exists(path):
        pytest.skip("golden fixture not generated yet (needs a GPU run of make_raster_golden.py)")
    gold = np.load(path)
    cam, g, mask, grads = build_case(name)
    o = OracleRender(cam, g, tile_mask=mask, precision="f32", tie_eps=1e-4)
    ref = {k: gold[k] for k in NAMES}
    st = helpers.compare_outputs(outputs(o), ref, tie=o.tie, tol=1e-4, label=name)
    assert st["radii_mismatch"] == 0
    assert o.num_rendered == int(gold["num_rendered"])
    gr = o.backward(*grads)
    for k in ("means3D", "shs", "opacities", "scales", "rotations"):
        jitter = float(gold["jitter_" + k])
        tol = max(1e-3, 10 * jitter)
        assert helpers.rel_err(gr[k], gold["grad_" + k]) < tol, (k, helpers.rel_err(gr[k], gold["grad_" + k]), jitter)


COLOR_SIDE = ("color", "hit_color", "hit_color_weight", "T_map", "radii")


def test_precomputed_colors_reproduce_the_sh_run(room):
    """colors_precomp equal to the SH run's colours renders identically; dL/dcolors_precomp is that run's dL/dcolors."""
    cam, g = room
    g64 = {k: v.astype(np.float64) for k, v in g.items()}
    gc, gd = scene.upstream_grads(cam)
    base = OracleRender(cam, g64, precision="f64")
    o = OracleRender(cam, g64, precision="f64", colors_precomp=base.geom()["rgb"])
    for k, v in outputs(base).items():
        assert np.array_equal(outputs(o)[k], v), k
    gb, go = base.backward(gc, gd), o.backward(gc, gd)
    assert "shs" not in go and np.abs(gb["colors"]).max() > 0
    # the backward sums per-thread partial gradients in a varying order: equal to f64 rounding
    assert helpers.rel_err(go["colors_precomp"], gb["colors"]) < 1e-12
    for k in ("opacities", "scales", "rotations", "means2D", "conic"):
        assert helpers.rel_err(go[k], gb[k]) < 1e-12, k


def test_precomputed_covariance_reproduces_the_scale_rotation_run(room):
    """cov3D_precomp equal to the run's own covariance: identical colour side and dL/dcov3D. Without scales there is no
    surfel, so the depth of a hit is the centre depth."""
    cam, g = room
    g64 = {k: v.astype(np.float64) for k, v in g.items()}
    gc, gd = scene.upstream_grads(cam)
    base = OracleRender(cam, g64, precision="f64")
    o = OracleRender(cam, g64, precision="f64", cov3D_precomp=base.geom()["cov3D"])
    for k in COLOR_SIDE + ("hit_depth", "hit_depth_weight"):
        assert np.array_equal(outputs(o)[k], outputs(base)[k]), k
    hit = o.hit_depth[0] >= 0
    assert hit.any()
    assert np.array_equal(o.depth[0][hit], o.geom()["depth"][o.hit_depth[0][hit]])
    gb, go = base.backward(gc, gd), o.backward(gc, gd)
    assert "scales" not in go and "rotations" not in go and np.abs(gb["cov3D"]).max() > 0
    assert helpers.rel_err(go["cov3D_precomp"], gb["cov3D"]) < 1e-12
    for k in ("opacities", "shs", "means2D", "conic"):
        assert helpers.rel_err(go[k], gb[k]) < 1e-12, k


def test_precomputed_input_gradients_match_finite_differences(room):
    cam, g = room
    g64 = {k: v.astype(np.float64) for k, v in g.items()}
    gc, gd = scene.upstream_grads(cam)
    ref = OracleRender(cam, g64, precision="f64")
    geom = ref.geom()
    rng = np.random.default_rng(1)
    vis = np.where(ref.radii > 0)[0]
    # colours outside [0, 1] as well: precomputed colours are not clamped
    cols = geom["rgb"] + rng.uniform(-0.3, 0.3, geom["rgb"].shape)
    for key, val in (("colors_precomp", cols), ("cov3D_precomp", geom["cov3D"])):
        base = OracleRender(cam, g64, precision="f64", **{key: val})
        an = base.backward(gc, gd)
        for name, x in (("xyz", None), (key, val)):
            for _ in range(4):
                i = int(rng.choice(vis))
                arr = g64[name] if x is None else x
                idx = (i,) + tuple(int(rng.integers(0, s)) for s in arr.shape[1:])
                h = 1e-6 * max(1e-2, abs(arr[idx]))
                vals = []
                for sgn in (1, -1):
                    a = arr.copy()
                    a[idx] += sgn * h
                    gm, kw = (dict(g64, xyz=a), {key: val}) if x is None else (g64, {key: a})
                    o = OracleRender(cam, gm, precision="f64", **kw)
                    vals.append(float((o.color * gc).sum() + (o.depth * gd).sum()))
                    o.close()
                fd = (vals[0] - vals[1]) / (2 * h)
                a_ = an["means3D" if x is None else key][idx]
                assert abs(fd - a_) <= 1e-4 * max(abs(fd), abs(a_)) + 1e-9, (key, name, idx, fd, a_)


@pytest.mark.parametrize("name", sorted(INPUT_CASES))
def test_oracle_matches_reference_cuda_golden_alternative_inputs(name):
    """Precomputed colours and a 4-coefficient SH table against the reference's own CUDA rasterizer."""
    path = os.path.join(GOLD, name + ".npz")
    if not os.path.exists(path):
        pytest.skip("golden fixture not generated yet (needs a GPU run of make_raster_inputs_golden.py)")
    gold = np.load(path)
    cam, inputs, mask, grads, over = build_input_case(name)
    g = {k: inputs.get(k) for k in ("xyz", "opacity", "shs", "scales", "rotations")}
    o = OracleRender(cam, g, tile_mask=mask, precision="f32", tie_eps=1e-4, colors_precomp=inputs.get("colors_precomp"), **over)
    st = helpers.compare_outputs(outputs(o), {k: gold[k] for k in NAMES}, tie=o.tie, tol=1e-4, label=name)
    assert st["radii_mismatch"] == 0
    assert o.num_rendered == int(gold["num_rendered"])
    gr = o.backward(*grads)
    keys = [k[len("grad_"):] for k in gold.files if k.startswith("grad_")]
    assert ("colors_precomp" in keys) == ("colors_precomp" in inputs) and len(keys) == 5
    for k in keys:
        tol = max(1e-3, 10 * float(gold["jitter_" + k]))
        assert helpers.rel_err(gr[k], gold["grad_" + k]) < tol, (k, helpers.rel_err(gr[k], gold["grad_" + k]))
