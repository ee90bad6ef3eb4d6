"""CPU tests of the per-Gaussian contribution statistics (rtg_splat_contributions, mapstats.gaussian_contributions): the
statement in oracle/contrib_oracle.py against a literal per-pixel walk of the forward's blend loop, its two identities
(sum of weights = sum of (1 - T_map); error = the colour intermediate of the backward under dL/dC = (e, 0, 0)), and the
C entry point's host validation.

The statement walks only the first n_contrib(p) entries of each pixel's list and blends every pair there that passes the
1/255 cut-off, without restating the T_threshold and opaque-hit termination. The literal walk below restates them, so
their agreement pins that shortcut: inside the prefix every blended pair adds colour, and nothing after it does."""
import ctypes as C

import numpy as np
import pytest

from oracle.antialias_oracle import AntialiasedOracleRender
from oracle.contrib_oracle import contributions
from oracle.splat_oracle import OracleRender
from rtg_slam_b200 import _lib, scene
from test_camera_grad_cpu import compact_scene, cov3d

CASES = ("plain", "colors_precomp", "cov3D_precomp", "masked", "antialiased")


def case(name, precision="f64"):
    """An OracleRender of about 200 overlapping surfels in a 32x32 view (2x2 tiles)."""
    cam = scene.Camera(32, 32, 30.0, 30.0, 15.5, 15.5, c2w=scene.small_pose())
    g = compact_scene(200, seed=61)
    kw = {}
    if name == "colors_precomp":
        kw["colors_precomp"] = np.random.default_rng(62).uniform(-0.25, 1.25, (200, 3))
    elif name == "cov3D_precomp":
        kw["cov3D_precomp"] = cov3d(g)
    elif name == "masked":
        kw["tile_mask"] = np.array([[1, 0], [0, 1]], np.int32)
    cls = AntialiasedOracleRender if name == "antialiased" else OracleRender
    return cls(cam, g, precision=precision, **kw)


def literal_walk(o, pixel_error):
    """Per pixel, forward.cu's blend loop over the whole tile list: power > 0 and alpha < 1/255 skip the entry, the first
    alpha >= opaque_threshold is the opaque hit, a pair whose T after it falls below T_threshold adds no colour and ends
    the pixel once it has its hit. Returns (n_pixels, weight, error) of the pairs that add colour."""
    H, W, P = o.H, o.W, o.P
    geo = o.geom()
    xy, co = geo["xy"], geo["conic_opacity"]
    pl, rg = o.binning()
    T_thr, op_thr = o.V.T_threshold, o.V.opaque_threshold
    n, w, e = np.zeros(P, np.int64), np.zeros(P), np.zeros(P)
    tw = (W + 15) // 16
    for py in range(H):
        for px in range(W):
            t = (py // 16) * tw + px // 16
            T, hit = 1.0, False
            for g in pl[rg[t, 0]:rg[t, 1]]:
                dx, dy = xy[g, 0] - px, xy[g, 1] - py
                power = -0.5 * (co[g, 0] * dx * dx + co[g, 2] * dy * dy) - co[g, 1] * dx * dy
                if power > 0:
                    continue
                alpha = min(0.99, co[g, 3] * np.exp(power))
                if alpha < 1.0 / 255.0:
                    continue
                if not hit and alpha >= op_thr:
                    hit = True
                test_T = T * (1 - alpha)
                if test_T < T_thr and hit:
                    break
                if test_T >= T_thr:
                    n[g] += 1
                    w[g] += alpha * T
                    e[g] += alpha * T * pixel_error[py, px]
                T = test_T
    return n, w, e


def pixel_errors(o, seed=3):
    return np.random.default_rng(seed).uniform(0.0, 1.0, (o.H, o.W))


@pytest.mark.parametrize("name", CASES)
def test_statement_matches_the_literal_blend_loop(name):
    o = case(name)
    e = pixel_errors(o)
    st = contributions(o, e)
    n, w, err = literal_walk(o, e)
    assert n.sum() > 5000 and (n > 0).sum() > 100, (n.sum(), (n > 0).sum())
    # the walk ends on T_threshold in some pixels and on the opaque hit in others: the prefix shortcut is exercised
    _, nc = o.image_state()
    lens = np.diff(o.binning()[1], axis=1)[:, 0]
    assert (nc < lens[(np.arange(o.H)[:, None] // 16) * 2 + np.arange(o.W)[None, :] // 16]).any()
    assert np.array_equal(st["n_pixels"], n)
    assert np.abs(st["weight"] - w).max() <= 1e-12 * np.abs(w).max()
    assert np.abs(st["error"] - err).max() <= 1e-12 * np.abs(err).max()
    vis = o.radii > 0
    assert np.all(st["n_pixels"][~vis] == 0) and np.all(st["weight"][~vis] == 0)
    assert np.all(st["in_prefix"] >= st["n_pixels"])
    if name == "masked":
        assert np.all(o.T_map[0][:16, 16:] == 1) and np.all(o.T_map[0][16:, :16] == 1)


@pytest.mark.parametrize("name", CASES)
def test_weights_sum_to_the_covered_fraction(name):
    o = case(name)
    st = contributions(o)
    lhs, rhs = st["weight"].sum(), (1.0 - o.T_map[0].astype(np.float64)).sum()
    assert rhs > 100
    assert abs(lhs - rhs) <= 1e-12 * rhs, (lhs, rhs)


@pytest.mark.parametrize("name", ["plain", "colors_precomp", "masked"])
def test_error_is_the_backward_colour_intermediate(name):
    o = case(name)
    e = pixel_errors(o)
    st = contributions(o, e)
    dC = np.zeros((3, o.H, o.W))
    dC[0] = e
    ref = o.backward(dC, np.zeros((1, o.H, o.W)))["colors"][:, 0]
    assert np.abs(ref).max() > 0
    assert np.all(np.abs(st["error"] - ref) <= 1e-10 * np.abs(ref) + 1e-14 * np.abs(ref).max())


def test_f32_statement_counts_match_f64_outside_ties():
    """The statement in the oracle's float32 agrees with the float64 one where no pixel decision is near a threshold."""
    o32, o64 = case("plain", "f32"), case("plain", "f64")
    a, b = contributions(o32), contributions(o64)
    assert np.abs(a["n_pixels"] - b["n_pixels"]).sum() <= 2
    assert np.abs(a["weight"] - b["weight"]).max() <= 1e-4 * np.abs(b["weight"]).max()


# ----------------------------------------------------------------------------------------------------------- C ABI
def _view(flags=0):
    v = _lib.RtgSplatView()
    v.image_height, v.image_width, v.sh_degree, v.prefiltered = 48, 64, 3, flags
    v.viewmatrix = v.projmatrix = v.campos = v.bg = 256  # never dereferenced: validation fails first
    return v


def test_host_validation_rejects_bad_arguments_before_cuda():
    L = _lib.lib()
    v = _view()
    ws, cnt, out = C.c_void_p(4096), C.c_void_p(8192), C.c_void_p(16384)

    def call(view=C.byref(v), P=10, geom=ws, img=ws, bin_=ws, r_cap=1024, counters=cnt, pixel_error=None, n_pixels=out,
             weight=out, error=None):
        return L.rtg_splat_contributions(view, P, geom, img, bin_, r_cap, counters, pixel_error, n_pixels, weight, error, None)

    bad = {
        "view is NULL": dict(view=None),
        "P < 0": dict(P=-1),
        "R_cap < 0": dict(r_cap=-1),
        "NULL workspace": dict(geom=None),
        "NULL workspace (img)": dict(img=None),
        "NULL workspace (bin)": dict(bin_=None),
        "NULL workspace (counters)": dict(counters=None),
        "NULL n_pixels": dict(n_pixels=None),
        "NULL weight": dict(weight=None),
        "error without pixel_error": dict(error=out),
        "pixel_error without error": dict(pixel_error=out),
        "4-byte aligned": dict(weight=C.c_void_p(16386)),
    }
    for what, kw in bad.items():
        assert call(**kw) == -1, what
        msg = _lib.lib().rtg_last_error()
        assert msg.startswith(b"rtg_splat_contributions"), (what, msg)
    for flags in (4, 1 << 30, -1):
        fv = _view(flags)
        assert call(view=C.byref(fv)) == -1
        assert b"unknown bits" in L.rtg_last_error()
    # P == 0 needs no output and does no work
    assert call(P=0, n_pixels=None, weight=None) == 0
