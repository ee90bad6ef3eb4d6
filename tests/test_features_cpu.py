"""CPU tests of per-Gaussian feature maps (rtg_splat_features / rtg_splat_features_backward, features.rasterize_features):
the float64 statement in oracle/features_oracle.py against identities with what the oracle already computes (F = 1 gives
1 - T_map, F = the colours gives the colour image without background, A^T 1 is the contribution weight, and the adjoint
identity <A F, G> = <F, A^T G>), the C entry points' host validation and the Python argument checks, none of which
touches CUDA."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle.contrib_oracle import contributions
from oracle.features_oracle import features
from rtg_slam_b200 import _lib
from test_contributions_cpu import CASES, case


@pytest.mark.parametrize("name", CASES)
def test_ones_give_the_covered_fraction(name):
    o = case(name)
    m = features(o, F=np.ones((o.P, 1)))["map"][0]
    want = 1.0 - o.T_map[0]
    assert want.sum() > 100
    assert np.abs(m - want).max() <= 1e-12


@pytest.mark.parametrize("name", CASES)
def test_colours_give_the_colour_image_without_background(name):
    """F = the colour the forward blends (colors_precomp, or the clamped SH colour of geom()) renders its colour image;
    the oracle's background is 0."""
    o = case(name)
    assert tuple(o.settings["bg"]) == (0.0, 0.0, 0.0)
    F = o.colors_precomp if o.colors_precomp is not None else o.geom()["rgb"]
    m = features(o, F=F)["map"]
    assert np.abs(o.color).max() > 0.1
    assert np.abs(m - o.color).max() <= 1e-12 * np.abs(o.color).max()


@pytest.mark.parametrize("name", CASES)
def test_transpose_of_ones_is_the_contribution_weight(name):
    o = case(name)
    g = features(o, G=np.ones((1, o.H, o.W)))["grad"][:, 0]
    w = contributions(o)["weight"]
    assert w.max() > 0
    assert np.abs(g - w).max() <= 1e-12 * w.max()
    assert np.all(g[o.radii == 0] == 0)


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("C_", [1, 5, 17])
def test_adjoint_identity(name, C_):
    o = case(name)
    rng = np.random.default_rng(100 + C_)
    F, G = rng.standard_normal((o.P, C_)), rng.standard_normal((C_, o.H, o.W))
    r = features(o, F=F, G=G)
    lhs, rhs = float((r["map"] * G).sum()), float((F * r["grad"]).sum())
    scale = float((np.abs(r["map"]) * np.abs(G)).sum())
    assert scale > 1
    assert abs(lhs - rhs) <= 1e-12 * scale, (lhs, rhs)


# ----------------------------------------------------------------------------------------------------------- C ABI
def test_both_symbols_are_exported_and_declared():
    L = _lib.lib()
    syms = _lib.header_symbols()
    for s in ("rtg_splat_features", "rtg_splat_features_backward"):
        assert s in syms and s in _lib.SIGNATURES and hasattr(L, s)
    assert _lib.RTG_FEATURES_MAX == 128


def _view(flags=0):
    v = _lib.RtgSplatView()
    v.image_height, v.image_width, v.sh_degree, v.prefiltered = 48, 64, 3, flags
    v.viewmatrix = v.projmatrix = v.campos = v.bg = 256  # never dereferenced: validation fails first
    return v


@pytest.mark.parametrize("sym", ["rtg_splat_features", "rtg_splat_features_backward"])
def test_host_validation_rejects_bad_arguments_before_cuda(sym):
    L = _lib.lib()
    fn = getattr(L, sym)
    v = _view()
    ws, cnt, inp, out = C.c_void_p(4096), C.c_void_p(8192), C.c_void_p(16384), C.c_void_p(32768)

    def call(view=C.byref(v), P=10, geom=ws, img=ws, bin_=ws, r_cap=1024, counters=cnt, C_=16, src=inp, dst=out):
        return fn(view, P, geom, img, bin_, r_cap, counters, C_, src, dst, None)

    bad = {
        "view is NULL": dict(view=None),
        "P < 0": dict(P=-1),
        "R_cap < 0": dict(r_cap=-1),
        "C = 0": dict(C_=0),
        "C < 0": dict(C_=-3),
        "C = 129": dict(C_=129),
        "NULL workspace (geom)": dict(geom=None),
        "NULL workspace (img)": dict(img=None),
        "NULL workspace (bin)": dict(bin_=None),
        "NULL counters": dict(counters=None),
        "NULL input": dict(src=None),
        "NULL output": dict(dst=None),
        "misaligned input": dict(src=C.c_void_p(16386)),
        "misaligned output": dict(dst=C.c_void_p(32770)),
    }
    for what, kw in bad.items():
        assert call(**kw) == -1, what
        msg = L.rtg_last_error()
        assert msg.startswith(sym.encode() + b":"), (what, msg)
    assert b"C must be 1..128" in (call(C_=129), L.rtg_last_error())[1]
    for flags in (4, 1 << 30, -1):
        fv = _view(flags)
        assert call(view=C.byref(fv)) == -1
        assert b"unknown bits" in L.rtg_last_error()
    bad_size = _view()
    bad_size.image_width = 0
    assert call(view=C.byref(bad_size)) == -1 and b"bad image size" in L.rtg_last_error()
    if sym == "rtg_splat_features":
        assert call(P=0, src=None, dst=None) == -1   # the map of P == 0 is still written (zeros)
    else:
        assert call(P=0, geom=None, img=None, bin_=None, counters=None, src=None, dst=None) == 0   # no row, no work


# ---------------------------------------------------------------------------------------------- Python argument checks
def test_python_argument_errors_are_raised_before_cuda():
    from rtg_slam_b200.features import rasterize_features
    P = 6
    means = torch.zeros(P, 3)
    opac = torch.zeros(P, 1)

    def call(f, m=means):
        return rasterize_features(None, m, opac, f, colors_precomp=torch.zeros(P, 3), scales=torch.zeros(P, 3),
                                  rotations=torch.zeros(P, 4))

    with pytest.raises(TypeError):
        call(np.zeros((P, 4), np.float32))           # not a tensor
    with pytest.raises(TypeError):
        call(torch.zeros(P, 4, dtype=torch.float64))  # dtype
    with pytest.raises(TypeError):
        call(torch.zeros(P, 4, dtype=torch.float16))
    with pytest.raises(ValueError):
        call(torch.zeros(P + 1, 4))                   # rows != P
    with pytest.raises(ValueError):
        call(torch.zeros(P * 4))                      # not (P, C)
    with pytest.raises(ValueError):
        call(torch.zeros(P, 0))                       # C = 0
    with pytest.raises(ValueError):
        call(torch.zeros(P, 129))                     # C > 128
    with pytest.raises(TypeError):
        call(torch.zeros(P, 4))                       # a CPU tensor
