"""CPU tests of the feature map's weight gradient (rtg_splat_features_backward_geometry, rasterize_features(weight_grad=
True)): the float64 statement of oracle/feature_weights_oracle.py against central finite differences of the feature map
itself (features_oracle.features) and, for F = 1, against the oracle's transmittance gradient, an independent path; then
the C entry point's host validation and the Python argument checks, none of which touches CUDA."""
import ctypes as C

import numpy as np
import pytest
import torch

import gradcheck as gck
from oracle.feature_weights_oracle import weight_gradient
from oracle.features_oracle import features
from oracle.splat_oracle import OracleRender
from rtg_slam_b200 import _lib, scene
from test_camera_grad_cpu import compact_scene, cov3d, make_cam
from test_transmittance_grad_cpu import fd_check, oracle_grads, perturbed_gaussians

SYM = "rtg_splat_features_backward_geometry"


def case(name, Cn):
    """(camera, gaussians, render kwargs, F (P, Cn), G (Cn, H, W)) on the transmittance tests' compact scene: F normal,
    G uniform >= 0 scaled 1/N and zero where a decision lies within 1e-3 of its threshold (gradcheck.decision_mask)."""
    g = compact_scene(160, seed=11)
    cam = make_cam(c2w=scene.small_pose())
    kw = {}
    if name == "cov":
        kw["cov3D_precomp"] = cov3d(g)
    elif name == "masked":
        kw["tile_mask"] = np.array([[1, 0, 1, 1], [0, 1, 0, 1], [1, 1, 0, 0]], np.int32)
    else:
        assert name == "plain"
    rng = np.random.default_rng(Cn)
    F = rng.standard_normal((160, Cn))
    G = rng.uniform(0.0, 1.0, (Cn, cam.height, cam.width)) / (cam.height * cam.width)
    G[:, gck.decision_mask(cam, g, kw)] = 0.0
    return cam, g, kw, F, G


def statement(cam, g, kw, F, G, camera=False):
    kw = dict(kw)
    return weight_gradient(cam, g, F, G, tile_mask=kw.pop("tile_mask", None), cov3D_precomp=kw.pop("cov3D_precomp", None),
                           camera=camera, **kw)


def map_loss(cam, g, kw, F, G):
    o = OracleRender(cam, g, precision="f64", **kw)
    v = float((features(o, F=F)["map"] * G).sum())
    o.close()
    return v


@pytest.mark.parametrize("name,Cn", [("plain", 1), ("plain", 5), ("cov", 4), ("masked", 3)])
def test_statement_matches_finite_differences(name, Cn):
    cam, g, kw, F, G = case(name, Cn)
    gr, _ = statement(cam, g, kw, F, G)
    o = OracleRender(cam, g, precision="f64", **kw)
    vis = np.where(o.radii > 0)[0]
    o.close()
    assert len(vis) > 100
    keys = ["means3D", "opacities"] + (["cov3D_precomp"] if "cov3D_precomp" in kw else ["scales"])
    rows = np.random.default_rng(22).choice(vis, 12, replace=False)
    values = []
    for k in keys:
        a = gr[k].reshape(len(g["xyz"]), -1)
        scale = float(np.abs(a).max())
        assert scale > 0, k
        par = (kw[k] if k in kw else g[{"means3D": "xyz", "opacities": "opacity"}.get(k, k)]).reshape(len(g["xyz"]), -1)
        values += [((k, int(i) * a.shape[1] + j), float(a[i, j]), scale, float(par[i, j])) for i in rows for j in range(a.shape[1])]

    def estimate(entry, h):
        k, idx = entry
        return (map_loss(cam, *perturbed_gaussians(g, kw, k, idx, h), F, G)
                - map_loss(cam, *perturbed_gaussians(g, kw, k, idx, -h), F, G)) / (2 * h)
    checked, skipped = fd_check(values, estimate, name, max_skip=len(values) // 50)
    print(f"{name} C={Cn}: {checked} entries checked, {len(skipped)} skipped")


@pytest.mark.parametrize("name", ["plain", "cov", "masked"])
def test_ones_give_the_transmittance_gradient(name):
    """F = 1 renders 1 - T_map, so <G, map> has the gradient of <-G, T_map>: the oracle's T term, a different path
    (the background term of its backward), per Gaussian and for the camera."""
    cam, g, kw, _, G = case(name, 1)
    ours, ours_cam = statement(cam, g, kw, np.ones((160, 1)), G, camera=True)
    zc, zd = np.zeros((3, cam.height, cam.width)), np.zeros((1, cam.height, cam.width))
    ref, ref_cam = oracle_grads(cam, g, kw, (zc, zd, -G))
    for k, v in ours.items():
        assert np.abs(v).max() > 0, k
        assert np.abs(v - ref[k]).max() <= 1e-10 * np.abs(ref[k]).max(), k
    for k, v in ours_cam.items():
        if k == "campos":  # the map reads no colour: campos has no gradient
            assert np.all(v == 0) and np.all(ref_cam[k] == 0)
            continue
        assert np.abs(v - ref_cam[k]).max() <= 1e-10 * np.abs(ref_cam[k]).max(), k


def test_statement_is_linear_in_the_channels():
    """Channels may be split anywhere (the kernel adds per chunk): the gradient of C = 5 is the sum of C = 2 and C = 3."""
    cam, g, kw, F, G = case("plain", 5)
    whole, cw = statement(cam, g, kw, F, G, camera=True)
    a, ca = statement(cam, g, kw, F[:, :2], G[:2], camera=True)
    b, cb = statement(cam, g, kw, F[:, 2:], G[2:], camera=True)
    for k in whole:
        assert np.abs(whole[k] - a[k] - b[k]).max() <= 1e-12 * np.abs(whole[k]).max(), k
    for k in ("viewmatrix", "projmatrix"):
        assert np.abs(cw[k] - ca[k] - cb[k]).max() <= 1e-12 * np.abs(cw[k]).max(), k


# ----------------------------------------------------------------------------------------------------------- C ABI
def test_symbol_is_exported_and_declared():
    assert SYM in _lib.header_symbols() and SYM in _lib.SIGNATURES and hasattr(_lib.lib(), SYM)


def _view(flags=0):
    v = _lib.RtgSplatView()
    v.image_height, v.image_width, v.sh_degree, v.prefiltered = 48, 64, 3, flags
    v.viewmatrix = v.projmatrix = v.campos = v.bg = 256  # never dereferenced: validation fails first
    return v


def test_host_validation_rejects_bad_arguments_before_cuda():
    L = _lib.lib()
    fn = getattr(L, SYM)
    v = _view()
    p = lambda a: C.c_void_p(a)
    base = dict(view=C.byref(v), P=10, means=p(1 << 12), scales=p(2 << 12), rots=p(3 << 12), cov=None, radii=p(4 << 12),
                geom=p(5 << 12), img=p(5 << 12), bin_=p(5 << 12), r_cap=1024, counters=p(6 << 12), C_=16, feat=p(7 << 12),
                dout=p(8 << 12), scratch=p(9 << 12), dmeans=p(10 << 12), dopac=p(11 << 12), dscales=p(12 << 12),
                drot=p(13 << 12), dcov=None, visible=0, dcam=None, cam_scratch=None)

    def call(**over):
        a = dict(base, **over)
        return fn(*a.values(), None)

    bad = {
        "view is NULL": dict(view=None),
        "P < 0": dict(P=-1),
        "R_cap < 0": dict(r_cap=-1),
        "C = 0": dict(C_=0),
        "C = 129": dict(C_=129),
        "NULL workspace (geom)": dict(geom=None),
        "NULL workspace (img)": dict(img=None),
        "NULL workspace (bin)": dict(bin_=None),
        "NULL counters": dict(counters=None),
        "NULL means3D": dict(means=None),
        "NULL features": dict(feat=None),
        "NULL dL_dout": dict(dout=None),
        "NULL scratch": dict(scratch=None),
        "no output at all": dict(dmeans=None, dopac=None, dscales=None, drot=None),
        "dL_dmeans3D missing": dict(dmeans=None),
        "dL_dopacity missing": dict(dopac=None),
        "dL_drotations missing": dict(drot=None),
        "radii missing (dense rows)": dict(radii=None),
        "dL_dcov3D without cov3D_precomp": dict(dcov=p(14 << 12)),
        "dL_dscales without scales": dict(scales=None, rots=None, cov=p(15 << 12), dcov=p(14 << 12)),
        "cov3D_precomp without dL_dcov3D": dict(scales=None, rots=None, cov=p(15 << 12), dscales=None, drot=None),
        "both geometry inputs": dict(cov=p(15 << 12)),
        "dL_dcamera without camera_scratch": dict(dcam=p(16 << 12)),
        "misaligned camera_scratch": dict(dcam=p(16 << 12), cam_scratch=p((17 << 12) + 4)),
        "misaligned features": dict(feat=p((7 << 12) + 2)),
        "misaligned dL_dout": dict(dout=p((8 << 12) + 1)),
        "misaligned dL_dmeans3D": dict(dmeans=p((10 << 12) + 2)),
        "misaligned rotations": dict(rots=p((3 << 12) + 4)),
        "misaligned dL_drotations": dict(drot=p((13 << 12) + 8)),
        "misaligned scratch": dict(scratch=p((9 << 12) + 4)),
    }
    for what, kw in bad.items():
        assert call(**kw) == -1, what
        msg = L.rtg_last_error()
        assert msg.startswith(SYM.encode() + b":") or b"exactly one of" in msg, (what, msg)
    assert b"C must be 1..128" in (call(C_=129), L.rtg_last_error())[1]
    assert b"without" in (call(dcov=p(14 << 12)), L.rtg_last_error())[1]
    for flags in (4, 1 << 30, -1):
        fv = _view(flags)
        assert call(view=C.byref(fv)) == -1
        assert b"unknown bits" in L.rtg_last_error()
    # P == 0 without a camera output: no row, no work, nothing dereferenced
    assert call(P=0, geom=None, img=None, bin_=None, counters=None, means=None, feat=None, dout=None, scratch=None) == 0
    # the pose-only form (every per-Gaussian output NULL) is accepted as far as the host goes: here it fails only for the
    # same missing workspace as the full one
    assert call(dmeans=None, dopac=None, dscales=None, drot=None, dcam=p(16 << 12), cam_scratch=p(17 << 12), geom=None) == -1
    assert b"NULL workspace" in L.rtg_last_error()


# ---------------------------------------------------------------------------------------------- Python argument checks
def test_python_argument_errors_are_raised_before_cuda():
    from rtg_slam_b200.features import rasterize_features
    P = 6
    args = (None, torch.zeros(P, 3), torch.zeros(P, 1), torch.zeros(P, 4))
    kw = dict(colors_precomp=torch.zeros(P, 3), scales=torch.zeros(P, 3), rotations=torch.zeros(P, 4))
    for bad in (1, 0, None, "yes", np.bool_(True), torch.tensor(True)):
        with pytest.raises(TypeError, match="weight_grad"):
            rasterize_features(*args, **kw, weight_grad=bad)
    with pytest.raises(TypeError):   # the feature checks still come before any CUDA work
        rasterize_features(*args, **kw, weight_grad=True)
