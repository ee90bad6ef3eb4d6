"""GPU tests of the rasterizer's alternative inputs (GaussianRasterizer's operator API): precomputed colours, precomputed
3-D covariances, SH tables narrower than 16 coefficients, scale_modifier != 1, the optional gradient outputs of the C ABI
(dL/dcolors_precomp, dL/dcov3D, dL/dmeans2D) and inputs that are contiguous views at an offset into their storage.

Metrics as in test_raster_gpu.py: float maps L_inf < 1e-4 outside the oracle's tie mask, per-tensor gradient
max|g-g_ref| / max|g_ref| < 1e-3 against the f32 oracle. Comparisons of two runs of this library that differ only in how
the same values are passed are bit-exact in the forward and, in the gradients, within max(1e-5, 10 x the run-to-run
difference of one of them repeated): the compositing backward accumulates with atomics, so its summation order varies
from run to run, and where a gradient cancels (translucent blobs) that moves it by more than 1e-5 of its largest entry."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import helpers
from golden.make_raster_inputs_golden import CASES as GOLDEN_CASES, build_case as golden_case
from oracle.splat_oracle import OracleRender
from rtg_slam_b200 import scene

pytestmark = pytest.mark.gpu
NAMES = ("color", "depth", "hit_color", "hit_depth", "hit_color_weight", "hit_depth_weight", "T_map", "radii")
COLOR_SIDE = ("color", "hit_color", "hit_color_weight", "T_map", "radii")
GRADS = ("means3D", "shs", "opacities", "scales", "rotations")
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# input name -> (GaussianRasterizer keyword, gradient name)
INPUTS = {"xyz": ("means3D", "means3D"), "opacity": ("opacities", "opacities"), "shs": ("shs", "shs"),
          "colors_precomp": ("colors_precomp", "colors_precomp"), "scales": ("scales", "scales"),
          "rotations": ("rotations", "rotations"), "cov3D_precomp": ("cov3D_precomp", "cov3D_precomp")}


def scene_case(name):
    """Small scenes: a surfel room, ragged image size (H, W not multiples of 16), a tile mask, and translucent blobs whose
    tile lists are longer than 4096 entries."""
    if name == "small":
        return scene.make_camera("small"), scene.surfel_room(3000, seed=41), None
    if name == "ragged":
        return scene.make_camera("ragged"), scene.random_blobs(1500, seed=42), None
    if name == "masked":
        cam = scene.make_camera("small", c2w=scene.small_pose())
        return cam, scene.surfel_room(3000, seed=43), scene.random_tile_mask(cam, 0.5, seed=143)
    assert name == "dense"
    return scene.make_camera("tiny"), scene.dense_blobs(30_000, seed=44), None


SCENES = ("small", "ragged", "masked", "dense")


def culled_scene():
    """P not a multiple of 32, about half of the Gaussians culled (behind the near plane or outside the frustum)."""
    return scene.make_camera("ragged"), scene.random_blobs(1037, seed=45)


def pick(g, *keys, **extra):
    d = {k: g[k] for k in keys}
    d.update(extra)
    return d


def cov3d_f64(scales, rotations, mod=1.0):
    """Sigma = R S S R^T from the quaternion as given (not normalised, computeCov3D), in float64, rounded to float32."""
    r, x, y, z = rotations.astype(np.float64).T
    R = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
                  np.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
                  np.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], 1)
    Ms = R * (mod * scales.astype(np.float64))[:, None, :]
    S = Ms @ Ms.transpose(0, 2, 1)
    return np.ascontiguousarray(S[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].astype(np.float32))


def render(cam, inputs, dev, mask=None, grads=None, **over):
    """Forward (and backward for `grads` = (dL/dcolor, dL/ddepth)) through GaussianRasterizer with exactly the inputs given
    (numpy arrays, or CUDA tensors that are passed as they are)."""
    from rtg_slam_b200.rasterizer import GaussianRasterizer
    rs = helpers.make_settings(cam, dev, **over)
    leaves = {k: (v if isinstance(v, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(v)).to(dev)) for k, v in inputs.items()}
    for v in leaves.values():
        v.requires_grad_(grads is not None)
    tm = None if mask is None else torch.from_numpy(np.ascontiguousarray(mask, dtype=np.int32)).to(dev)
    out = GaussianRasterizer(rs)(**{INPUTS[k][0]: v for k, v in leaves.items()}, tile_mask=tm)
    res = dict(zip(NAMES, [o.detach().cpu().numpy() for o in out]))
    if grads is not None:
        gc, gd = (torch.from_numpy(x).to(dev) for x in grads)
        ((out[0] * gc).sum() + (out[1] * gd).sum()).backward()
        res["grads"] = {INPUTS[k][1]: v.grad.cpu().numpy() for k, v in leaves.items()}
    return res


def oracle(cam, inputs, mask=None, **over):
    g = {k: inputs.get(k) for k in ("xyz", "opacity", "shs", "scales", "rotations")}
    return OracleRender(cam, g, tile_mask=mask, precision="f32", tie_eps=1e-4, colors_precomp=inputs.get("colors_precomp"),
                        cov3D_precomp=inputs.get("cov3D_precomp"), **over)


def compare(a, b, tie, keys=NAMES, label=""):
    """helpers.compare_outputs restricted to `keys` (the others are taken from `b`)."""
    a = dict(a, **{k: b[k] for k in NAMES if k not in keys})
    st = helpers.compare_outputs(a, b, tie=tie, tol=1e-4, label=label)
    assert st["radii_mismatch"] <= max(0, int(1e-5 * len(b["radii"]))), (label, st)
    return st


def check_against_oracle(ours, o, upstream, grad_keys, keys=NAMES, label=""):
    compare(ours, dict(zip(NAMES, o.outputs())), o.tie, keys, label)
    og = o.backward(*upstream)
    for k in grad_keys:
        assert np.abs(og[k]).max() > 0, (label, k)
        e = helpers.rel_err(ours["grads"][k], og[k])
        assert e < 1e-3, f"{label}: d{k} rel err {e:.2e}"
    return og


def grad_tol(a, a_again, k):
    """max(1e-5, 10 x the run-to-run relative difference of gradient k between two runs on the same inputs)."""
    return max(1e-5, 10 * helpers.rel_err(a_again["grads"][k], a["grads"][k]))


def assert_identical_forward(a, b, label=""):
    for k in NAMES:
        assert np.array_equal(a[k], b[k]), (label, k)


# ---------------------------------------------------------------------------------------------------- a. colors_precomp
@pytest.mark.parametrize("case", SCENES)
def test_colors_precomp_matches_oracle(cuda_device, case):
    """Precomputed colours below 0 and above 1 (they are not clamped, unlike SH colours): every output and the gradients
    of means3D, opacities, scales, rotations and colors_precomp."""
    cam, g, mask = scene_case(case)
    cols = np.random.default_rng(46).uniform(-0.25, 1.25, (len(g["xyz"]), 3)).astype(np.float32)
    inputs = pick(g, "xyz", "opacity", "scales", "rotations", colors_precomp=cols)
    up = scene.upstream_grads(cam, seed=5)
    ours = render(cam, inputs, cuda_device, mask, grads=up)
    o = oracle(cam, inputs, mask)
    check_against_oracle(ours, o, up, ("means3D", "opacities", "scales", "rotations", "colors_precomp"), label=case)
    if case == "dense":
        _, rg = o.binning()
        assert int((rg[:, 1] - rg[:, 0]).max()) > 4096


# ---------------------------------------------------------------------------------------------------- b. cov3D_precomp
@pytest.mark.parametrize("case", SCENES)
def test_cov3D_precomp_matches_oracle(cuda_device, case):
    """Colour side and the gradients of means3D, opacities, shs and cov3D_precomp with dL/ddepth = 0. Without scales a
    Gaussian has no surfel (DESIGN.md section 4): with a non-zero dL/ddepth every output and gradient is finite, and the
    depth side is the centre depth of the first opaque Gaussian, as the oracle defines it."""
    cam, g, mask = scene_case(case)
    inputs = pick(g, "xyz", "opacity", "shs", cov3D_precomp=cov3d_f64(g["scales"], g["rotations"]))
    gc, gd = scene.upstream_grads(cam, seed=5)
    ours = render(cam, inputs, cuda_device, mask, grads=(gc, np.zeros_like(gd)))
    o = oracle(cam, inputs, mask)
    check_against_oracle(ours, o, (gc, np.zeros_like(gd)), ("means3D", "opacities", "shs", "cov3D_precomp"), COLOR_SIDE, case)

    full = render(cam, inputs, cuda_device, mask, grads=(gc, gd))
    for k in NAMES:
        assert np.isfinite(full[k]).all(), k
    for k, v in full["grads"].items():
        assert np.isfinite(v).all(), k
    check_against_oracle(full, o, (gc, gd), ("means3D",), NAMES, case + " depth side")

    # the same covariance from scales / rotations: same colour side
    sr = render(cam, pick(g, "xyz", "opacity", "shs", "scales", "rotations"), cuda_device, mask)
    compare(ours, sr, oracle(cam, pick(g, "xyz", "opacity", "shs", "scales", "rotations"), mask).tie, COLOR_SIDE, case + " vs scales")


# ---------------------------------------------------------------------------------------------------- c. short SH tables
SH_CASES = [(M, deg) for M in (1, 4, 9) for deg in range(int(round(np.sqrt(M))))]


@pytest.mark.parametrize("M,deg", SH_CASES)
def test_short_sh_table_matches_zero_padded_table(cuda_device, M, deg):
    """M = (max_sh_degree + 1)^2 < 16 coefficients per row: the forward is bit-identical to the same coefficients
    zero-padded to 16 (only the load differs), dL/dshs equals the padded run's first M columns, the padded columns get
    exactly 0, culled rows exactly 0, and both runs match the oracle."""
    cam, g = culled_scene()
    P = len(g["xyz"])
    shs = np.ascontiguousarray(g["shs"][:, :M])
    pad = np.zeros((P, 16, 3), np.float32)
    pad[:, :M] = shs
    up = scene.upstream_grads(cam, seed=6)
    short = render(cam, pick(g, "xyz", "opacity", "scales", "rotations", shs=shs), cuda_device, grads=up, sh_degree=deg)
    full = render(cam, pick(g, "xyz", "opacity", "scales", "rotations", shs=pad), cuda_device, grads=up, sh_degree=deg)
    again = render(cam, pick(g, "xyz", "opacity", "scales", "rotations", shs=pad), cuda_device, grads=up, sh_degree=deg)
    assert_identical_forward(short, full, f"M={M} deg={deg}")
    assert short["grads"]["shs"].shape == (P, M, 3)
    assert helpers.rel_err(short["grads"]["shs"], full["grads"]["shs"][:, :M]) < grad_tol(full, again, "shs")
    assert np.all(full["grads"]["shs"][:, M:] == 0)
    culled = short["radii"] == 0
    assert P % 32 and culled.sum() > P // 4
    for r in (short, full):
        for k, v in r["grads"].items():
            assert np.all(v[culled] == 0), k
    og = check_against_oracle(short, oracle(cam, pick(g, "xyz", "opacity", "scales", "rotations", shs=shs), sh_degree=deg), up,
                              GRADS, label=f"M={M} deg={deg}")
    for k in GRADS:
        assert helpers.rel_err(full["grads"][k][:, :M] if k == "shs" else full["grads"][k], og[k]) < 1e-3, k


# ---------------------------------------------------------------------------------------------------- d. scale_modifier
@pytest.mark.parametrize("mod", [0.5, 1.7])
def test_scale_modifier(cuda_device, mod):
    """Against the oracle; and metamorphic: (float32(s * scales), modifier 1) and (scales, modifier s) form the same float32
    product, so their forwards are bit-identical. Like the reference (computeCov3D, backward.cu:426-487), dL/dscales is
    the gradient with respect to the scaled scales, so it is the same in both runs. The check runs with dL/ddepth = 0:
    the depth-hit backward compares with max(scales) without the modifier, as the reference does (backward.cu:1009)."""
    cam, g, mask = scene_case("small")
    inputs = pick(g, "xyz", "opacity", "shs", "scales", "rotations")
    up = scene.upstream_grads(cam, seed=5)
    ours = render(cam, inputs, cuda_device, mask, grads=up, scale_modifier=mod)
    check_against_oracle(ours, oracle(cam, inputs, mask, scale_modifier=mod), up, GRADS, label=f"modifier {mod}")

    up0 = (up[0], np.zeros_like(up[1]))
    pre = render(cam, dict(inputs, scales=np.float32(mod) * g["scales"]), cuda_device, mask, grads=up0, scale_modifier=1.0)
    again = render(cam, dict(inputs, scales=np.float32(mod) * g["scales"]), cuda_device, mask, grads=up0, scale_modifier=1.0)
    mdf = render(cam, inputs, cuda_device, mask, grads=up0, scale_modifier=mod)
    assert_identical_forward(pre, mdf, f"modifier {mod}")
    for k in GRADS:
        assert helpers.rel_err(mdf["grads"][k], pre["grads"][k]) < grad_tol(pre, again, k), k


# ---------------------------------------------------------------------------------------------------- e. optional outputs
def native_backward(cam, inputs, dev, up, **over):
    """Forward through the operator's native call, then rtg_splat_backward through the C ABI with every gradient output --
    including the optional dL/dcolors_precomp, dL/dcov3D and dL/dmeans2D -- pre-filled with NaN."""
    from rtg_slam_b200 import _lib, rasterizer as R
    rs = helpers.make_settings(cam, dev, **over)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in inputs.items()}
    outs, saved, ins = R._forward_native(rs, t["xyz"], t.get("shs"), t.get("colors_precomp"), t["opacity"], t.get("scales"),
                                         t.get("rotations"), t.get("cov3D_precomp"), None)
    means3D, sh, colors, scales, rots, cov = ins
    st = R._state(dev)
    st.read(saved.pending, block=True)
    assert not saved.pending.overflow
    P, M = means3D.size(0), (sh.size(1) if sh is not None else 0)
    nan = lambda *s: torch.full(s, float("nan"), dtype=torch.float32, device=dev)
    out = {"means3D": nan(P, 3), "opacities": nan(P, 1), "colors": nan(P, 3), "cov3D": nan(P, 6), "means2D": nan(P, 3),
           "shs": nan(P, M, 3) if sh is not None else None, "scales": nan(P, 3) if scales is not None else None,
           "rotations": nan(P, 4) if rots is not None else None}
    view, keep = R._make_view(rs, dev)
    gc, gd = (torch.from_numpy(x).to(dev) for x in up)
    p = R._ptr
    L = _lib.lib()
    _lib.check(L.rtg_splat_backward(
        C.byref(view), P, M, p(means3D), p(sh), p(colors), p(scales), p(rots), p(cov), p(outs[7]), C.c_void_p(saved.geom),
        C.c_void_p(saved.img), C.c_void_p(saved.bin), saved.r_cap, C.c_void_p(saved.counters), p(outs[6]), p(outs[3]), p(gc),
        p(gd), p(st.get_scratch(P)), p(out["means3D"]), p(out["shs"]), p(out["colors"]), p(out["opacities"]), p(out["scales"]),
        p(out["rotations"]), p(out["cov3D"]), p(out["means2D"]), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
        "rtg_splat_backward")
    torch.cuda.synchronize(dev)
    return outs[7].cpu().numpy(), {k: v.cpu().numpy() for k, v in out.items() if v is not None}


@pytest.mark.parametrize("mode", ["sh16", "sh4", "precomp"])
def test_optional_gradient_outputs_of_the_c_abi(cuda_device, mode):
    """Every row of every gradient output is written (culled rows exactly 0); dL/dcolors, dL/dcov3D and dL/dmeans2D
    (third component 0) match the oracle's intermediates."""
    cam, g = culled_scene()
    if mode == "precomp":
        cols = np.random.default_rng(47).uniform(-0.25, 1.25, (len(g["xyz"]), 3)).astype(np.float32)
        inputs = pick(g, "xyz", "opacity", colors_precomp=cols, cov3D_precomp=cov3d_f64(g["scales"], g["rotations"]))
        over = {}
    else:
        M = 16 if mode == "sh16" else 4
        inputs = pick(g, "xyz", "opacity", "scales", "rotations", shs=np.ascontiguousarray(g["shs"][:, :M]))
        over = dict(sh_degree=3 if M == 16 else 1)
    up = scene.upstream_grads(cam, seed=7)
    radii, ours = native_backward(cam, inputs, cuda_device, up, **over)
    culled = radii == 0
    assert culled.sum() > len(radii) // 4
    for k, v in ours.items():
        assert not np.isnan(v).any(), f"{mode}: d{k} has unwritten rows"
        assert np.all(v[culled] == 0), k
    assert np.all(ours["means2D"][:, 2] == 0)
    og = oracle(cam, inputs, **over).backward(*up)
    for k in ours:
        ref = og[k]
        assert np.abs(ref).max() > 0, k
        assert helpers.rel_err(ours[k], ref) < 1e-3, (mode, k, helpers.rel_err(ours[k], ref))


# ---------------------------------------------------------------------------------------------------- f. shim checks
def misaligned(a, dev):
    """A contiguous CUDA view of `a` that starts 4 bytes into its storage."""
    flat = torch.empty(a.size + 1, dtype=torch.float32, device=dev)
    v = flat[1:].view(a.shape)
    v.copy_(torch.from_numpy(np.ascontiguousarray(a)))
    assert v.is_contiguous() and v.data_ptr() % 16 == 4
    return v


def test_misaligned_inputs_are_copied(cuda_device):
    cam, g, _ = scene_case("ragged")
    inputs = pick(g, "xyz", "opacity", "shs", "scales", "rotations")
    up = scene.upstream_grads(cam, seed=5)
    ref = render(cam, inputs, cuda_device, grads=up)
    again = render(cam, inputs, cuda_device, grads=up)
    mis = render(cam, {k: misaligned(v, cuda_device) for k, v in inputs.items()}, cuda_device, grads=up)
    assert_identical_forward(mis, ref)
    for k in GRADS:
        assert helpers.rel_err(mis["grads"][k], ref["grads"][k]) < grad_tol(ref, again, k), k


def test_misaligned_grad_buffer_is_rejected(cuda_device):
    from rtg_slam_b200.rasterizer import grad_buffers
    cam, g, _ = scene_case("ragged")
    bad = misaligned(np.zeros((len(g["xyz"]), 4), np.float32), cuda_device)
    with grad_buffers({"rotations": bad}), pytest.raises(ValueError, match="16-byte aligned"):
        render(cam, pick(g, "xyz", "opacity", "shs", "scales", "rotations"), cuda_device, grads=scene.upstream_grads(cam))


def test_sh_degree_beyond_the_table_is_rejected(cuda_device):
    cam, g, _ = scene_case("ragged")
    inputs = pick(g, "xyz", "opacity", "scales", "rotations", shs=np.ascontiguousarray(g["shs"][:, :4]))
    with pytest.raises(ValueError, match="needs 16 SH coefficients"):
        render(cam, inputs, cuda_device, sh_degree=3)


# ---------------------------------------------------------------------------------------------------- reference goldens
@pytest.mark.parametrize("name", sorted(GOLDEN_CASES))
def test_matches_reference_cuda_golden(cuda_device, name):
    """Against stored outputs of the reference's own CUDA rasterizer (tests/golden/make_raster_inputs_golden.py)."""
    gold = np.load(os.path.join(GOLD, name + ".npz"))
    cam, inputs, mask, up, over = golden_case(name)
    ours = render(cam, inputs, cuda_device, mask, grads=up, **over)
    o = oracle(cam, inputs, mask, **over)  # only for the tie mask
    st = helpers.compare_outputs(ours, {k: gold[k] for k in NAMES}, tie=o.tie, tol=1e-4, label=name)
    assert st["radii_mismatch"] == 0
    for k in ours["grads"]:
        tol = max(1e-3, 10 * float(gold["jitter_" + k]))
        assert helpers.rel_err(ours["grads"][k], gold["grad_" + k]) < tol, k
