"""Generates tests/golden/raster_inputs_*.npz from the reference's OWN CUDA rasterizer (oracle/_ref/_C_depth*.so, built by
oracle/build_ref.py) for two of GaussianRasterizer's alternative inputs: precomputed colours (some below 0 and above 1)
and an SH table of M = 4 coefficients (max_sh_degree 1). Needs an H100:

    python tests/golden/make_raster_inputs_golden.py [OUT_DIR]     # default: tests/golden

Precomputed covariances are not covered: the reference's render kernel reads scales[] unconditionally
(forward.cu:556,779), so it cannot run without them. Inputs are regenerated from the recipes below by the tests.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CASES = {
    # name: (scene fn, P, seed, camera, input mode)
    "raster_inputs_colors_small": ("surfel_room", 3000, 61, "small", "colors"),
    "raster_inputs_colors_ragged": ("random_blobs", 1500, 62, "ragged", "colors"),
    "raster_inputs_sh4_small": ("surfel_room", 3000, 63, "small", "sh4"),
    "raster_inputs_sh4_ragged": ("random_blobs", 1500, 64, "ragged", "sh4"),
}


def build_case(name):
    """(camera, inputs by name as the tests pass them, tile mask, upstream gradients, settings overrides)"""
    from rtg_slam_b200 import scene
    fn, P, seed, camname, mode = CASES[name]
    cam = scene.make_camera(camname)
    g = getattr(scene, fn)(P, seed=seed)
    inputs = {k: g[k] for k in ("xyz", "opacity", "scales", "rotations")}
    if mode == "colors":
        inputs["colors_precomp"] = np.random.default_rng(seed + 300).uniform(-0.25, 1.25, (P, 3)).astype(np.float32)
        over = {}
    else:
        inputs["shs"] = np.ascontiguousarray(g["shs"][:, :4])
        over = {"sh_degree": 1}
    return cam, inputs, None, scene.upstream_grads(cam, seed=seed + 200), over


def run_reference(cam, inputs, up, over, device):
    """rasterize_gaussians / rasterize_gaussians_backward of the reference, called as its python shim does
    (RAST/diff_gaussian_rasterization_depth/__init__.py:69-97,200-232); see tests/helpers.py:run_ref_cuda."""
    import torch
    import helpers
    mod = helpers.ref_cuda_module()
    assert mod is not None, "oracle/_ref/_C_depth*.so missing: run __graft_entry__.build() with the reference checkout"
    st = dict(helpers.DEFAULT_SETTINGS)
    st.update(over)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in inputs.items()}
    e = torch.Tensor([])
    cols, shs = t.get("colors_precomp", e), t.get("shs", e)
    H, W = cam.height, cam.width
    tm = torch.ones(((H + 15) // 16, (W + 15) // 16), dtype=torch.int32, device=device)
    bg = torch.zeros(3, dtype=torch.float32, device=device)
    vm, pm = torch.from_numpy(cam.viewmatrix).to(device), torch.from_numpy(cam.projmatrix).to(device)
    cp = torch.from_numpy(cam.campos).to(device)
    (num_rendered, num_tile, color, depth, hit_color, hit_depth, hcw, hdw, T_map, radii, geomB, binB, imgB, tile_indices) = \
        mod.rasterize_gaussians(bg, t["xyz"], cols, t["opacity"], t["scales"], t["rotations"], st["scale_modifier"], e, vm, pm, tm,
                                cam.tanfovx, cam.tanfovy, H, W, cam.cx, cam.cy, shs, st["sh_degree"], st["color_sigma"], cp,
                                st["opaque_threshold"], st["depth_threshold"], st["normal_threshold"], st["T_threshold"], False, False)
    res = dict(color=color, depth=depth, hit_color=hit_color, hit_depth=hit_depth, hit_color_weight=hcw, hit_depth_weight=hdw,
               T_map=T_map, radii=radii)
    res = {k: v.cpu().numpy() for k, v in res.items()}
    res["num_rendered"] = num_rendered
    gc, gd = (torch.from_numpy(x).to(device) for x in up)
    (g2d, gcol, gop, gm3, gcov, gsh, gsc, grot) = mod.rasterize_gaussians_backward(
        tile_indices, num_tile, bg, t["xyz"], radii, cols, t["scales"], t["rotations"], st["scale_modifier"], e, vm, pm, cam.tanfovx,
        cam.tanfovy, cam.cx, cam.cy, st["depth_threshold"], st["normal_threshold"], gc, gd, shs, st["sh_degree"], cp, geomB,
        num_rendered, binB, imgB, hit_depth, False)
    grads = dict(means3D=gm3, opacities=gop, scales=gsc, rotations=grot)
    if "colors_precomp" in inputs:
        grads["colors_precomp"] = gcol
    else:
        grads["shs"] = gsh
    res["grads"] = {k: v.cpu().numpy() for k, v in grads.items()}
    return res


def main():
    import torch
    import helpers
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.dirname(os.path.abspath(__file__))
    os.makedirs(out, exist_ok=True)
    dev = torch.device("cuda", 0)
    for name in CASES:
        cam, inputs, _, up, over = build_case(name)
        r = run_reference(cam, inputs, up, over, dev)
        r2 = run_reference(cam, inputs, up, over, dev)  # atomics jitter of the reference itself
        jit = {k: helpers.rel_err(r["grads"][k], r2["grads"][k]) for k in r["grads"]}
        np.savez_compressed(
            os.path.join(out, name + ".npz"),
            **{k: r[k] for k in ("color", "depth", "hit_color", "hit_depth", "hit_color_weight", "hit_depth_weight", "T_map", "radii")},
            num_rendered=np.int64(r["num_rendered"]),
            **{"grad_" + k: v for k, v in r["grads"].items()}, **{"jitter_" + k: np.float64(v) for k, v in jit.items()})
        print(name, "R", r["num_rendered"], "jitter", {k: f"{v:.1e}" for k, v in jit.items()})


if __name__ == "__main__":
    main()
