"""Device time of per-Gaussian feature maps (rtg_splat_features and its backward) against the compositing kernels of the
same forward and against the workaround they replace, at 1 M Gaussians and 1200x680.

    python tools/bench_features.py [--iters N] [--gaussians P] [--camera replica|hd]

One frame: scene.surfel_room (seed 2024), all tiles, precomputed colours. render_fwd and render_bwd are timed by the
library's own per-kernel events (rtg_profile_enable) over N rasterizer forward + backward passes of the frame, which also
give the device time of all the library's kernels of one such pass. Then, for C in 1, 3, 8, 16, 32, 64, 128 and N
rounds, alternating within each round: the feature forward and the feature backward (its zero fill included) of that
frame's saved state, each between two CUDA events; the weight-gradient backward, dL/dF plus the geometry gradients through
the blend weights (rtg_splat_features_backward + rtg_splat_features_backward_geometry, dense rows, no camera), between two
CUDA events; and the workaround, ceil(C / 3) GaussianRasterizer forward + backward passes with the features as
`colors_precomp` three channels at a time (which give both halves of that gradient), between two CUDA events. Medians are reported,
after a few untimed rounds. Prints one JSON line with the card name, power limit and max SM clock read in the same run
and the blended (pixel, Gaussian) pairs of the frame."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CHANNELS = (1, 3, 8, 16, 32, 64, 128)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--camera", default="replica")
    a = ap.parse_args()
    import numpy as np
    import torch

    import helpers
    from rtg_slam_b200 import _lib, mapstats, rasterizer, scene
    from rtg_slam_b200._lib import check
    from rtg_slam_b200.rasterizer import GaussianRasterizer

    if not torch.cuda.is_available():
        raise SystemExit("bench_features needs a CUDA device")
    dev = torch.device("cuda", 0)
    L = _lib.lib()
    P = a.gaussians
    g = helpers.to_torch(scene.surfel_room(P, seed=2024), dev)
    cam = scene.make_camera(a.camera)
    H, W = cam.height, cam.width
    rs = helpers.make_settings(cam, dev)
    cols = torch.rand((P, 3), generator=torch.Generator(device=dev).manual_seed(1), device=dev)
    geo = dict(means3D=g["xyz"], opacities=g["opacity"], scales=g["scales"], rotations=g["rotations"])
    res = {"card": card(), "gaussians": P, "camera": a.camera, "height": H, "width": W, "iters": a.iters}

    def rasterizer_pass(colors, grad):
        c = colors.detach().requires_grad_(True)
        out = GaussianRasterizer(rs)(**geo, colors_precomp=c)
        torch.autograd.backward(out[0], grad)

    G3 = torch.rand((3, H, W), generator=torch.Generator(device=dev).manual_seed(2), device=dev)
    for _ in range(a.warmup):
        rasterizer_pass(cols, G3)
    _lib.profile_enable(True)
    _lib.profile_read(reset=True)
    for _ in range(a.iters):
        rasterizer_pass(cols, G3)
    prof = _lib.profile_read(reset=True)
    _lib.profile_enable(False)
    per = {k: v[0] / a.iters for k, v in prof.items() if v[1] > 0}
    res["render_fwd_ms"] = round(per["render_fwd"], 4)
    res["render_bwd_ms"] = round(per["render_bwd"], 4)
    res["rasterizer_pass_kernels_ms"] = round(sum(per.values()), 4)   # every library kernel of one forward + backward

    with torch.no_grad():
        _, st = mapstats.gaussian_contributions(rs, **geo, colors_precomp=cols)
    res["blended_pairs"] = int(st["n_pixels"].sum().item())

    with torch.no_grad():
        outs, saved, _ = rasterizer._forward_native(rs, geo["means3D"], None, cols, geo["opacities"], geo["scales"],
                                                    geo["rotations"], None, None)
    rasterizer._state(dev).read(saved.pending, block=True)
    assert not saved.pending.overflow
    view, keep = rasterizer._make_view(rs, dev, saved.antialiased)
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    ws = (C.c_void_p(saved.geom), C.c_void_p(saved.img), C.c_void_p(saved.bin), saved.r_cap, C.c_void_p(saved.counters))
    gen = torch.Generator(device=dev).manual_seed(3)
    data = {}
    for c in CHANNELS:
        F = torch.randn((P, c), generator=gen, device=dev)
        G = torch.rand((c, H, W), generator=gen, device=dev)
        n = -(-c // 3)
        Fp = torch.zeros((P, 3 * n), device=dev)
        Fp[:, :c] = F
        Gp = torch.zeros((3 * n, H, W), device=dev)
        Gp[:c] = G
        data[c] = (F, G, torch.empty((c, H, W), device=dev), torch.empty((P, c), device=dev),
                   [(Fp[:, 3 * k:3 * k + 3].contiguous(), Gp[3 * k:3 * k + 3].contiguous()) for k in range(n)])

    def feat_fwd(c):
        F, _, out, _, _ = data[c]
        check(L.rtg_splat_features(C.byref(view), P, *ws, c, C.c_void_p(F.data_ptr()), C.c_void_p(out.data_ptr()), stream),
              "rtg_splat_features")

    def feat_bwd(c):
        _, G, _, dF, _ = data[c]
        check(L.rtg_splat_features_backward(C.byref(view), P, *ws, c, C.c_void_p(G.data_ptr()), C.c_void_p(dF.data_ptr()),
                                            stream), "rtg_splat_features_backward")

    record = rasterizer._state(dev).get_scratch(P)
    grads = [torch.empty((P, k), device=dev) for k in (3, 1, 3, 4)]
    vp = lambda t: C.c_void_p(t.data_ptr())

    def weight_bwd(c):
        feat_bwd(c)
        F, G = data[c][0], data[c][1]
        check(L.rtg_splat_features_backward_geometry(
            C.byref(view), P, vp(geo["means3D"]), vp(geo["scales"]), vp(geo["rotations"]), None, vp(outs[7]), *ws, c, vp(F),
            vp(G), vp(record), *[vp(t) for t in grads], None, 0, None, None, stream), "rtg_splat_features_backward_geometry")

    def workaround(c):
        for Fk, Gk in data[c][4]:
            rasterizer_pass(Fk, Gk)

    def timed(fn, c):
        s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn(c)
        t.record()
        t.synchronize()
        return s.elapsed_time(t)

    times = {c: {"fwd": [], "bwd": [], "weight_bwd": [], "workaround": []} for c in CHANNELS}
    for i in range(a.warmup + a.iters):
        for c in CHANNELS:
            for key, fn in (("fwd", feat_fwd), ("bwd", feat_bwd), ("weight_bwd", weight_bwd), ("workaround", workaround)):
                ms = timed(fn, c)
                if i >= a.warmup:
                    times[c][key].append(ms)
    rows = {}
    for c in CHANNELS:
        med = {k: float(np.median(v)) for k, v in times[c].items()}
        total = med["fwd"] + med["bwd"]
        rows[str(c)] = {"features_fwd_ms": round(med["fwd"], 4), "features_bwd_ms": round(med["bwd"], 4),
                        "features_total_ms": round(total, 4), "workaround_passes": -(-c // 3),
                        "workaround_ms": round(med["workaround"], 4), "speedup": round(med["workaround"] / total, 2),
                        "fwd_ratio_to_render_fwd": round(med["fwd"] / per["render_fwd"], 3),
                        "bwd_ratio_to_render_bwd": round(med["bwd"] / per["render_bwd"], 3),
                        "weight_bwd_ms": round(med["weight_bwd"], 4),
                        "weight_total_ms": round(med["fwd"] + med["weight_bwd"], 4),
                        "weight_speedup": round(med["workaround"] / (med["fwd"] + med["weight_bwd"]), 2)}
    res["channels"] = rows
    torch.cuda.synchronize()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
