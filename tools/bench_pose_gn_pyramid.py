"""Coarse-to-fine, robust Gauss-Newton tracking on the benchmark scene (surfel room, 1 M Gaussians, seed 2024, SH degree
3) at 1200x680 and at a TUM-sized 640x480:

(a) ms per PoseRefiner.refine_gn iteration at each pyramid level s = 4, 2, 1 (the level camera and downsampled targets
    run as a single level), plain and with Huber weights: host clock around `iters` iterations that end in a device
    synchronise, best of `repeats`;
(b) device time per launch of frame_downsample_kernel (s = 2, 4) and of render_tangent_kernel's plain and robust
    normal-equation rows at full size, from torch.profiler's CUDA activity in a profiled run of its own;
(c) convergence from two starts -- 1 deg / 2 cm, and the start of the basin test (tests/test_pose_gn_pyramid_gpu.py,
    BASIN times that twist on the 140-pixel-focal test camera) scaled by 140 / fx so that it moves the image by as many
    pixels: the iterations and wall time (host clock, synchronised) to a tenth of both errors, or the errors after the
    last count tried, for refine (Adam, lr 1e-3), single-scale refine_gn, and refine_gn over scales (4, 2, 1) with Huber
    weights and n iterations per level.

The card name and power limit are read in the same run.

    python tools/bench_pose_gn_pyramid.py [--gaussians N] [--iters I] [--out FILE]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch

from rtg_slam_b200 import scene
from rtg_slam_b200.render import Renderer
from rtg_slam_b200.tracking import PoseRefiner, downsample_frame, level_camera
from test_pose_gn_pyramid_gpu import BASIN
from tools.bench_camera_grad import card
from tools.bench_pose_gn import OFF, pose_error, synced
from tools.bench_pose_refine import ARGS, se3_exp, view_camera

TEST_FX = 140.0  # the focal length of the basin test's camera ("small")


def tenth(err, err0):
    return err[0] < 0.1 * err0[0] and err[1] < 0.1 * err0[1]


def level_ms(ref, cam, g, tgt_c, tgt_d, w2c0, iters, repeats):
    """ms per iteration of each level run on its own (level camera, downsampled targets), plain and robust."""
    out = {}
    for s in (4, 2, 1):
        c0 = view_camera(cam, w2c0)
        if s == 1:
            lc, c, d = c0, tgt_c, tgt_d
        else:
            lc = level_camera(c0, s)
            c, d = downsample_frame(tgt_c, tgt_d[0], s)[:2]
        for robust in (None, "huber"):
            fn = lambda: ref.refine_gn(lc, g, c, d, iters=iters, color_weight=1.0, depth_weight=1.0, robust=robust)
            fn()
            out[f"level{s}_{'huber' if robust else 'plain'}_ms_per_iter"] = min(synced(fn)[1] for _ in range(repeats)) / iters
    return out


def kernel_ms(ref, cam, g, tgt_c, tgt_d, w2c0):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            for s in (2, 4):
                downsample_frame(tgt_c, tgt_d[0], s)
        for robust in (None, "huber"):
            ref.refine_gn(view_camera(cam, w2c0), g, tgt_c, tgt_d, iters=5, color_weight=1.0, depth_weight=1.0, robust=robust)
        torch.cuda.synchronize()
    kt = {}
    for e in prof.key_averages():
        k = e.key
        name = None
        if "frame_downsample_kernel" in k:
            name = "frame_downsample_ms"
        elif "render_tangent_kernel" in k and ("<1>" in k or "ILi1E" in k):
            name = "render_tangent_normal_eq_ms"
        elif "render_tangent_kernel" in k and ("<2>" in k or "ILi2E" in k):
            name = "render_tangent_normal_eq_robust_ms"
        elif "render_fwd_kernel" in k:
            name = "render_fwd_ms"
        if name:
            kt[name] = e.device_time_total / 1e3 / max(1, e.count)
    return kt


def convergence(ref, cam, g, tgt_c, tgt_d, w2c_true, w2c0, max_gn, max_levels, max_adam):
    err0 = pose_error(w2c0, w2c_true)
    res = dict(start_error_deg=err0[0], start_error_cm=100 * err0[1])
    gn = lambda **a: ref.refine_gn(view_camera(cam, w2c0), g, tgt_c, tgt_d, color_weight=1.0, depth_weight=1.0, **a)
    adam = lambda n: ref.refine(view_camera(cam, w2c0), g, tgt_c, tgt_d, iters=n, lr_rot=1e-3, lr_trans=1e-3, color_weight=1.0,
                                depth_weight=1.0)
    runs = (("gn", [dict(iters=n) for n in range(1, max_gn + 1)], lambda a: a["iters"]),
            ("pyramid_huber", [dict(iters=(n,) * 3, scales=(4, 2, 1), robust="huber") for n in range(1, max_levels + 1)],
             lambda a: sum(a["iters"])),
            ("adam", [n for n in range(25, max_adam + 1, 25)], lambda n: n))
    for name, tries, count in runs:
        res[f"{name}_iters"] = None
        for a in tries:
            (w2c, _), ms = synced(lambda: adam(a) if name == "adam" else gn(**a))
            err = pose_error(w2c, w2c_true)
            if tenth(err, err0):
                res.update({f"{name}_iters": count(a), f"{name}_wall_ms": ms})
                break
        res.update({f"{name}_error_deg": err[0], f"{name}_error_cm": 100 * err[1]})
        if res[f"{name}_iters"] is None:
            res[f"{name}_note"] = f"not reached within {count(a)} iterations"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--max-gn", type=int, default=20)
    ap.add_argument("--max-levels", type=int, default=8)
    ap.add_argument("--max-adam", type=int, default=300)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    g = {k: torch.from_numpy(v).to(dev) for k, v in scene.surfel_room(a.gaussians, seed=2024).items()}
    name, power = card()
    lines = []
    ref = PoseRefiner(ARGS)
    for cam_name in ("replica", "tum"):
        cam = scene.make_camera(cam_name)
        w2c_true = torch.eye(4, device=dev)
        with torch.no_grad():
            tgt = Renderer(ARGS).render(view_camera(cam, w2c_true), g)
        tgt_c, tgt_d = tgt["render"].clone(), tgt["depth"].clone()
        base = dict(gpu=name, power_limit=power, gaussians=a.gaussians, image=f"{cam.width}x{cam.height}")
        w2c0 = se3_exp(torch.tensor(OFF, device=dev)) @ w2c_true
        r = dict(base, what="cost")
        r.update(level_ms(ref, cam, g, tgt_c, tgt_d, w2c0, a.iters, a.repeats))
        r.update(kernel_ms(ref, cam, g, tgt_c, tgt_d, w2c0))
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
        for start, k in (("1deg_2cm", 1.0), ("basin_scaled", BASIN * TEST_FX / cam.fx)):
            w2c0 = se3_exp(k * torch.tensor(OFF, device=dev)) @ w2c_true
            r = dict(base, what="convergence", start=start, twist_scale=k)
            r.update(convergence(ref, cam, g, tgt_c, tgt_d, w2c_true, w2c0, a.max_gn, a.max_levels, a.max_adam))
            lines.append(json.dumps(r))
            print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
