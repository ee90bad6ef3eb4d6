"""Cost of estimating the frame's exposure with the pose, on the benchmark scene (surfel room, 1 M Gaussians, seed 2024, SH
degree 3) at 1200x680 and at a TUM-sized 640x480. The frame is the render at the identity pose seen under the exposure
(a, b) = (0.2, 0.05); the start is 1 deg / 2 cm off.

(a) ms per PoseRefiner.refine_gn iteration without and with the exposure unknowns, plain and with Huber weights: the two
    alternate in one process, host clock around `iters` iterations that end in a device synchronise, best of `repeats`;
(b) device time per launch of render_tangent_kernel's four normal-equation instantiations and of the two step kernels,
    from torch.profiler's CUDA activity in a profiled run of its own;
(c) convergence from that start: the iterations to a tenth of both pose errors (or the errors after the last count tried)
    without and with the exposure unknowns, and the exposure estimate.

The card name and power limit are read in the same run. No device setting is changed.

    python tools/bench_pose_gn_exposure.py [--gaussians N] [--iters I] [--out FILE]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from rtg_slam_b200 import scene
from rtg_slam_b200.render import Renderer
from rtg_slam_b200.tracking import PoseRefiner, apply_exposure
from tools.bench_camera_grad import card
from tools.bench_pose_gn import OFF, pose_error, synced
from tools.bench_pose_refine import ARGS, se3_exp, view_camera

EXPOSURE = (0.2, 0.05)
KERNELS = {"ILi1E": "render_tangent_normal_eq_ms", "ILi2E": "render_tangent_normal_eq_robust_ms",
           "ILi3E": "render_tangent_normal_eq_exposure_ms", "ILi4E": "render_tangent_normal_eq_exposure_robust_ms",
           "<1>": "render_tangent_normal_eq_ms", "<2>": "render_tangent_normal_eq_robust_ms",
           "<3>": "render_tangent_normal_eq_exposure_ms", "<4>": "render_tangent_normal_eq_exposure_robust_ms"}


def cost(gn, iters, repeats):
    out = {}
    variants = [(robust, exposure) for robust in (None, "huber") for exposure in (None, (0.0, 0.0))]
    for v in variants:
        gn(iters=2, robust=v[0], exposure=v[1])  # module loads, allocator
    best = {v: float("inf") for v in variants}
    for _ in range(repeats):
        for v in variants:  # alternating, so that a drift of the clocks meets every variant alike
            best[v] = min(best[v], synced(lambda: gn(iters=iters, robust=v[0], exposure=v[1]))[1] / iters)
    for (robust, exposure), ms in best.items():
        out[f"{'huber' if robust else 'plain'}_{'exposure' if exposure else 'pose_only'}_ms_per_iter"] = ms
    return out


def kernel_ms(gn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for robust in (None, "huber"):
            for exposure in (None, (0.0, 0.0)):
                gn(iters=5, robust=robust, exposure=exposure)
        torch.cuda.synchronize()
    kt = {}
    for e in prof.key_averages():
        k = e.key
        name = None
        if "render_tangent_kernel" in k:
            name = next((v for tag, v in KERNELS.items() if tag in k), None)
        elif "pose_gn_exposure_step_kernel" in k:
            name = "pose_gn_exposure_step_ms"
        elif "pose_gn_step_kernel" in k:
            name = "pose_gn_step_ms"
        if name:
            kt[name] = e.device_time_total / 1e3 / max(1, e.count)
    return kt


def convergence(gn, w2c_true, w2c0, max_gn):
    err0 = pose_error(w2c0, w2c_true)
    res = dict(start_error_deg=err0[0], start_error_cm=100 * err0[1], exposure=list(EXPOSURE))
    for name, exposure in (("pose_only", None), ("exposure", (0.0, 0.0))):
        res[f"{name}_iters"] = None
        for n in range(1, max_gn + 1):
            out, ms = synced(lambda: gn(iters=n, robust=None, exposure=exposure))
            err = pose_error(out[0], w2c_true)
            if err[0] < 0.1 * err0[0] and err[1] < 0.1 * err0[1]:
                res.update({f"{name}_iters": n, f"{name}_wall_ms": ms})
                break
        res.update({f"{name}_error_deg": err[0], f"{name}_error_cm": 100 * err[1]})
        if exposure is not None:
            res["exposure_estimate"] = out[2].cpu().tolist()
        if res[f"{name}_iters"] is None:
            res[f"{name}_note"] = f"not reached within {max_gn} iterations"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--max-gn", type=int, default=15)
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
        tgt_c, tgt_d = apply_exposure(tgt["render"], EXPOSURE).contiguous(), tgt["depth"].clone()
        w2c0 = se3_exp(torch.tensor(OFF, device=dev)) @ w2c_true
        gn = lambda **kw: ref.refine_gn(view_camera(cam, w2c0), g, tgt_c, tgt_d, color_weight=1.0, depth_weight=1.0, **kw)
        base = dict(gpu=name, power_limit=power, gaussians=a.gaussians, image=f"{cam.width}x{cam.height}")
        r = dict(base, what="cost")
        r.update(cost(gn, a.iters, a.repeats))
        r.update(kernel_ms(gn))
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
        r = dict(base, what="convergence")
        r.update(convergence(gn, w2c_true, w2c0, a.max_gn))
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
