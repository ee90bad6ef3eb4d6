"""Cost of the Gauss-Newton pose refiner against the Adam one, on the benchmark scene (surfel room, 1 M Gaussians, SH
degree 3) at 1200x680 and at a TUM-sized 640x480:

(a) ms per iteration of PoseRefiner.refine_gn and PoseRefiner.refine (host clock around `iters` iterations that end in a
    device synchronise, best of `repeats`), from 1 deg / 2 cm off the pose the targets were rendered at;
(b) the two new kernels, preprocess_tangent_kernel and render_tangent_kernel (both modes), and the forward's render kernel
    for scale: mean device time per launch from torch.profiler's CUDA activity, in a profiled run of its own;
(c) convergence: the iterations Gauss-Newton needs to bring both errors to a tenth of their start, the error it reaches,
    and the iterations and wall time (host clock, synchronised) Adam (lr 1e-3) needs to reach the same error.

The card name and power limit are read in the same run.

    python tools/bench_pose_gn.py [--gaussians N] [--iters I] [--out FILE]"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from rtg_slam_b200 import scene
from rtg_slam_b200.render import Renderer
from rtg_slam_b200.tracking import PoseRefiner, pose_jacobian
from tools.bench_camera_grad import card
from tools.bench_pose_refine import ARGS, se3_exp, view_camera

OFF = (0.012, -0.010, 0.012, 0.010, -0.012, 0.008)  # 2 cm, 1.0 deg


def pose_error(w2c, w2c_true):
    d = (w2c.double() @ torch.linalg.inv(w2c_true.double())).cpu()
    ang = float(torch.rad2deg(torch.arccos(((torch.trace(d[:3, :3]) - 1) / 2).clamp(-1, 1))))
    c = torch.linalg.inv(w2c.double().cpu())[:3, 3] - torch.linalg.inv(w2c_true.double().cpu())[:3, 3]
    return ang, float(c.norm())


def synced(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def run(cam, g, dev, iters, repeats, max_adam):
    r = Renderer(ARGS)
    w2c_true = torch.eye(4, device=dev)
    with torch.no_grad():
        tgt = r.render(view_camera(cam, w2c_true), g)
    tgt_c, tgt_d = tgt["render"].clone(), tgt["depth"].clone()
    w2c0 = se3_exp(torch.tensor(OFF, device=dev)) @ w2c_true
    ang0, tr0 = pose_error(w2c0, w2c_true)
    ref = PoseRefiner(ARGS)
    gn = lambda n: ref.refine_gn(view_camera(cam, w2c0), g, tgt_c, tgt_d, iters=n, color_weight=1.0, depth_weight=1.0)
    adam = lambda n: ref.refine(view_camera(cam, w2c0), g, tgt_c, tgt_d, iters=n, lr_rot=1e-3, lr_trans=1e-3, color_weight=1.0,
                                depth_weight=1.0)
    gn(2), adam(2)  # first forward of the shape, module loads, allocator
    res = dict(start_error_deg=ang0, start_error_cm=100 * tr0)
    res["refine_gn_ms_per_iter"] = min(synced(lambda: gn(iters))[1] for _ in range(repeats)) / iters
    res["refine_adam_ms_per_iter"] = min(synced(lambda: adam(iters))[1] for _ in range(repeats)) / iters

    # (b) kernel times, profiled run of its own
    rs = r_settings(cam, dev)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            pose_jacobian(rs, g["xyz"], g["opacity"], shs=g["shs"], scales=g["scales"], rotations=g["rotations"])
        gn(5)
        torch.cuda.synchronize()
    kt = {}
    for e in prof.key_averages():
        k = e.key
        if "render_tangent_kernel" in k:
            name = "render_tangent_images_ms" if ("<0>" in k or "ILi0E" in k) else "render_tangent_normal_eq_ms"
        else:
            name = next((n + "_ms" for n in ("preprocess_tangent_kernel", "pose_gn_step_kernel", "render_fwd_kernel") if n in k), None)
        if name:
            kt[name] = e.device_time_total / 1e3 / max(1, e.count)
    res.update(kt)

    # (c) convergence: Gauss-Newton to a tenth of both errors, Adam to the error Gauss-Newton reached
    for n in range(1, 21):
        (w2c, _), ms = synced(lambda: gn(n))
        ang, tr = pose_error(w2c, w2c_true)
        if ang < 0.1 * ang0 and tr < 0.1 * tr0:
            break
    res.update(gn_iters=n, gn_wall_ms=ms, gn_error_deg=ang, gn_error_cm=100 * tr)
    target = (ang, tr)
    res.update(adam_iters=None, adam_wall_ms=None)
    for n in range(25, max_adam + 1, 25):
        (w2c, _), ms = synced(lambda: adam(n))
        a2, t2 = pose_error(w2c, w2c_true)
        if a2 <= target[0] and t2 <= target[1]:
            res.update(adam_iters=n, adam_wall_ms=ms, adam_error_deg=a2, adam_error_cm=100 * t2)
            break
    if res["adam_iters"] is None:
        res.update(adam_error_deg=a2, adam_error_cm=100 * t2, adam_note=f"not reached within {max_adam} iterations")
    return res


def r_settings(cam, dev):
    from rtg_slam_b200.rasterizer import GaussianRasterizationSettings
    import numpy as np
    return GaussianRasterizationSettings(
        image_height=cam.height, image_width=cam.width, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=torch.zeros(3, device=dev),
        scale_modifier=1.0, viewmatrix=torch.from_numpy(cam.viewmatrix).to(dev), projmatrix=torch.from_numpy(cam.projmatrix).to(dev),
        sh_degree=3, campos=torch.from_numpy(cam.campos).to(dev), opaque_threshold=0.6,
        normal_threshold=float(np.cos(np.deg2rad(60.0))), depth_threshold=1.0, prefiltered=False, debug=False, cx=cam.cx, cy=cam.cy)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--max-adam", type=int, default=300)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    g = {k: torch.from_numpy(v).to(dev) for k, v in scene.surfel_room(a.gaussians, seed=2024).items()}
    name, power = card()
    lines = []
    for cam_name in ("replica", "tum"):
        cam = scene.make_camera(cam_name)
        r = dict(gpu=name, power_limit=power, gaussians=a.gaussians, image=f"{cam.width}x{cam.height}")
        r.update(run(cam, g, dev, a.iters, a.repeats, a.max_adam))
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
