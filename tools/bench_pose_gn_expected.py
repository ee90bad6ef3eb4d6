"""Gauss-Newton tracking against the expected (alpha-blended) depth against the hit depth, on the benchmark scene (surfel
room, 1 M Gaussians, seed 2024, SH degree 3) at 1200x680 and 640x480, and on the GN test scene (tests/test_pose_gn_gpu.py
gn_inputs: 20 k surfels, 160x112):

(a) ms per PoseRefiner.refine_gn iteration, depth="hit" and "expected", plain and Huber: host clock around `iters`
    iterations that end in a device synchronise, best of `repeats`;
(b) device time per launch of the normal-equation rows (render_tangent_kernel<1|2> against
    render_tangent_expected_kernel<1|2>), from torch.profiler's CUDA activity in a profiled run of its own;
(c) the share of pixels in the expected-depth set S_e (m1 >= 0.5, gt_depth > 0, D - gt_depth < 0.1) against the hit-depth
    set (hit != -1, gt_depth > 0, depth - gt_depth < 0.1) at pyramid levels s = 1, 2, 4, plain and antialiased, at the
    1 deg / 2 cm start;
(d) convergence from 1 deg / 2 cm: single scale (12 iterations) and the pyramid (4, 2, 1) with coarse_antialias (4 per
    level); colour + depth and depth only; hit against expected: the remaining rotation and translation errors as
    fractions of the start.

The card name and power limit are read in the same run.

    python tools/bench_pose_gn_expected.py [--gaussians N] [--iters I] [--out FILE]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch

from rtg_slam_b200 import rasterizer, scene
from rtg_slam_b200.rasterizer import GaussianRasterizationSettings
from rtg_slam_b200.render import Renderer
from rtg_slam_b200.tracking import PoseRefiner, downsample_frame, level_camera, pose_jacobian
from tools.bench_camera_grad import card
from tools.bench_pose_gn import OFF, pose_error, synced
from tools.bench_pose_refine import ARGS, se3_exp, view_camera


def iter_ms(ref, cam, g, tgt_c, tgt_d, w2c0, iters, repeats):
    out = {}
    for depth in ("hit", "expected"):
        for robust in (None, "huber"):
            fn = lambda: ref.refine_gn(view_camera(cam, w2c0), g, tgt_c, tgt_d, iters=iters, color_weight=1.0, depth_weight=1.0,
                                       robust=robust, depth=depth)
            fn()
            out[f"{depth}_{'huber' if robust else 'plain'}_ms_per_iter"] = min(synced(fn)[1] for _ in range(repeats)) / iters
    return out


def kernel_ms(ref, cam, g, tgt_c, tgt_d, w2c0):
    for depth in ("hit", "expected"):  # warm
        ref.refine_gn(view_camera(cam, w2c0), g, tgt_c, tgt_d, iters=2, depth=depth)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for depth in ("hit", "expected"):
            for robust in (None, "huber"):
                ref.refine_gn(view_camera(cam, w2c0), g, tgt_c, tgt_d, iters=10, color_weight=1.0, depth_weight=1.0, robust=robust,
                              depth=depth)
        torch.cuda.synchronize()
    kt = {}
    for e in prof.key_averages():
        k = e.key
        for kern, tag in (("render_tangent_kernel", "hit"), ("render_tangent_expected_kernel", "expected")):
            if kern + "<" not in k and kern + "I" not in k and not k.startswith("void rtg::" + kern + "<"):
                continue
            if "<1," in k or "ILi1E" in k:
                kt[f"render_tangent_{tag}_plain_ms"] = e.device_time_total / 1e3 / max(1, e.count)
            elif "<2," in k or "ILi2E" in k:
                kt[f"render_tangent_{tag}_huber_ms"] = e.device_time_total / 1e3 / max(1, e.count)
        if "render_fwd_kernel" in k:
            kt["render_fwd_ms"] = e.device_time_total / 1e3 / max(1, e.count)
    return kt


def settings(camera, dev, w2c):
    r = Renderer(ARGS)
    import math
    view = w2c.t().contiguous()
    proj = (w2c.t().double() @ camera.projection_matrix.to(dev).double()).float().contiguous()
    campos = torch.linalg.inv(w2c.double())[:3, 3].float().contiguous()
    return GaussianRasterizationSettings(
        image_height=int(camera.image_height), image_width=int(camera.image_width), tanfovx=math.tan(camera.FoVx * 0.5),
        tanfovy=math.tan(camera.FoVy * 0.5), bg=r.bg_color.to(dev), scale_modifier=r.scaling_modifier, viewmatrix=view,
        projmatrix=proj, sh_degree=r.active_sh_degree, campos=campos, opaque_threshold=r.renderer_opaque_threshold,
        depth_threshold=r.renderer_depth_threshold, normal_threshold=r.renderer_normal_threshold, color_sigma=r.color_sigma,
        prefiltered=False, debug=False, cx=camera.cx, cy=camera.cy, T_threshold=0.0001)


def coverage(cam, g, tgt_c, tgt_d, w2c0, dev):
    """Shares of the level's pixels in S_e and in the hit-depth set, s = 1, 2, 4, plain and antialiased."""
    out = {}
    base = view_camera(cam, w2c0)
    t = dict(means3D=g["xyz"], opacities=g["opacity"], shs=g["shs"], scales=g["scales"], rotations=g["rotations"])
    for s in (1, 2, 4):
        lc = base if s == 1 else level_camera(base, s)
        gd = tgt_d[0] if s == 1 else downsample_frame(tgt_c, tgt_d[0], s)[1]
        for aa in (False, True):
            with rasterizer.antialiased(aa):
                outs, _, ex = pose_jacobian(settings(lc, dev, w2c0), depth="expected", **t)
            n = gd.numel()
            se = (ex[1] >= 0.5) & (gd > 0) & (ex[0] - gd < 0.1)
            sh = (outs[3][0] != -1) & (gd > 0) & (outs[1][0] - gd < 0.1)
            tag = f"s{s}_{'aa' if aa else 'plain'}"
            out[f"{tag}_expected_share"] = float(se.sum()) / n
            out[f"{tag}_hit_share"] = float(sh.sum()) / n
    return out


def convergence(ref, cam, g, tgt_c, tgt_d, w2c_true, w2c0):
    ang0, tr0 = pose_error(w2c0, w2c_true)
    res = dict(start_error_deg=ang0, start_error_cm=100 * tr0)
    for run, kw in (("single", dict(iters=12)), ("pyramid_aa", dict(iters=(4, 4, 4), scales=(4, 2, 1), coarse_antialias=True))):
        for terms, cw in (("colour_depth", 1.0), ("depth_only", 0.0)):
            for depth in ("hit", "expected"):
                (w2c, rep), ms = synced(lambda: ref.refine_gn(view_camera(cam, w2c0), g, tgt_c, tgt_d, color_weight=cw,
                                                              depth_weight=1.0, depth=depth, **kw))
                ang, tr = pose_error(w2c, w2c_true)
                res[f"{run}_{terms}_{depth}"] = dict(rotation=round(ang / ang0, 4), translation=round(tr / tr0, 4),
                                                    N_d=float(rep[4]), status=int(rep[7]), wall_ms=round(ms, 2))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    name, power = card()
    lines = []
    ref = PoseRefiner(ARGS)

    def emit(r):
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)

    g = {k: torch.from_numpy(v).to(dev) for k, v in scene.surfel_room(a.gaussians, seed=2024).items()}
    for cam_name in ("replica", "tum"):
        cam = scene.make_camera(cam_name)
        w2c_true = torch.eye(4, device=dev)
        with torch.no_grad():
            tgt = Renderer(ARGS).render(view_camera(cam, w2c_true), g)
        tgt_c, tgt_d = tgt["render"].clone(), tgt["depth"].clone()
        w2c0 = se3_exp(torch.tensor(OFF, device=dev)) @ w2c_true
        base = dict(gpu=name, power_limit=power, scene="room", gaussians=a.gaussians, image=f"{cam.width}x{cam.height}")
        r = dict(base, what="cost")
        r.update(iter_ms(ref, cam, g, tgt_c, tgt_d, w2c0, a.iters, a.repeats))
        r.update(kernel_ms(ref, cam, g, tgt_c, tgt_d, w2c0))
        emit(r)
        emit(dict(base, what="coverage", **coverage(cam, g, tgt_c, tgt_d, w2c0, dev)))
        if cam_name == "replica":
            emit(dict(base, what="convergence", **convergence(ref, cam, g, tgt_c, tgt_d, w2c_true, w2c0)))
    # the GN test scene (gn_inputs)
    from test_pose_gn_gpu import gn_inputs
    cam, gs, tgt, w2c_true, w2c0, _ = gn_inputs(dev)
    from test_pose_refine_gpu import refiner_camera
    base = dict(gpu=name, power_limit=power, scene="gn_inputs", gaussians=int(gs["xyz"].shape[0]), image=f"{cam.width}x{cam.height}")
    ang0, tr0 = pose_error(w2c0, w2c_true)
    conv = dict(start_error_deg=ang0, start_error_cm=100 * tr0)
    for run, kw in (("single", dict(iters=12)), ("pyramid_aa", dict(iters=(4, 4, 4), scales=(4, 2, 1), coarse_antialias=True))):
        for terms, cw in (("colour_depth", 1.0), ("depth_only", 0.0)):
            for depth in ("hit", "expected"):
                w2c, rep = ref.refine_gn(refiner_camera(cam, w2c0), gs, tgt["render"], tgt["depth"], color_weight=cw, depth_weight=1.0,
                                         depth=depth, **kw)
                ang, tr = pose_error(w2c, w2c_true)
                conv[f"{run}_{terms}_{depth}"] = dict(rotation=round(ang / ang0, 4), translation=round(tr / tr0, 4),
                                                     N_d=float(rep[4]), status=int(rep[7]))
    emit(dict(base, what="convergence", **conv))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
