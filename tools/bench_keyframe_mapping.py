"""Cost of refining keyframe poses and exposures with the map, per mapping iteration at 1200x680 with 1 M Gaussians
(scene.surfel_room, seed 2024). One iteration is Renderer.render at the keyframe's camera, loss.mapping_loss (colour L1,
depth L1 and the SSIM term: no render mask, so that the SSIM term and its exposure path run), backward and
MapOptimizer.step at the base.yaml rates, in four configurations:

    map          the map alone (the keyframe's pose and exposure fixed: the loop of before)
    exposure     + the keyframe's exposure (rtg_loss_mapping_exposure, rtg_ssim_loss_exposure, one FusedAdam step)
    pose         + the keyframe's pose (camera gradients in the backward, one rtg_pose_adam_step)
    both         both

The four alternate in rounds; each iteration is timed with CUDA events, and the per-iteration median, 10th and 90th
percentiles are printed. Then rtg_ssim_loss against rtg_ssim_loss_exposure on (3, 680, 1200) images, with both gradients,
per call. The card name and power limit are read in the same run. No device setting is changed.

    python tools/bench_keyframe_mapping.py [--gaussians 1000000] [--iters 50] [--warmup 10] [--rounds 3]"""
import argparse
import ctypes as C
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

ARGS = types.SimpleNamespace(renderer_opaque_threshold=0.6, renderer_normal_threshold=60, renderer_depth_threshold=1.0,
                             max_sh_degree=3, color_sigma=3.0, active_sh_degree=3)
LRS = dict(xyz=1e-3, f_dc=5e-4, f_rest=5e-4 / 20.0, opacity=0.0, scaling=4e-3, rotation=1e-3)   # configs/base.yaml:82-86


def camera(cam, w2c):
    import math
    return types.SimpleNamespace(FoVx=2 * math.atan(cam.tanfovx), FoVy=2 * math.atan(cam.tanfovy), image_height=cam.height,
                                 image_width=cam.width, world_view_transform=w2c.t().contiguous(),
                                 projection_matrix=torch.from_numpy(np.ascontiguousarray(cam.projection)).to(w2c.device),
                                 cx=cam.cx, cy=cam.cy)


def pct(xs):
    xs = np.sort(np.asarray(xs))
    return {"median": round(float(np.median(xs)), 4), "p10": round(float(np.percentile(xs, 10)), 4),
            "p90": round(float(np.percentile(xs, 90)), 4)}


def mapping(a, dev):
    from rtg_slam_b200 import scene
    from rtg_slam_b200.keyframes import KeyframeTable
    from rtg_slam_b200.loss import mapping_loss
    from rtg_slam_b200.mapoptim import MapOptimizer
    from rtg_slam_b200.render import Renderer
    from rtg_slam_b200.tracking import apply_exposure
    cam = scene.make_camera("replica")
    g = {k: torch.from_numpy(v).to(dev) for k, v in scene.surfel_room(a.gaussians, seed=2024).items()}
    w2c = torch.from_numpy(np.linalg.inv(scene.small_pose()).astype(np.float32)).to(dev)
    table0 = KeyframeTable(1e-3, 1e-3, 1e-2)
    k0 = table0.add(camera(cam, w2c), fix_pose=True)
    with torch.no_grad():
        tgt = Renderer(ARGS).render(table0.camera(k0), g)
    image = {"color_map": apply_exposure(tgt["render"], (0.2, 0.05)).contiguous(), "depth_map": tgt["depth"].contiguous()}
    start = w2c.clone()
    start[:3, 3] += 0.01
    shs = g["shs"]
    mo = MapOptimizer(g["xyz"], shs[:, :1].contiguous(), shs[:, 1:].contiguous(), torch.logit(g["opacity"].clamp(1e-4, 1 - 1e-4)),
                      torch.log(g["scales"]), g["rotations"], LRS)
    configs = {}
    for name, (pose, exposure) in {"map": (False, False), "exposure": (False, True), "pose": (True, False), "both": (True, True)}.items():
        t = KeyframeTable(1e-3, 1e-3, 1e-2)
        t.add(camera(cam, start), exposure=(0.0, 0.0) if exposure else None, fix_pose=not pose)
        configs[name] = t
    renderer = Renderer(ARGS)

    def iteration(t):
        out = renderer.render(t.camera(0), mo.gaussian_data())
        loss, _ = mapping_loss(out, image, None, ssim_weight=0.2, exposure=t.exposure(0))
        loss.backward()
        mo.step()
        t.step(0)

    for t in configs.values():
        for _ in range(a.warmup):
            iteration(t)
    torch.cuda.synchronize()
    times = {name: [] for name in configs}
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.iters)]
    for _ in range(a.rounds):
        for name, t in configs.items():
            for s, e in ev:
                s.record()
                iteration(t)
                e.record()
            torch.cuda.synchronize()
            times[name] += [s.elapsed_time(e) for s, e in ev]
    return {name: pct(v) for name, v in times.items()}


def ssim(a, dev):
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    Cn, H, W = 3, 680, 1200
    gen = torch.Generator(device=dev).manual_seed(0)
    x = torch.rand(Cn, H, W, device=dev, generator=gen)
    y = (0.7 * x + 0.3 * torch.rand(Cn, H, W, device=dev, generator=gen)).contiguous()
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    g, out, ge = torch.empty_like(x), torch.empty(2, device=dev), torch.empty(2, device=dev)
    e = torch.tensor([0.1, 0.02], device=dev)
    ws = torch.empty(L.rtg_ssim_exposure_workspace_bytes(Cn, H, W), dtype=torch.uint8, device=dev)
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    calls = {"rtg_ssim_loss": lambda: L.rtg_ssim_loss(p(x), p(y), Cn, H, W, p(g), p(out), p(ws), stream),
             "rtg_ssim_loss_exposure": lambda: L.rtg_ssim_loss_exposure(p(x), p(y), Cn, H, W, p(e), p(g), p(ge), p(out), p(ws), stream)}
    n = 200
    best = {k: float("inf") for k in calls}
    s, f = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for fn in calls.values():
        for _ in range(20):
            _lib.check(fn())
    for _ in range(a.rounds):
        for k, fn in calls.items():
            s.record()
            for _ in range(n):
                fn()
            f.record()
            f.synchronize()
            best[k] = min(best[k], s.elapsed_time(f) * 1e3 / n)
    return {k: round(v, 2) for k, v in best.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_keyframe_mapping needs a CUDA device")
    from tools.bench_camera_grad import card
    name, power = card()
    dev = torch.device("cuda", 0)
    res = {"card": name, "power_limit": power, "gaussians": a.gaussians, "size": "1200x680",
           "ms_per_mapping_iteration": mapping(a, dev), "ssim_us_per_call": ssim(a, dev)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
