"""Cost of the camera gradient: the rasterizer backward with and without dL/d(viewmatrix, projmatrix, campos) at the
benchmark scene (surfel room, 1 M Gaussians, 1200x680, SH degree 3).

Each timed call is one backward of a fresh forward (the backward consumes the forward's gradient records). The two modes
alternate call by call so that both see the same machine state. Reported: the whole backward (CUDA events around
torch.autograd.backward) and the per-Gaussian pass alone (the library's event profiler, `preprocess_bwd`, which covers
the camera reduction too), median over the calls, with the card name and power limit read in the same run.

    python tools/bench_camera_grad.py [--gaussians N] [--calls K] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from rtg_slam_b200 import _lib, scene
from rtg_slam_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
    except Exception:  # noqa: BLE001 -- the numbers are still worth printing
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    cam = scene.make_camera("replica")
    g = {k: torch.from_numpy(v).to(dev) for k, v in scene.surfel_room(a.gaussians, seed=2024).items()}
    up = [torch.from_numpy(x).to(dev) for x in scene.upstream_grads(cam, seed=5)]
    leaves = {k: g[k].clone().requires_grad_(True) for k in ("xyz", "opacity", "shs", "scales", "rotations")}
    vm0, pm0, cp0 = (torch.from_numpy(x).to(dev) for x in (cam.viewmatrix, cam.projmatrix, cam.campos))

    def settings(camera):
        vm, pm, cp = (t.clone().requires_grad_(camera) for t in (vm0, pm0, cp0))
        return GaussianRasterizationSettings(
            image_height=cam.height, image_width=cam.width, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
            bg=torch.zeros(3, device=dev), scale_modifier=1.0, viewmatrix=vm, projmatrix=pm, sh_degree=3, campos=cp,
            opaque_threshold=0.6, normal_threshold=float(np.cos(np.deg2rad(60.0))), depth_threshold=1.0, prefiltered=False,
            debug=False, cx=cam.cx, cy=cam.cy), (vm, pm, cp)

    ev = lambda: torch.cuda.Event(enable_timing=True)

    def one(camera):
        rs, cam_t = settings(camera)
        out = GaussianRasterizer(rs)(means3D=leaves["xyz"], opacities=leaves["opacity"], shs=leaves["shs"],
                                     scales=leaves["scales"], rotations=leaves["rotations"])
        torch.cuda.synchronize()
        _lib.profile_read(reset=True)
        s, e = ev(), ev()
        s.record()
        torch.autograd.backward([out[0], out[1]], up)
        e.record()
        torch.cuda.synchronize()
        prof = _lib.profile_read(reset=True)["preprocess_bwd"]
        for t in list(leaves.values()) + list(cam_t):
            t.grad = None
        return s.elapsed_time(e), prof[0] / max(1, prof[1])

    _lib.profile_enable(True)
    for _ in range(a.warmup):
        one(False), one(True)
    res = {False: [], True: []}
    for _ in range(a.calls):
        for camera in (False, True):
            res[camera].append(one(camera))
    _lib.profile_enable(False)
    name, power = card()
    med = lambda xs, i: statistics.median(x[i] for x in xs)
    r = dict(gpu=name, power_limit=power, gaussians=a.gaussians, image=f"{cam.width}x{cam.height}", calls=a.calls,
             backward_ms_off=med(res[False], 0), backward_ms_on=med(res[True], 0),
             preprocess_bwd_ms_off=med(res[False], 1), preprocess_bwd_ms_on=med(res[True], 1))
    r["backward_ms_delta"] = r["backward_ms_on"] - r["backward_ms_off"]
    r["preprocess_bwd_ms_delta"] = r["preprocess_bwd_ms_on"] - r["preprocess_bwd_ms_off"]
    line = json.dumps(r)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
