"""Device time of the per-Gaussian contribution pass (rtg_splat_contributions) against the forward's compositing kernel
(render_fwd) of the same forward, at 1 M Gaussians, 1200x680 and 1920x1080.

    python tools/bench_contributions.py [--iters N] [--gaussians P]

Per camera: one forward (scene.surfel_room, seed 2024, all tiles), then N calls of the stats pass without and N with a
per-pixel error, alternating, each between two CUDA events (warm: a few untimed calls first); the median is reported.
render_fwd is timed by the library's own per-kernel events (rtg_profile_enable) over N forwards of the same frame. Prints
one JSON line with the card name and power limit read in the same run."""
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=60)
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    a = ap.parse_args()
    import numpy as np
    import torch

    import helpers
    from rtg_slam_b200 import _lib, rasterizer, scene
    from rtg_slam_b200._lib import check

    if not torch.cuda.is_available():
        raise SystemExit("bench_contributions needs a CUDA device")
    dev = torch.device("cuda", 0)
    rasterizer.set_capacity_checks("sync", dev)
    L = _lib.lib()
    g = helpers.to_torch(scene.surfel_room(a.gaussians, seed=2024), dev)
    P = a.gaussians
    res = {"card": card(), "gaussians": P, "iters": a.iters}
    for name in ("replica", "hd"):
        cam = scene.make_camera(name)
        rs = helpers.make_settings(cam, dev)
        args = (rs, g["xyz"], g["shs"], None, g["opacity"], g["scales"], g["rotations"], None, None)
        for _ in range(3):
            rasterizer._forward_native(*args)
        _lib.profile_enable(True)
        _lib.profile_read(reset=True)
        for _ in range(a.iters):
            rasterizer._forward_native(*args)
        prof = _lib.profile_read(reset=True)
        _lib.profile_enable(False)
        fwd_ms = prof["render_fwd"][0] / max(prof["render_fwd"][1], 1)
        outs, saved, _ = rasterizer._forward_native(*args)
        view, keep = rasterizer._make_view(rs, dev, saved.antialiased)
        n = torch.zeros(P, dtype=torch.int32, device=dev)
        w = torch.zeros(P, dtype=torch.float32, device=dev)
        err = torch.zeros(P, dtype=torch.float32, device=dev)
        e = torch.rand((cam.height, cam.width), device=dev)
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())

        def call(with_error):
            check(L.rtg_splat_contributions(C.byref(view), P, C.c_void_p(saved.geom), C.c_void_p(saved.img), C.c_void_p(saved.bin),
                                            saved.r_cap, C.c_void_p(saved.counters), ptr(e if with_error else None), ptr(n), ptr(w),
                                            ptr(err if with_error else None), stream), "rtg_splat_contributions")

        times = {False: [], True: []}
        for _ in range(5):
            call(False)
            call(True)
        for _ in range(a.iters):
            for we in (False, True):
                s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                call(we)
                t.record()
                t.synchronize()
                times[we].append(s.elapsed_time(t))
        pairs = int(n.sum().item()) // (5 + a.iters) // 2   # every call adds the frame's pairs once
        res[name] = {"render_fwd_ms": round(fwd_ms, 4),
                     "contributions_ms": round(float(np.median(times[False])), 4),
                     "contributions_error_ms": round(float(np.median(times[True])), 4),
                     "ratio_to_render_fwd": round(float(np.median(times[False])) / fwd_ms, 3),
                     "ratio_error_to_render_fwd": round(float(np.median(times[True])) / fwd_ms, 3),
                     "blended_pairs": pairs,
                     "gaussians_with_pixels": int((n > 0).sum().item()),
                     "visible": int((outs[7] > 0).sum().item())}
        torch.cuda.synchronize()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
