"""Device time of the TSDF ray-cast (rtg_tsdf_raycast, `TsdfVolume.raycast`).

Volumes as in tools/bench_tsdf.py: 301x151x301 voxels at 2 cm over the benchmark room and 512^3 voxels at 1.25 cm over a
6.4 m cube around it, both with colour, each holding 8 fused noise-free `raycast_room_rgbd` frames. The ray-cast is
timed at 1200x680 (replica intrinsics) and 640x480 (TUM) from the first frame's pose, float64 pose on the device: CUDA
events around `calls` back-to-back ray-casts, best of `repeats`. Beside each time: the fraction of pixels with a hit, and
the mean number of cells a ray visits, counted on the host from the output depth and the pose (the cells the ray's line
crosses from where it enters the grid to its hit, or to where it leaves the grid without one; a back face ends a ray
earlier, so misses are counted high). The card name and power limit are read in the same run; no device setting is
changed.

    python tools/bench_tsdf_raycast.py [--calls 20] [--warmup 5] [--repeats 3] [--out FILE]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import torch

from bench_tsdf import VOLUMES, card, frames, timed


def cells_per_ray(depth, w2c, K, origin, s, dims):
    """Mean number of cells the walk visits per ray that enters the grid: floor steps between entry and end per axis."""
    H, W = depth.shape
    fx, fy, cx, cy = (float(np.float32(k)) for k in K)
    P = np.asarray(w2c, np.float64)
    v, u = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    dc = np.stack([((u - cx) / fx).ravel(), ((v - cy) / fy).ravel(), np.ones(H * W)])
    o = -P[:3, :3].T @ P[:3, 3]
    d = P[:3, :3].T @ dc
    s = float(np.float32(s))
    g0 = (o - np.asarray(origin, np.float32).astype(np.float64)) / s
    dg = d / s
    hi = np.asarray(dims, np.float64)[:, None] - 1
    with np.errstate(divide="ignore", invalid="ignore"):
        ta, tb = -g0[:, None] / dg, (hi - g0[:, None]) / dg
    t_in = np.maximum(0.0, np.nanmax(np.fmin(ta, tb), axis=0))
    t_out = np.nanmin(np.fmax(ta, tb), axis=0)
    inside = t_in < t_out
    z = depth.ravel().astype(np.float64)
    t_end = np.where(z > 0, z, t_out)
    c_in = np.clip(np.floor(g0[:, None] + t_in * dg), 0, hi - 1)
    c_end = np.clip(np.floor(g0[:, None] + t_end * dg), 0, hi - 1)
    n = np.abs(c_end - c_in).sum(0) + 1
    return float(n[inside].mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tsdf_raycast needs a CUDA device")
    from rtg_slam_b200.reconstruct import TsdfVolume
    dev = torch.device("cuda", 0)
    name, limit = card()
    res = {"card": name, "power_limit": limit, "raycast": {}}
    fr = frames("replica", dev)
    views = {"1200x680": fr[0], "640x480": frames("tum", dev, n=1)[0]}
    for vname, (origin, s, dims, trunc) in VOLUMES.items():
        vol = TsdfVolume(origin, s, dims, trunc, color=True, device=dev)
        for d, c, w2c, K in fr:
            vol.integrate(d, w2c, K, color=c, color_channels_last=True)
        for label, (d, _, w2c, K) in views.items():
            H, W = d.shape
            ms = timed(lambda: vol.raycast(w2c, K, H, W), a.calls, a.warmup, a.repeats)
            out = vol.raycast(w2c, K, H, W)
            depth = out["depth"].cpu().numpy()
            res["raycast"][f"{vname} @ {label}"] = {
                "ms": round(ms, 4), "hit_fraction": round(float((depth > 0).mean()), 4),
                "cells_per_ray": round(cells_per_ray(depth, w2c.cpu().numpy(), K, origin, s, dims), 1)}
        del vol
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
