"""Device time of TSDF fusion (rtg_tsdf_integrate) and marching-tetrahedra extraction (rtg_tsdf_extract_count + emit).

Volumes: 301x151x301 voxels at 2 cm over the benchmark room (6 x 3 x 6 m, 13.7 M voxels) and 512^3 voxels at 1.25 cm over
a 6.4 m cube around it (134 M voxels), both with colour. Frames: noise-free `raycast_room_rgbd` views at 1200x680
(replica intrinsics) and 640x480 (TUM), float64 poses on the device, colour channels-last as the dataset loaders give
it. Integration is timed per frame with CUDA events around `calls` back-to-back integrations of one frame into a
volume that already holds 8 frames (so that the running mean is read), best of `repeats`. Extraction is timed after
those 8 fused frames: the count pass with its scans, the host read-back of the two sizes, and the emit pass, as
`TsdfVolume.extract_mesh` runs them; the vertex and triangle counts are reported beside the time. The card name and
power limit are read in the same run; no device setting is changed.

    python tools/bench_tsdf.py [--calls 20] [--warmup 5] [--repeats 3] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

VOLUMES = {"301x151x301": ((-3.0, -1.5, -3.0), 0.02, (301, 151, 301), 0.08),
           "512^3": ((-3.2, -3.2, -3.2), 0.0125, (512, 512, 512), 0.05)}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def frames(cam_name, dev, n=8):
    from rtg_slam_b200 import scene
    out = []
    for k in range(n):
        a = 360.0 * k / n
        cam = scene.make_camera(cam_name, c2w=scene.small_pose((3.0, a, -2.0), (0.3 * np.cos(k), 0.1, 0.3 * np.sin(k))))
        depth, color = scene.raycast_room_rgbd(cam)
        out.append((torch.from_numpy(depth).to(dev), torch.from_numpy(color).to(dev),
                    torch.from_numpy(cam.w2c).to(dev), (cam.fx, cam.fy, cam.cx, cam.cy)))
    return out


def timed(fn, calls, warmup, repeats):
    for _ in range(warmup):
        fn()
    best = float("inf")
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(calls):
            fn()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b) / calls)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tsdf needs a CUDA device")
    from rtg_slam_b200.reconstruct import TsdfVolume
    dev = torch.device("cuda", 0)
    name, limit = card()
    res = {"card": name, "power_limit": limit, "integrate_ms": {}, "extract": {}}
    for cam_name, label in (("replica", "1200x680"), ("tum", "640x480")):
        fr = frames(cam_name, dev)
        for vname, (origin, s, dims, trunc) in VOLUMES.items():
            vol = TsdfVolume(origin, s, dims, trunc, color=True, device=dev)
            for d, c, w2c, K in fr:
                vol.integrate(d, w2c, K, color=c, color_channels_last=True)
            d, c, w2c, K = fr[0]
            ms = timed(lambda: vol.integrate(d, w2c, K, color=c, color_channels_last=True), a.calls, a.warmup, a.repeats)
            res["integrate_ms"][f"{vname} @ {label}"] = round(ms, 4)
            if label == "1200x680":
                vol = TsdfVolume(origin, s, dims, trunc, color=True, device=dev)
                for d, c, w2c, K in fr:
                    vol.integrate(d, w2c, K, color=c, color_channels_last=True)
                mesh = vol.extract_mesh()
                ms = timed(vol.extract_mesh, max(1, a.calls // 4), 2, a.repeats)
                res["extract"][vname] = {"ms": round(ms, 3), "vertices": int(mesh["vertices"].shape[0]),
                                         "triangles": int(mesh["faces"].shape[0])}
            del vol
            torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
