"""Cost of the photometric term of the ICP tracker: IcpTracker.predict_pose against RgbdIcpTracker.predict_pose.

    python tools/bench_icp_rgbd.py [--calls N] [--warmup W]

Scene: the textured room (scene.raycast_room_rgbd, spheres included, 2 mm depth noise), frame 0 at the identity and
frame 1 at scene.small_pose(), at 640x480 (TUM intrinsics) and 1200x680 (Replica intrinsics); 3 levels x 5 iterations,
frame-to-frame (icp_use_model_depth=False, so a call is the solve and its read-back, no pyramid). Per size the two
trackers' predict_pose calls alternate, W untimed rounds then N timed ones; predict_pose ends in its own event wait, so a
host clock around it is a device-complete time. The intensity pyramid (build_intensity_pyramid) and, for scale, the depth
pyramid (build_pyramids) are timed separately between CUDA events. Medians are reported, with each tracker's pose error
against the ground truth. Convergence on a planar view (scene.wall_cameras at 640x480, 2 mm depth noise): each tracker's
in-plane error from a 2 cm / 1.5 cm, 1 degree start, and its drift over ten frames sliding 1 cm per frame along the wall,
frame-to-model with the ray-cast depth at each tracked pose as the render depth. Prints one JSON line with the card name,
power limit and max SM clock read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def tracker_args(use_model_depth=False):
    return types.SimpleNamespace(icp_downscales=[0.25, 0.5, 1.0], icp_warmup_frames=0, icp_use_model_depth=use_model_depth,
                                 icp_downscale_iters=[5, 5, 5], icp_distance_threshold=0.1, icp_normal_threshold=20,
                                 icp_damping=1e-4, verbose=False, icp_sample_distance_threshold=0.01,
                                 icp_sample_normal_threshold=0.01, icp_fail_threshold=0.02)


def wall_outcomes(dev):
    import numpy as np
    import torch

    from rtg_slam_b200 import icp, scene

    cam0, cam1, _ = scene.wall_cameras(640, 480)
    Kt = torch.from_numpy(cam0.K)
    Kf = (cam0.fx, cam0.fy, cam0.cx, cam0.cy)
    d0, c0 = scene.raycast_room_rgbd(cam0, spheres=(), noise_sigma=0.002, seed=3)
    d1, c1 = scene.raycast_room_rgbd(cam1, spheres=(), noise_sigma=0.002, seed=4)
    out = {"start": scene.wall_in_plane_error(cam0, cam1, np.eye(4))}
    for name, trk in (("IcpTracker", icp.IcpTracker(tracker_args())), ("RgbdIcpTracker", icp.RgbdIcpTracker(tracker_args()))):
        for k, (d, c) in enumerate(((d0, c0), (d1, c1))):
            col = (torch.from_numpy(c).to(dev),) if name == "RgbdIcpTracker" else ()
            trk.update_curr_status(torch.from_numpy(d).to(dev), Kt, *col)
            if k == 0:
                trk.move_last_status()
        pose, _ = trk.predict_pose({"K": Kt, "frame_id": 1})
        out[name] = scene.wall_in_plane_error(cam0, cam1, pose)
    gts = [scene.wall_cameras(640, 480, dx=0.01 * k, dy=0.0, deg=0.0)[1] for k in range(10)]
    frames = [scene.raycast_room_rgbd(c, spheres=(), noise_sigma=0.002, seed=100 + k) for k, c in enumerate(gts)]
    drift = {}
    for name, trk in (("IcpTracker", icp.IcpTracker(tracker_args(True))), ("RgbdIcpTracker", icp.RgbdIcpTracker(tracker_args(True)))):
        c2w = cam0.c2w.copy()
        for k, (d, c) in enumerate(frames):
            td = torch.from_numpy(d).to(dev)
            col = (torch.from_numpy(c).to(dev),) if name == "RgbdIcpTracker" else ()
            trk.update_curr_status(td, Kt, *col)
            if k > 0:
                c2w = c2w @ trk.predict_pose({"K": Kt, "frame_id": k})[0].astype(np.float64)
            trk.move_last_status()
            cam_t = scene.Camera(cam0.width, cam0.height, cam0.fx, cam0.fy, cam0.cx, cam0.cy, c2w=c2w)
            tm = torch.from_numpy(scene.raycast_room_depth(cam_t, spheres=())).to(dev)
            _, rn = icp.build_pyramids(tm, Kf, 1)
            trk.update_last_status(None, tm[..., None].contiguous().clone(), td[..., None], rn[0], trk.normal_pyramid_t1[-1])
        drift[name] = float(np.linalg.norm(c2w[:3, 3] - gts[-1].c2w[:3, 3]))
    out["drift_10_frames_m"] = drift
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    import numpy as np
    import torch

    from rtg_slam_b200 import icp, scene

    if not torch.cuda.is_available():
        raise SystemExit("bench_icp_rgbd needs a CUDA device")
    dev = torch.device("cuda", 0)
    result = {"card": card(), "calls": a.calls, "warmup": a.warmup, "sizes": {}}
    for camname in ("tum", "replica"):
        cam0 = scene.make_camera(camname)
        gt = scene.small_pose()
        cam1 = scene.make_camera(camname, c2w=gt)
        d0, c0 = scene.raycast_room_rgbd(cam0, noise_sigma=0.002, seed=3)
        d1, c1 = scene.raycast_room_rgbd(cam1, noise_sigma=0.002, seed=4)
        Kt = torch.from_numpy(cam0.K)
        td0, td1 = torch.from_numpy(d0).to(dev), torch.from_numpy(d1).to(dev)
        tc0, tc1 = torch.from_numpy(c0).to(dev), torch.from_numpy(c1).to(dev)
        geo, rgbd = icp.IcpTracker(tracker_args()), icp.RgbdIcpTracker(tracker_args())
        geo.update_curr_status(td0, Kt)
        geo.move_last_status()
        geo.update_curr_status(td1, Kt)
        rgbd.update_curr_status(td0, Kt, tc0)
        rgbd.move_last_status()
        rgbd.update_curr_status(td1, Kt, tc1)
        frame = {"K": Kt, "frame_id": 1}
        times = {"IcpTracker": [], "RgbdIcpTracker": []}
        poses = {}
        for i in range(a.warmup + a.calls):
            for name, trk in (("IcpTracker", geo), ("RgbdIcpTracker", rgbd)):
                t = time.perf_counter()
                pose, _ = trk.predict_pose(frame)
                dt = time.perf_counter() - t
                if i >= a.warmup:
                    times[name].append(dt * 1e3)
                poses[name] = pose
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        t_int, t_dep = [], []
        for i in range(a.warmup + a.calls):
            ev[0].record()
            icp.build_intensity_pyramid(tc1, 3)
            ev[1].record()
            icp.build_pyramids(td1, (cam0.fx, cam0.fy, cam0.cx, cam0.cy), 3)
            ev[2].record()
            ev[2].synchronize()
            if i >= a.warmup:
                t_int.append(ev[0].elapsed_time(ev[1]))
                t_dep.append(ev[1].elapsed_time(ev[2]))
        med = {k: statistics.median(v) for k, v in times.items()}
        result["sizes"][f"{cam0.width}x{cam0.height}"] = {
            "predict_pose_ms": {k: round(v, 4) for k, v in med.items()},
            "added_ms": round(med["RgbdIcpTracker"] - med["IcpTracker"], 4),
            "intensity_pyramid_ms": round(statistics.median(t_int), 4),
            "depth_pyramid_ms": round(statistics.median(t_dep), 4),
            "pose_error_vs_gt": {k: float(np.linalg.norm(p.astype(np.float64) - gt)) for k, p in poses.items()},
            "photometric_ratio": rgbd.last_photometric_ratio, "photometric_rmse": rgbd.last_photometric_rmse,
            "valid_ratio": {"IcpTracker": geo.last_valid_ratio, "RgbdIcpTracker": rgbd.last_valid_ratio},
        }
    result["planar_wall_640x480"] = wall_outcomes(dev)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
