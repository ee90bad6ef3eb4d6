"""Device time and HBM rate of rtg_map_transform (mapsurgery.transform) on maps of P in {300 k, 1 M, 4 M} Gaussians with
degree-3 SH (features_rest (P,15,3)) and normals, K = 2000 anchor frames, and of one 128-row block:

    all      every anchor moved (a global alignment, or a loop closure that corrects the whole trajectory)
    10pct    a random 10 % of the anchors moved

Anchors are assigned as `_add_tick` assigns them: Gaussians are appended frame by frame, so row i belongs to frame
i * K // P and the moved rows come in runs. Bytes are computed from the shapes: every row reads its 4-byte anchor, a
moved row reads xyz, rotation, normal and features_rest (220 B) and writes them back; the per-anchor table is K * 672 B
(two poses in, 416 B out, read back per moved row from cache and not counted). CUDA events around `calls` back-to-back
calls of the C entry point (poses already on the device) after `warmup` calls, best of `repeats`. The wall time of one
Python `transform` call (host validation and pose upload included) is reported beside it. The card name and power limit
are read in the same run; no device setting is changed. P = 128 (one block of rows) measures the call's fixed part: the
memset, the per-anchor table kernel for all K anchors and the two launches.

    python tools/bench_map_transform.py [--calls 50] [--warmup 10] [--repeats 3] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

PEAK_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
K = 2000


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def poses(rng, frac_moved):
    from oracle import maptransform_oracle as mo
    old = np.stack([mo.random_pose(rng) for _ in range(K)])
    new = np.stack([mo.corrected_pose(rng, o, max_deg=5.0, max_trans=0.2) for o in old])
    keep = rng.uniform(size=K) >= frac_moved
    new[keep] = old[keep]
    return old, new, ~keep


def measure(P, frac_moved, calls, warmup, repeats):
    from rtg_slam_b200 import _lib, mapsurgery
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(P)
    g = torch.Generator(device=dev).manual_seed(P)
    params = {"xyz": torch.rand(P, 3, device=dev, generator=g) * 8 - 4, "rotation": torch.randn(P, 4, device=dev, generator=g),
              "normal": torch.nn.functional.normalize(torch.randn(P, 3, device=dev, generator=g), dim=1),
              "features_rest": torch.randn(P, 15, 3, device=dev, generator=g) * 0.1}
    anchor = (torch.arange(P, device=dev, dtype=torch.int64) * K // P).to(torch.int32)
    old, new, moved_k = poses(rng, frac_moved)
    moved_rows = int(moved_k[(np.arange(P, dtype=np.int64) * K // P)].sum())
    L = _lib.lib()
    dp = torch.from_numpy(np.stack([old, new])).to(dev)
    n_skipped = torch.empty(1, dtype=torch.int64, device=dev)
    ws = torch.empty(L.rtg_map_transform_workspace_bytes(K), dtype=torch.uint8, device=dev)
    xf = _lib.RtgMapTransform(P=P, K=K, sh_rest=15, _pad=0, anchor=anchor.data_ptr(), old_c2w=dp[0].data_ptr(),
                              new_c2w=dp[1].data_ptr(), xyz=params["xyz"].data_ptr(), rotation=params["rotation"].data_ptr(),
                              normal=params["normal"].data_ptr(), features_rest=params["features_rest"].data_ptr(),
                              n_skipped=n_skipped.data_ptr())
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    call = lambda: _lib.check(L.rtg_map_transform(C.byref(xf), C.c_void_p(ws.data_ptr()), stream), "rtg_map_transform")
    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(calls):
            call()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b) / calls)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mapsurgery.transform(params, anchor, old, new)
    torch.cuda.synchronize()
    py_ms = (time.perf_counter() - t0) * 1e3
    nbytes = P * 4 + moved_rows * 2 * (12 + 16 + 12 + 180) + K * (2 * 128 + 416)
    gbs = nbytes / (best * 1e-3) / 1e9
    return {"P": P, "moved": "all" if frac_moved >= 1 else "10pct", "moved_rows": moved_rows, "ms_per_call": round(best, 4),
            "bytes": nbytes, "GB_per_s": round(gbs, 1), "share_of_3.35TB_s": round(gbs * 1e9 / PEAK_BYTES_PER_S, 3),
            "python_call_ms": round(py_ms, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_map_transform needs a CUDA device")
    name, limit = card()
    rows = []
    for P in (128, 300_000, 1_000_000, 4_000_000):
        for frac in ((1.0,) if P == 128 else (1.0, 0.1)):
            r = measure(P, frac, args.calls, args.warmup, args.repeats)
            r.update(card=name, power_limit=limit)
            print(json.dumps(r), flush=True)
            rows.append(r)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
