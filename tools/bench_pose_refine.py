"""Cost of pose refinement against a frozen map, on the benchmark scene (surfel room, 1 M Gaussians, SH degree 3) at
1200x680 and at a TUM-sized 640x480:

(a) the rasterizer backward of one forward whose only differentiated inputs are viewmatrix / projmatrix / campos, through
    the full camera backward (rtg_splat_backward_camera: every per-Gaussian gradient plus the zero fill, which autograd
    then discards) and through the pose-only backward (rtg_splat_backward_pose). The autograd graph is kept and the same
    forward is replayed; the two paths alternate call by call. Reported: the whole backward (CUDA events around
    torch.autograd.backward) and the per-Gaussian pass (`preprocess_bwd` of the library's event profiler), medians.
(b) the time per iteration of PoseRefiner.refine against the loop of test_camera_grad_gpu.test_pose_refinement_with_adam
    (a twist through torch.matrix_exp, torch.linalg.inv for campos, Renderer.render, an L1 colour + masked depth loss
    and torch.optim.Adam), which now takes the pose-only backward as well, and that loop with the camera backward it
    took before; all from 1 deg / 2 cm off the pose the targets were rendered at, host clock around a run that ends in a
    device synchronise.

The card name and power limit are read in the same run.

    python tools/bench_pose_refine.py [--gaussians N] [--calls K] [--iters I] [--out FILE]"""
import argparse
import contextlib
import ctypes as C
import json
import math
import os
import statistics
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from rtg_slam_b200 import _lib, scene
from rtg_slam_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer
from rtg_slam_b200.render import Renderer
from rtg_slam_b200.tracking import PoseRefiner
from tools.bench_camera_grad import card

ARGS = types.SimpleNamespace(renderer_opaque_threshold=0.6, renderer_normal_threshold=60, renderer_depth_threshold=1.0,
                             max_sh_degree=3, color_sigma=3.0, active_sh_degree=3)


class _Route:
    """The loaded library with rtg_splat_backward_pose answered by rtg_splat_backward_camera when `camera` is set (the path
    the same autograd call took before the pose-only backward existed)."""

    def __init__(self, L, outs):
        self.L, self.outs, self.camera = L, outs, False

    def __getattr__(self, name):
        if self.camera and name == "rtg_splat_backward_pose":
            o = self.outs
            return lambda *a: self.L.rtg_splat_backward_camera(*a[:19], a[20], *o, 0, a[21], a[22], a[23])
        return getattr(self.L, name)


def skew(w):
    z = torch.zeros((), dtype=w.dtype, device=w.device)
    return torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]), torch.stack([-w[1], w[0], z])])


def se3_exp(xi):
    m = torch.nn.functional.pad(skew(xi[3:]), (0, 1, 0, 1)) + torch.nn.functional.pad(xi[:3, None], (3, 0, 0, 1))
    return torch.matrix_exp(m)


def view_camera(cam, w2c):
    vm = w2c.transpose(0, 1)
    proj = torch.from_numpy(np.ascontiguousarray(cam.projection)).to(w2c.device)
    return types.SimpleNamespace(FoVx=2 * math.atan(cam.tanfovx), FoVy=2 * math.atan(cam.tanfovy), image_height=cam.height,
                                 image_width=cam.width, world_view_transform=vm, full_proj_transform=vm @ proj,
                                 projection_matrix=proj, camera_center=torch.linalg.inv(w2c)[:3, 3], cx=cam.cx, cy=cam.cy)


@contextlib.contextmanager
def routed(route, camera):
    """While active, the rasterizer shim calls `route` instead of the library; camera=True selects the camera backward."""
    real, route.camera = _lib.lib, camera
    _lib.lib = lambda: route
    try:
        yield
    finally:
        _lib.lib = real


def make_route(P, dev):
    f32 = dict(dtype=torch.float32, device=dev)
    outs = [torch.empty(n, **f32) for n in (3 * P, 48 * P)] + [None] + [torch.empty(n, **f32) for n in (P, 3 * P, 4 * P)] + [None, None]
    route = _Route(_lib.lib(), [None if o is None else C.c_void_p(o.data_ptr()) for o in outs])
    route.keep = outs
    return route


def backward_paths(cam, g, dev, route, calls, warmup):
    """(a): medians of (whole backward ms, preprocess_bwd ms) per path on one retained forward."""
    vm, pm, cp = (torch.from_numpy(x).to(dev).requires_grad_(True) for x in (cam.viewmatrix, cam.projmatrix, cam.campos))
    rs = GaussianRasterizationSettings(
        image_height=cam.height, image_width=cam.width, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=torch.zeros(3, device=dev),
        scale_modifier=1.0, viewmatrix=vm, projmatrix=pm, sh_degree=3, campos=cp, opaque_threshold=0.6,
        normal_threshold=float(np.cos(np.deg2rad(60.0))), depth_threshold=1.0, prefiltered=False, debug=False, cx=cam.cx, cy=cam.cy)
    out = GaussianRasterizer(rs)(means3D=g["xyz"], opacities=g["opacity"], shs=g["shs"], scales=g["scales"], rotations=g["rotations"])
    up = [torch.from_numpy(x).to(dev) for x in scene.upstream_grads(cam, seed=5)]
    ev = lambda: torch.cuda.Event(enable_timing=True)

    def one(camera):
        route.camera = camera
        torch.cuda.synchronize()
        _lib.profile_read(reset=True)
        s, e = ev(), ev()
        s.record()
        torch.autograd.backward([out[0], out[1]], up, retain_graph=True)
        e.record()
        torch.cuda.synchronize()
        prof = _lib.profile_read(reset=True)
        for k in ("viewmatrix", "projmatrix", "campos"):
            getattr(rs, k).grad = None
        pb, bz = prof["preprocess_bwd"], prof["bwd_zero"]
        return s.elapsed_time(e), pb[0] / max(1, pb[1]), bz[0] / max(1, bz[1])

    _lib.profile_enable(True)
    try:
        with routed(route, False):
            for _ in range(warmup):
                one(True), one(False)
            res = {True: [], False: []}
            for _ in range(calls):
                for camera in (True, False):
                    res[camera].append(one(camera))
    finally:
        _lib.profile_enable(False)
    med = lambda xs, i: statistics.median(x[i] for x in xs)
    return dict(backward_ms_camera=med(res[True], 0), backward_ms_pose=med(res[False], 0),
                preprocess_bwd_ms_camera=med(res[True], 1), preprocess_bwd_ms_pose=med(res[False], 1),
                bwd_zero_ms_camera=med(res[True], 2))


def refine_loops(cam, g, dev, route, iters, repeats):
    """(b): ms per iteration of PoseRefiner.refine and of the torch loop (through the pose-only backward, and through the
    camera backward it took before), best of `repeats` runs of `iters` iterations."""
    r = Renderer(ARGS)
    w2c_true = torch.eye(4, device=dev)
    with torch.no_grad():
        tgt = r.render(view_camera(cam, w2c_true), g)
        tgt_c, tgt_d = tgt["render"].clone(), tgt["depth"].clone()
    off = torch.tensor([0.012, -0.010, 0.012, 0.010, -0.012, 0.008], device=dev)
    w2c0 = se3_exp(off) @ w2c_true
    refiner = PoseRefiner(ARGS)

    def run_refiner(n):
        return refiner.refine(view_camera(cam, w2c0), g, tgt_c, tgt_d, iters=n, lr_rot=1e-3, lr_trans=1e-3, color_weight=1.0,
                              depth_weight=1.0)

    def run_torch(n):
        xi = torch.zeros(6, device=dev, requires_grad=True)
        opt = torch.optim.Adam([xi], lr=1e-3)
        valid = tgt_d > 0
        for _ in range(n):
            opt.zero_grad()
            out = r.render(view_camera(cam, se3_exp(xi) @ w2c0), g)
            loss = (out["render"] - tgt_c).abs().mean() + (out["depth"] - tgt_d).abs()[valid].mean()
            loss.backward()
            opt.step()
        return xi

    def timed(fn):
        best = float("inf")
        for _ in range(repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn(iters)
            torch.cuda.synchronize()
            best = min(best, (time.perf_counter() - t0) * 1e3 / iters)
        return best

    def run_torch_camera_path(n):
        with routed(route, True):
            run_torch(n)

    run_refiner(3), run_torch(3), run_torch_camera_path(3)  # first forward of the shape, module loads, allocator
    return dict(refine_ms_per_iter=timed(run_refiner), torch_loop_ms_per_iter=timed(run_torch),
                torch_loop_camera_backward_ms_per_iter=timed(run_torch_camera_path), iters=iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    g = {k: torch.from_numpy(v).to(dev) for k, v in scene.surfel_room(a.gaussians, seed=2024).items()}
    name, power = card()
    route = make_route(a.gaussians, dev)
    lines = []
    for cam_name in ("replica", "tum"):
        cam = scene.make_camera(cam_name)
        r = dict(gpu=name, power_limit=power, gaussians=a.gaussians, image=f"{cam.width}x{cam.height}", calls=a.calls)
        r.update(backward_paths(cam, g, dev, route, a.calls, a.warmup))
        r.update(refine_loops(cam, g, dev, route, a.iters, a.repeats))
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
