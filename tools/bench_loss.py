"""Device time of the fused frame losses at 1200x680, per call of the Python entry point (three kernel launches each):

    l1           l1_color_depth_loss(render, gt (3,H,W), depth)                    -> rtg_loss_l1
    l1_exposure  the same with exposure = (0.1, 0.02)                              -> rtg_loss_l1_exposure
    mapping      mapping_loss(normal_weight=0.1, a render mask over 60 % of pixels) -> rtg_loss_mapping

Inputs are random frames (seed 0): every pixel is read and written as in a real one, and the selection rules see a mix of
hit / missed, measured / unmeasured and near / far depth pixels. CUDA events around `calls` back-to-back calls after
`warmup` calls, best of `repeats`, the three modes alternating (host time included where the host is the slower side),
and the loss kernels' device time per call from torch.profiler. Each mode also reports a digest of its loss parts and one
of its gradients, so that two libraries can be checked to compute the same bits.

With --lib PATH (repeatable) each library runs in a subprocess of its own (RTG_SPLAT_LIB=PATH), `rounds` times in
alternation, and the per-round numbers of every library are printed side by side. The card name and power limit are
read in the same run. No device setting is changed.

    python tools/bench_loss.py [--calls 300] [--warmup 30] [--repeats 3] [--lib A.so --lib B.so [--rounds 3]]"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

H, W = 680, 1200


def frame(dev):
    g = torch.Generator(device=dev).manual_seed(0)
    rand = lambda *s: torch.rand(*s, device=dev, generator=g)
    depth = rand(1, H, W) * 3
    gt_depth = depth[0] + 0.1 * (rand(H, W) - 0.5)
    gt_depth[rand(H, W) < 0.1] = 0
    normal = torch.nn.functional.normalize(rand(3, H, W) - 0.5, dim=0)
    gt_normal = torch.nn.functional.normalize(rand(H, W, 3) - 0.5, dim=-1)
    gt_normal[rand(H, W) < 0.15] = 0
    out = {"render": rand(3, H, W).requires_grad_(True), "depth": depth.requires_grad_(True), "normal": normal.requires_grad_(True),
           "depth_index_map": torch.randint(-1, 100000, (1, H, W), device=dev, dtype=torch.int32, generator=g)}
    return out, {"color_map": rand(H, W, 3), "depth_map": gt_depth, "normal_map": gt_normal}, rand(H, W) < 0.6


def measure(calls, warmup, repeats):
    from rtg_slam_b200.loss import l1_color_depth_loss, mapping_loss
    dev = torch.device("cuda", 0)
    out, img, mask = frame(dev)
    gt_chw = img["color_map"].permute(2, 0, 1).contiguous()
    ab = torch.tensor([0.1, 0.02], device=dev, requires_grad=True)
    modes = {
        "l1": lambda: l1_color_depth_loss(out, gt_chw, img["depth_map"]),
        "l1_exposure": lambda: l1_color_depth_loss(out, gt_chw, img["depth_map"], exposure=ab),
        "mapping": lambda: mapping_loss(out, img, render_mask=mask, normal_weight=0.1),
    }
    res = {}
    for name, fn in modes.items():
        loss, parts = fn()
        grads = torch.autograd.grad(loss, [out["render"], out["depth"]] + ([out["normal"]] if name == "mapping" else []))
        digest = lambda ts: hashlib.sha1(b"".join(t.detach().cpu().numpy().tobytes() for t in ts)).hexdigest()[:16]
        res[name] = {"parts": [float(x) for x in parts.cpu()], "parts_digest": digest([parts]), "grad_digest": digest(grads)}
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = {name: float("inf") for name in modes}
    for _ in range(repeats):
        for name, fn in modes.items():
            a.record()
            for _ in range(calls):
                fn()
            b.record()
            b.synchronize()
            best[name] = min(best[name], a.elapsed_time(b) * 1e3 / calls)
    for name, fn in modes.items():
        # the events include the host's share when it is the slower side; the loss kernels' own device time, from
        # torch.profiler's CUDA activity
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(calls):
                fn()
            torch.cuda.synchronize()
        kern = {e.key.split("(")[0].replace("void rtg::", ""): e.device_time_total / calls for e in prof.key_averages() if "loss" in e.key}
        res[name].update(us_per_call=round(best[name], 2), kernel_us_per_call=round(sum(kern.values()), 2),
                         kernels={k: round(v, 2) for k, v in kern.items()})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--lib", action="append", default=[])
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not a.lib:
        print(json.dumps(measure(a.calls, a.warmup, a.repeats)))
        return
    from tools.bench_camera_grad import card
    name, power = card()
    print(f"{name}, power limit {power}, {H}x{W}, {a.calls} calls, best of {a.repeats}")
    args = [sys.executable, os.path.abspath(__file__), "--calls", str(a.calls), "--warmup", str(a.warmup), "--repeats", str(a.repeats)]
    for r in range(a.rounds):
        for lib in a.lib:
            env = dict(os.environ, RTG_SPLAT_LIB=os.path.abspath(lib))
            res = json.loads(subprocess.run(args, env=env, check=True, capture_output=True, text=True).stdout.strip().splitlines()[-1])
            row = "  ".join(f"{m} {v['us_per_call']:7.2f} us, kernels {v['kernel_us_per_call']:6.2f} us (parts {v['parts_digest']}, "
                            f"grads {v['grad_digest']})" for m, v in res.items())
            print(f"round {r} {os.path.basename(lib):>24}: {row}")
            print(" " * 34, "  ".join(f"{k} {v:.2f}" for m in res.values() for k, v in m["kernels"].items()))


if __name__ == "__main__":
    main()
