"""GPU tests of the rasterizer backward held to the float64 oracle Gaussian by Gaussian (gradcheck.py), with the depth-hit
path tested on its own and on every surfel axis. All through the public GaussianRasterizer.

Each comparison: the GPU forward and the two oracle forwards give the decision mask (pixels within 1e-3 of a threshold
or whose hit indices differ), the upstream gradients are zeroed there, and every visible row i of every gradient tensor
must satisfy  max_j |g_ij - ref_ij| <= RTOL * n_i + C * max_i n_i  with n_i = max_j |ref_ij|, RTOL = 1e-3, C = 5e-6.
C = 1e-6 holds every row of the float32 oracle but two (an opacity row and a two-pixel rotation row whose terms cancel, at
1.1 x the bound); 5e-6 is half the largest value at which the absolute term still means anything. For the gradients behind
the 2-D covariance RTOL grows with the squared condition number of that covariance past 30
(gradcheck.covariance_condition: a needle seen along its length, ragged blob 293 at kappa = 54, is 8e-4 off in the float32
oracle and 1.2e-3 off here). The bound widens to 10 x the library's own run-to-run row difference (the float atomics of the
compositing backward) where that is larger; it never did. `ratio` in the output is the left side over the right side.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit (worst ratio / worst run-to-run jitter in the same units, over
every scene x inputs x loss and every backward mode below): dmeans3D 0.18 / 0.004, dshs 0.06 / 0.001, dcolors_precomp
0.06 / 0.000, dopacities 0.48 / 0.002, dscales 0.38 / 0.034, drotations 0.23 / 0.068, dcov3D_precomp 0.09 / 0.040.
Depth-only loss on axis_room by (thin axis, branch), dmeans3D / drotations worst ratio: axis 0 plane (492 pixels, 136
Gaussians) 0.004 / 0.172, axis 0 centre (215, 70) 0.001 / 0.009, axis 1 plane (453, 107) 0.002 / 0.070, axis 1 centre
(157, 71) 0.000 / 0.020, axis 2 plane (357, 107) 0.003 / 0.143, axis 2 centre (131, 68) 0.002 / 0.046. 300 000 surfels at
1200x680 (RTOL 5e-3, see the test): dmeans3D 0.65, dshs 0.07, dopacities 0.34, dscales 0.31, drotations 0.26, jitter <=
0.006. Masked pixels: small 10 of 17 920, ragged 37 of 7 500, masked 14 of 17 920, axis_room 28 of 17 920, dense 713 of
3 072, 300 k 20 028 of 816 000; the GPU forward's index maps added none to the oracles' masks. Rows left out: 0 everywhere but
dense (2 colour clamps, 1 scale tie of 30 000) and 300 k (1 colour clamp of 116 902)."""
import functools

import numpy as np
import pytest
import torch

import gradcheck as gck
import helpers
from rtg_slam_b200 import scene
from test_camera_grad_gpu import KW, NAMES, inputs_for
from test_transmittance_grad_cpu import oracle_grads, t_weights
from test_transmittance_grad_gpu import run

pytestmark = pytest.mark.gpu

SCENES = ("small", "ragged", "masked", "dense", "axis_room")   # `dense`: tile lists past the on-chip sort capacity
MODES = ("sh", "colors_precomp", "cov3D_precomp", "M4")


@pytest.fixture(scope="module", autouse=True)
def own_capacity_checks(cuda_device):
    """Every forward here waits for its own instance count, as in test_transmittance_grad_gpu.py."""
    from rtg_slam_b200 import rasterizer
    prev = rasterizer._state(cuda_device).mode
    rasterizer.set_capacity_checks("sync", cuda_device)
    yield
    rasterizer.set_capacity_checks(prev, cuda_device)


def gpu_forward(cam, inputs, dev, mask=None, **over):
    from rtg_slam_b200.rasterizer import GaussianRasterizer
    rs = helpers.make_settings(cam, dev, **over)
    t = {KW[k]: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in inputs.items()}
    tm = None if mask is None else torch.from_numpy(np.ascontiguousarray(mask, dtype=np.int32)).to(dev)
    with torch.no_grad():
        out = GaussianRasterizer(rs)(**t, tile_mask=tm)
    return dict(zip(NAMES, [o.cpu().numpy() for o in out]))


@functools.lru_cache(maxsize=None)
def oracle_side(name, mode, over_items=()):
    """Scene, inputs and both oracle forwards (the GPU forward is added per test: it needs the device)."""
    cam, g, mask = gck.scene_case(name)
    inputs, over = inputs_for(g, mode)
    over = dict(over, **dict(over_items))
    g, kw = gck.oracle_args(inputs, mask, over)
    return cam, inputs, mask, over, g, kw, gck.forwards(cam, g, kw)


def prepare(name, mode, dev, **extra):
    cam, inputs, mask, over, g, kw, (o32, o64) = oracle_side(name, mode, tuple(sorted(extra.items())))
    fwd = gpu_forward(cam, inputs, dev, mask, **over)
    dm = gck.decision_mask(cam, g, kw, gpu_forward=fwd, oracles=(o32, o64))
    assert dm.mean() <= gck.MAX_MASKED_SHARE.get(name, 0.01), (name, int(dm.sum()), dm.size)
    rows, excluded = gck.comparable_rows(cam, g, kw, o32, o64, gpu_radii=fwd["radii"])
    print(f"{name}/{mode}: {int(dm.sum())} of {dm.size} pixels masked, {int(rows.sum())} rows compared, left out {excluded}")
    return cam, inputs, mask, over, g, kw, o64, dm, rows


def none_if_zero(up):
    return tuple(None if (u is None or not np.any(u)) else u for u in up)


def reference(o64, up):
    gr = o64.backward(up[0], up[1])
    return {k: v for k, v in gr.items() if k not in ("means2D", "conic", "colors", "cov3D")}


def assert_depth_only_zeros(grads, o64, dm):
    """Depth-only loss: the depth reaches dL/dmeans3D and dL/drotations of the hit Gaussians and no other visible row
    (under visible_rows_only the culled rows are left unwritten)."""
    hit, vis = gck.hit_rows(o64, dm), o64.radii > 0
    for k, v in grads.items():
        zero = vis & (~hit if k in ("means3D", "rotations") else np.ones_like(hit))
        assert np.all(v[zero] == 0), f"d{k} must be exactly zero outside the depth-hit rows"


@pytest.mark.parametrize("loss", gck.LOSSES)
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", SCENES)
def test_rows_match_f64_oracle(cuda_device, name, mode, loss):
    cam, inputs, mask, over, g, kw, o64, dm, rows = prepare(name, mode, cuda_device)
    up = gck.upstream(cam, loss, dm)
    a = run(cam, inputs, cuda_device, none_if_zero(up + (None,)), mask, **over)["grads"]
    b = run(cam, inputs, cuda_device, none_if_zero(up + (None,)), mask, **over)["grads"]
    ref = reference(o64, up)
    assert set(a) == set(ref)
    gck.check_rows(f"{name}/{mode}/{loss}", a, ref, rows, o64, g, again=b)
    assert all(np.all(v[o64.radii == 0] == 0) for v in a.values())
    if loss == "depth":
        assert_depth_only_zeros(a, o64, dm)


def test_depth_path_per_axis(cuda_device):
    """Depth-only loss on axis_room: the rows of each (thin axis, plane / centre-depth) cell bounded on their own."""
    cam, inputs, mask, over, g, kw, o64, dm, rows = prepare("axis_room", "sh", cuda_device)
    cells = gck.depth_coverage(o64, g, dm)
    gck.assert_coverage(cells)
    up = gck.upstream(cam, "depth", dm)
    a = run(cam, inputs, cuda_device, (None, up[1], None), mask, **over)["grads"]
    b = run(cam, inputs, cuda_device, (None, up[1], None), mask, **over)["grads"]
    ref = reference(o64, up)
    assert_depth_only_zeros(a, o64, dm)
    for (axis, branch), (n, ids) in sorted(cells.items()):
        subset = np.zeros(len(rows), bool)
        subset[ids] = True
        only = {k: a[k] for k in ("means3D", "rotations")}
        rep = gck.check_rows(f"axis {axis} {branch} ({n} pixels, {len(ids)} Gaussians)", only, ref, rows, o64, g,
                             again=b, subset=subset)
        assert np.abs(ref["means3D"][ids]).max() > 0   # the cell's rows do carry a gradient
        assert (np.abs(ref["rotations"][ids]).max() > 0) == (branch == "plane") or branch == "centre"


MODE_CASES = {
    "visible_rows_only": ("small", {}),
    "background": ("masked", {"bg": (0.3, 0.55, 0.8)}),
    "modifier_axis_room": ("axis_room", {"scale_modifier": 1.7}),
    "record_exchange_identity": ("ragged", {}),
}


@pytest.mark.parametrize("loss", ["mixed", "depth"])
@pytest.mark.parametrize("case", sorted(MODE_CASES))
def test_rows_in_the_other_backward_modes(cuda_device, case, loss):
    """The same rows through the backward modes that share the kernels: the visible-rows finish pass, a background colour
    (the transmittance term), a scale modifier (the forward tests the plane with it, the backward without it, as the
    reference does and the oracle restates), and the two-phase render / finish backward of the record exchange."""
    from rtg_slam_b200.rasterizer import set_grad_record_hook, visible_rows_only
    name, extra = MODE_CASES[case]
    cam, inputs, mask, over, g, kw, o64, dm, rows = prepare(name, "sh", cuda_device, **extra)
    up = gck.upstream(cam, loss, dm)
    prev = set_grad_record_hook((lambda rec: None) if case == "record_exchange_identity" else None)
    try:
        with visible_rows_only(case == "visible_rows_only"):
            a = run(cam, inputs, cuda_device, none_if_zero(up + (None,)), mask, **over)["grads"]
            b = run(cam, inputs, cuda_device, none_if_zero(up + (None,)), mask, **over)["grads"]
    finally:
        set_grad_record_hook(prev)
    gck.check_rows(f"{case}/{loss}", a, reference(o64, up), rows, o64, g, again=b)
    if loss == "depth":
        assert_depth_only_zeros(a, o64, dm)


@pytest.mark.parametrize("name", ["small", "axis_room"])
def test_rows_with_a_transmittance_loss(cuda_device, name):
    """Colour + depth + T_map loss; the reference gradient is test_transmittance_grad_cpu.oracle_grads."""
    cam, inputs, mask, over, g, kw, o64, dm, rows = prepare(name, "sh", cuda_device)
    gc, gd = gck.upstream(cam, "mixed", dm)
    gT = (t_weights(cam, seed=6) * ~dm[None]).astype(np.float32)
    a = run(cam, inputs, cuda_device, (gc, gd, gT), mask, **over)["grads"]
    b = run(cam, inputs, cuda_device, (gc, gd, gT), mask, **over)["grads"]
    g64 = {k: (None if v is None else v.astype(np.float64)) for k, v in g.items()}
    ref, _ = oracle_grads(cam, g64, kw, tuple(x.astype(np.float64) for x in (gc, gd, gT)), camera=False)
    gck.check_rows(f"{name}/T_map", a, {k: ref[k] for k in a}, rows, o64, g, again=b)


def test_rows_of_a_tile_sharded_frame_after_record_exchange(cuda_device):
    """Three tile shards, their gradient records summed and handed to one shard's finish pass (TileShard.exchange_records
    emulated on one GPU as in test_raster_gpu.test_two_phase_backward_with_record_exchange): the rows of the full frame."""
    from rtg_slam_b200 import rasterizer
    from rtg_slam_b200.parallel import TileShard
    cam, inputs, mask, over, g, kw, o64, dm, rows = prepare("axis_room", "sh", cuda_device)
    up = gck.upstream(cam, "mixed", dm)
    shards = [TileShard(cam.height, cam.width, 3, r) for r in range(3)]
    captured = []
    prev = rasterizer.set_grad_record_hook(lambda rec: captured.append(rec.clone()))
    try:
        for sh in shards:
            run(cam, inputs, cuda_device, up + (None,), sh.mask.numpy(), **over)
        assert len(captured) == 3
        total = sum(captured)
        rasterizer.set_grad_record_hook(lambda rec: rec.copy_(total))
        a = run(cam, inputs, cuda_device, up + (None,), shards[1].mask.numpy(), **over)["grads"]
    finally:
        rasterizer.set_grad_record_hook(prev)
    gck.check_rows("tile shards, world 3", a, reference(o64, up), rows, o64, g)


TIMED_RTOL = 5e-3


def test_rows_at_a_timed_size(cuda_device):
    """300 000 surfels at 1200x680 (the live Replica case of test_raster_gpu.test_matches_live_reference_cuda; the float64
    oracle takes seconds on the host): realistic per-Gaussian pixel counts and atomic contention. RTOL is 5e-3 here: most
    surfels project below the 0.3 px^2 dilation of the 2-D covariance, and the dL/dmean of such a splat is a sum over a
    20-40 pixel footprint of terms that change sign across it. The float32 oracle, which has no atomics, is already 3e-3
    away from the float64 one on such rows (0.65 of this bound at worst); a sign, a missing pixel or a 1 % error still fails."""
    from golden import make_reference_cuda_golden as refgold
    cam, g0, mask, _ = refgold.live_inputs("replica", 300_000, None)
    inputs, over = inputs_for(g0, "sh")
    g, kw = gck.oracle_args(inputs, mask, over)
    o32, o64 = gck.forwards(cam, g, kw)
    fwd = gpu_forward(cam, inputs, cuda_device, mask)
    dm = gck.decision_mask(cam, g, kw, gpu_forward=fwd, oracles=(o32, o64))
    assert dm.mean() <= 0.04, (int(dm.sum()), dm.size)
    rows, excluded = gck.comparable_rows(cam, g, kw, o32, o64, gpu_radii=fwd["radii"])
    print(f"live replica 300k: {int(dm.sum())} of {dm.size} pixels masked, {int(rows.sum())} rows compared, left out {excluded}")
    up = gck.upstream(cam, "mixed", dm)
    a = run(cam, inputs, cuda_device, up + (None,), mask)["grads"]
    b = run(cam, inputs, cuda_device, up + (None,), mask)["grads"]
    gck.check_rows("live replica 300k", a, reference(o64, up), rows, o64, g, again=b, rtol=TIMED_RTOL)
