"""Operator API of the reference rasterizer, backed by librtg_splat_b200.so.

Mirrors `diff_gaussian_rasterization_depth/__init__.py` of the reference (RAST/...:29-372): same
`GaussianRasterizationSettings` fields and defaults, same `GaussianRasterizer.forward` signature and
exactly-one-of checks, same 8-tuple of outputs, same gradient tuple. What is different underneath:

* the native side is a C ABI called through ctypes with raw pointers and the current stream;
* no blocking read-backs on the steady path: the instance count stays on the device. The binning buffer is
  sized from earlier calls (1.5x the largest instance count seen); the scan kernel drops the counters into
  pinned host memory. The first call of a (P, H, W) shape waits for that kernel (the rest of the forward keeps
  running) and re-runs the forward with a larger buffer on overflow; later calls do not wait at all -- their
  counters are read when they have arrived (at the next call, and at the latest at the call's own backward), and
  an overflow, which left that frame empty, raises instead of passing silently (`set_capacity_checks`);
* outputs and gradients are `torch.empty` -- the kernels write every element (the reference fills 9
  tensors with `torch::full` / `zeros` first).
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple

import torch
import torch.nn as nn

from . import _lib
from ._lib import RtgSplatView, check


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    opaque_threshold: float
    normal_threshold: float
    depth_threshold: float
    prefiltered: bool
    debug: bool
    cx: float
    cy: float
    color_sigma: float = 3.0
    T_threshold: float = 0.0001


class CapacityOverflow(RuntimeError):
    """A forward needed more (Gaussian, tile) instances than its binning buffer held and rendered that frame empty. The
    capacity has been raised by the time this is raised: rendering the frame again succeeds."""


# ----------------------------------------------------------------------------- per-device state
class _Pending:
    """Counters of one forward call that have not been read yet: pinned buffer + the event recorded after the scan kernel."""
    __slots__ = ("pinned", "event", "r_cap", "done", "num_rendered", "overflow")

    def __init__(self, pinned, event, r_cap):
        self.pinned, self.event, self.r_cap = pinned, event, r_cap
        self.done, self.num_rendered, self.overflow = False, 0, False


class _DeviceState:
    """Capacity hint for the binning buffer, pinned counters, gradient scratch; one per CUDA device."""

    def __init__(self, device):
        self.device = device
        self.r_hint = 1 << 16
        self.scratch = None  # (P*16,) zeros, cleared by the backward kernel itself
        self.ones_masks = {}
        self.free = []      # free list of (pinned tensor, event): only buffers whose event has completed
        self.pending = []   # _Pending of calls whose counters have not been read yet, oldest first
        self.mode = "auto"  # "sync" | "auto" | "deferred"
        self.seen = set()   # (P, H, W) shapes whose capacity has been measured by a waiting call
        self.last = (0, 0, 0, 0)  # counters of the most recent call that has been read

    def get_pinned(self):
        if self.free:
            return self.free.pop()
        t = torch.zeros(_lib.RTG_CNT_WORDS, dtype=torch.int32).pin_memory()
        ev = torch.cuda.Event()
        with torch.cuda.device(self.device):
            ev.record()  # torch creates the cudaEvent_t lazily, at the first record(); the library needs the handle
        if not ev.cuda_event:
            raise RuntimeError("could not create a CUDA event for the capacity check")
        return t, ev

    def read(self, p: _Pending, block: bool) -> bool:
        """Reads the counters of call `p` if its scan kernel has finished (or waits for it). True if read."""
        if p.done:
            return True
        if block:
            p.event.synchronize()
        elif not p.event.query():
            return False
        p.num_rendered, p.overflow = int(p.pinned[0]), bool(int(p.pinned[2]))
        self.last = tuple(int(x) for x in p.pinned[:4])
        p.done = True
        # entries the buffer must hold: the instances with every tile's bucket padded to a 16-byte boundary (counters[4]);
        # 1.5x head room: the steady path does not wait for the count of the current frame
        self.r_hint = max(self.r_hint, int(max(p.num_rendered, int(p.pinned[4])) * 1.5) + 4096)
        self.free.append((p.pinned, p.event))  # the event has completed: the buffer may be reused
        p.pinned = p.event = None
        if p in self.pending:
            self.pending.remove(p)
        return True

    def reap(self, block: bool = False):
        """Reads every outstanding call's counters that has arrived; raises if one of them overflowed unnoticed."""
        bad = None
        for p in list(self.pending):
            if self.read(p, block) and p.overflow:
                bad = p
        if bad is not None:
            raise CapacityOverflow(
                f"rasterizer: an earlier forward needed {bad.num_rendered} (Gaussian, tile) instances but its binning buffer "
                f"held {bad.r_cap}; that frame was rendered empty. The capacity has been raised -- render the frame again, "
                "or call set_capacity_checks('sync') to have every forward wait for its own count.")

    def get_scratch(self, P):
        n = P * 16
        if self.scratch is None or self.scratch.numel() < n:
            self.scratch = torch.zeros(max(n, 1024), dtype=torch.float32, device=self.device)
        return self.scratch

    def ones_mask(self, th, tw):
        key = (th, tw)
        if key not in self.ones_masks:
            self.ones_masks[key] = torch.ones((th, tw), dtype=torch.int32, device=self.device)
        return self.ones_masks[key]


_STATES = {}


def _state(device) -> _DeviceState:
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _STATES:
        _STATES[idx] = _DeviceState(torch.device("cuda", idx))
    return _STATES[idx]


def set_capacity_checks(mode: str, device=None) -> None:
    """How a forward learns whether its binning buffer was large enough (the instance count is only known on the device):
    'sync'     every forward waits for its scan kernel (not for the rest of the forward) and re-runs on overflow;
    'auto'     (default) the first forward of a (P, H, W) shape does that; later ones do not wait -- the buffer holds 1.5x
               the largest count seen, their counters are read once they have arrived, and an overflow (which leaves that
               frame empty) raises CapacityOverflow (a RuntimeError) at the next rasterizer call or at the frame's own backward;
    'deferred' like 'auto' without the waiting first call."""
    if mode not in ("sync", "auto", "deferred"):
        raise ValueError("mode must be 'sync', 'auto' or 'deferred'")
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    _state(dev).mode = mode


def set_async_capacity_checks(enabled: bool, device=None) -> None:
    """Round-1 name: True = 'sync' (wait for the scan kernel in every forward), False = 'deferred'."""
    set_capacity_checks("sync" if enabled else "deferred", device)


def last_counters(device=None):
    """(num_rendered, active tiles, overflow, longest tile list) of the most recent forward on `device` (waits for it)."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    st = _state(dev)
    st.reap(block=True)
    return st.last


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _opt(t):
    """Empty tensor encodes 'not provided' (reference: torch.Tensor([]) -> nullptr)."""
    return None if (t is None or t.numel() == 0) else t


def _f32_cuda(t, name, device):
    if t is None:
        return None
    if not t.is_cuda or t.dtype != torch.float32:
        raise TypeError(f"{name} must be a CUDA float32 tensor (got {t.dtype} on {t.device})")
    if t.device != device:
        raise ValueError(f"{name} is on {t.device}, expected {device}")
    t = t.contiguous()
    # the kernels read rotations and 16-coefficient SH rows with 128-bit loads; a view at an offset into its storage may
    # be contiguous and still misaligned
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _make_view(rs: GaussianRasterizationSettings, device, antialiased: bool = False) -> tuple[RtgSplatView, tuple]:
    keep = tuple(_f32_cuda(x, n, device) for x, n in ((rs.viewmatrix, "viewmatrix"), (rs.projmatrix, "projmatrix"),
                                                      (rs.campos, "campos"), (rs.bg, "bg")))
    v = RtgSplatView()
    v.image_height, v.image_width = int(rs.image_height), int(rs.image_width)
    v.tanfovx, v.tanfovy = float(rs.tanfovx), float(rs.tanfovy)
    v.cx, v.cy = float(rs.cx), float(rs.cy)
    v.scale_modifier, v.color_sigma = float(rs.scale_modifier), float(rs.color_sigma)
    v.opaque_threshold, v.depth_threshold = float(rs.opaque_threshold), float(rs.depth_threshold)
    v.normal_threshold, v.T_threshold = float(rs.normal_threshold), float(rs.T_threshold)
    v.sh_degree = int(rs.sh_degree)
    v.prefiltered = ((_lib.RTG_VIEW_PREFILTERED if rs.prefiltered else 0) |
                     (_lib.RTG_VIEW_ANTIALIASED if antialiased else 0))
    v.viewmatrix, v.projmatrix, v.campos, v.bg = (k.data_ptr() for k in keep)
    return v, keep


class _Saved:
    """State kept between forward and backward (the reference keeps geomBuffer / binningBuffer / imgBuffer)."""
    __slots__ = ("ws", "geom", "img", "bin", "r_cap", "counters", "view_keep", "pending", "antialiased")


def _forward_native(rs, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, tile_mask):
    L = _lib.lib()
    device = means3D.device
    if means3D.dim() != 2 or means3D.size(1) != 3:
        raise ValueError("means3D must have dimensions (num_points, 3)")  # rasterize_points.cu:67-70
    st = _state(device)
    P = means3D.size(0)
    H, W = int(rs.image_height), int(rs.image_width)
    th, tw = (H + 15) // 16, (W + 15) // 16
    means3D = _f32_cuda(means3D, "means3D", device)
    sh = _f32_cuda(_opt(sh), "shs", device)
    colors_precomp = _f32_cuda(_opt(colors_precomp), "colors_precomp", device)
    opacities = _f32_cuda(opacities, "opacities", device)
    scales = _f32_cuda(_opt(scales), "scales", device)
    rotations = _f32_cuda(_opt(rotations), "rotations", device)
    cov3Ds_precomp = _f32_cuda(_opt(cov3Ds_precomp), "cov3D_precomp", device)
    if tile_mask is None:
        tile_mask = st.ones_mask(th, tw)
    if not tile_mask.is_cuda or tile_mask.dtype != torch.int32:
        raise TypeError("tile_mask must be a CUDA int32 tensor")
    tile_mask = tile_mask.contiguous()
    if tile_mask.numel() != th * tw:
        raise ValueError(f"tile_mask must have {th}x{tw} entries")
    M = sh.size(1) if sh is not None else 0
    if sh is not None and (int(rs.sh_degree) + 1) ** 2 > M:
        raise ValueError(f"sh_degree {int(rs.sh_degree)} needs {(int(rs.sh_degree) + 1) ** 2} SH coefficients per Gaussian, shs has {M}")
    antialiased = _ANTIALIASED[0]
    view, keep = _make_view(rs, device, antialiased)
    stream = torch.cuda.current_stream(device).cuda_stream  # fetched per call: autograd runs backward on its own thread

    f32 = dict(dtype=torch.float32, device=device)
    i32 = dict(dtype=torch.int32, device=device)
    color = torch.empty((3, H, W), **f32)
    depth = torch.empty((1, H, W), **f32)
    hit_color = torch.empty((1, H, W), **i32)
    hit_depth = torch.empty((1, H, W), **i32)
    hit_cw = torch.empty((1, H, W), **f32)
    hit_dw = torch.empty((1, H, W), **f32)
    T_map = torch.empty((1, H, W), **f32)
    radii = torch.empty((P,), **i32)

    gb, ib, bb = C.c_size_t(), C.c_size_t(), C.c_size_t()
    saved = _Saved()
    saved.view_keep = keep
    saved.antialiased = antialiased  # the backward and the tangents of this forward use its mode, whatever the context then
    st.reap()  # counters of earlier calls that have arrived meanwhile (raises on an unnoticed overflow)
    shape_key = (P, H, W)
    wait = st.mode == "sync" or (st.mode == "auto" and shape_key not in st.seen)
    r_cap = int(st.r_hint)
    while True:
        check(L.rtg_splat_workspace_bytes(P, H, W, r_cap, C.byref(gb), C.byref(ib), C.byref(bb)), "rtg_splat_workspace_bytes")
        # one allocation for the three workspaces and the device counters (256-byte aligned pieces)
        ws = torch.empty(gb.value + ib.value + bb.value + 256, dtype=torch.uint8, device=device)
        base = ws.data_ptr()
        saved.ws = ws
        saved.geom, saved.img, saved.bin = base, base + gb.value, base + gb.value + ib.value
        saved.counters = base + gb.value + ib.value + bb.value
        saved.r_cap = r_cap
        pinned, event = st.get_pinned()
        check(L.rtg_splat_forward(
            C.byref(view), P, M, _ptr(means3D), _ptr(sh), _ptr(colors_precomp), _ptr(opacities), _ptr(scales), _ptr(rotations),
            _ptr(cov3Ds_precomp), _ptr(tile_mask), C.c_void_p(saved.geom), C.c_void_p(saved.img), C.c_void_p(saved.bin), r_cap,
            _ptr(color), _ptr(depth), _ptr(hit_color), _ptr(hit_depth), _ptr(hit_cw), _ptr(hit_dw), _ptr(T_map), _ptr(radii),
            C.c_void_p(saved.counters), C.c_void_p(pinned.data_ptr()), C.c_void_p(event.cuda_event), C.c_void_p(stream)),
            "rtg_splat_forward")
        pend = _Pending(pinned, event, r_cap)
        saved.pending = pend
        if not wait:
            st.pending.append(pend)  # read at the next call / at this call's backward
            break
        st.read(pend, block=True)  # waits for the scan kernel only; scatter / sort / render are still running
        if not pend.overflow:
            st.seen.add(shape_key)
            break
        r_cap = int(st.r_hint)
    return (color, depth, hit_color, hit_depth, hit_cw, hit_dw, T_map, radii), saved, (means3D, sh, colors_precomp, scales, rotations,
                                                                                    cov3Ds_precomp)


class _RasterizeGaussians(torch.autograd.Function):
    """The three trailing inputs are the settings' own viewmatrix / projmatrix / campos tensors, passed only when one of them
    requires grad (rasterize_gaussians): autograd then asks for their gradients through ctx.needs_input_grad."""

    @staticmethod
    def forward(ctx, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, tile_mask, raster_settings,
                viewmatrix=None, projmatrix=None, campos=None):
        outs, saved, inputs = _forward_native(raster_settings, means3D, sh, colors_precomp, opacities, scales, rotations,
                                              cov3Ds_precomp, tile_mask)
        color, depth, hit_color, hit_depth, hit_cw, hit_dw, T_map, radii = outs
        ctx.raster_settings = raster_settings
        ctx.native = saved
        if _SAVED_SINK[0] is not None:
            _SAVED_SINK[0].append(saved)
        ctx.provided = tuple(x is not None for x in inputs)
        ctx.camera_shapes = tuple(None if t is None else t.shape for t in (viewmatrix, projmatrix, campos))
        e = torch.empty(0, device=means3D.device)
        ctx.save_for_backward(*[x if x is not None else e for x in inputs], radii, hit_depth, T_map)
        ctx.mark_non_differentiable(hit_color, hit_depth, radii)
        # an output outside the loss arrives as None: an unused T_map selects the backward without the T term
        ctx.set_materialize_grads(False)
        return color, depth, hit_color, hit_depth, hit_cw, hit_dw, T_map, radii

    @staticmethod
    def backward(ctx, grad_out_color, grad_out_depth, grad_hit_color, grad_hit_depth, grad_hit_color_weight,
                 grad_hit_depth_weight, grad_T_map, _):
        L = _lib.lib()
        rs = ctx.raster_settings
        saved = ctx.native
        means3D, sh, colors_precomp, scales, rotations, cov3Ds_precomp, radii, hit_depth, T_map = ctx.saved_tensors
        has = ctx.provided
        sh = sh if has[1] else None
        colors_precomp = colors_precomp if has[2] else None
        scales = scales if has[3] else None
        rotations = rotations if has[4] else None
        cov3Ds_precomp = cov3Ds_precomp if has[5] else None
        device = means3D.device
        P = means3D.size(0)
        M = sh.size(1) if sh is not None else 0
        H, W = int(rs.image_height), int(rs.image_width)
        f32 = dict(dtype=torch.float32, device=device)
        if grad_out_color is None:
            grad_out_color = torch.zeros((3, H, W), **f32)
        if grad_out_depth is None:
            grad_out_depth = torch.zeros((1, H, W), **f32)
        grad_out_color = _f32_cuda(grad_out_color, "grad_out_color", device)
        grad_out_depth = _f32_cuda(grad_out_depth, "grad_out_depth", device)
        # dL/dT_map (None: T_map is not in the loss); T_map.sum() delivers a stride-0 view, made contiguous here
        grad_T = _f32_cuda(grad_T_map, "grad_T_map", device)
        view, keep = _make_view(rs, device, saved.antialiased)
        stream = torch.cuda.current_stream(device).cuda_stream
        st = _state(device)

        buf = _GRAD_BUFFERS[0]
        camera = any(ctx.needs_input_grad[9:])  # only present when rasterize_gaussians passed the camera tensors
        hook = _GRAD_RECORD_HOOK[0]
        # A frozen map (pose refinement): only the camera is differentiated. Autograd would discard per-Gaussian gradients
        # here, so rtg_splat_backward_pose computes none of them.
        pose_only = (camera and hook is None and buf is None and not _VISIBLE_ROWS_ONLY[0]
                     and not any(ctx.needs_input_grad[:7]))

        def out(name, shape):
            """Gradient tensor: a fresh allocation, or -- inside `grad_buffers(...)` -- a fresh alias of the caller's buffer
            (e.g. a view into parallel.FlatGrads: the kernels write straight into the all-reduce buffer, no packing)."""
            if buf is not None and name in buf:
                t = buf[name]
                if t.numel() != int(torch.Size(shape).numel()) or t.dtype != torch.float32 or t.device != device or not t.is_contiguous():
                    raise ValueError(f"grad buffer '{name}' must be a contiguous float32 tensor of {tuple(shape)} on {device}")
                if t.data_ptr() % 16:
                    raise ValueError(f"grad buffer '{name}' must start at a 16-byte aligned address (the kernels store 128 bits at a time)")
                return t.view(shape)
            return torch.empty(shape, **f32)
        if pose_only:
            g_means = g_opac = g_sh = g_colors = g_scales = g_rot = g_cov = None
        else:
            g_means = out("means3D", (P, 3))
            g_opac = out("opacities", (P, 1))
            g_sh = out("shs", (P, M, 3)) if sh is not None else None
            g_colors = torch.empty((P, 3), **f32) if colors_precomp is not None else None
            g_scales = out("scales", (P, 3)) if scales is not None else None
            g_rot = out("rotations", (P, 4)) if rotations is not None else None
            g_cov = torch.empty((P, 6), **f32) if cov3Ds_precomp is not None else None
        scratch = st.get_scratch(P)
        if not saved.pending.done:  # a forward that did not wait for its count: it has arrived by now
            st.read(saved.pending, block=True)
        if saved.pending.overflow:
            raise CapacityOverflow(f"rasterizer: this frame needed {saved.pending.num_rendered} (Gaussian, tile) instances but its "
                               f"binning buffer held {saved.pending.r_cap}; it was rendered empty. The capacity has been raised: "
                               "render it again (set_capacity_checks('sync') makes every forward check its own count).")
        if camera and hook is not None:
            raise RuntimeError("rasterizer: camera gradients (viewmatrix / projmatrix / campos with requires_grad) are not "
                               "available with a gradient-record exchange hook (set_grad_record_hook, tile-sharded frames)")
        g_cam = torch.zeros((35,), **f32) if camera else None  # (view 16, proj 16, campos 3); stays 0 for P == 0
        if P > 0:
            args = (C.byref(view), P, M, _ptr(means3D), _ptr(sh), _ptr(colors_precomp), _ptr(scales), _ptr(rotations),
                    _ptr(cov3Ds_precomp), _ptr(radii), C.c_void_p(saved.geom), C.c_void_p(saved.img), C.c_void_p(saved.bin), saved.r_cap,
                    C.c_void_p(saved.counters), _ptr(T_map), _ptr(hit_depth), _ptr(grad_out_color), _ptr(grad_out_depth), _ptr(scratch),
                    _ptr(g_means), _ptr(g_sh), _ptr(g_colors), _ptr(g_opac), _ptr(g_scales), _ptr(g_rot), _ptr(g_cov), None,
                    C.c_void_p(stream))
            if pose_only:
                cam_scratch = torch.empty((int(L.rtg_splat_camera_scratch_bytes(P)),), dtype=torch.uint8, device=device)
                check(L.rtg_splat_backward_pose(*args[:19], _ptr(grad_T), _ptr(scratch), _ptr(g_cam), _ptr(cam_scratch), args[-1]),
                      "rtg_splat_backward_pose")
            elif grad_T is not None:
                args_T = args[:19] + (_ptr(grad_T),) + args[19:]  # dL_dT goes right after dL_ddepth
                if hook is None:
                    cam_out = (None, None)
                    if camera:
                        cam_scratch = torch.empty((int(L.rtg_splat_camera_scratch_bytes(P)),), dtype=torch.uint8, device=device)
                        cam_out = (_ptr(g_cam), _ptr(cam_scratch))
                    check(L.rtg_splat_backward_dt(*args_T[:-1], 1 if _VISIBLE_ROWS_ONLY[0] else 0, *cam_out, args_T[-1]),
                          "rtg_splat_backward_dt")
                else:
                    check(L.rtg_splat_backward_render_dt(0, P, *args_T), "rtg_splat_backward_render_dt")
                    hook(scratch[:P * 16].view(P, 16))
                    check(L.rtg_splat_backward_finish(*args), "rtg_splat_backward_finish")
            elif camera:
                cam_scratch = torch.empty((int(L.rtg_splat_camera_scratch_bytes(P)),), dtype=torch.uint8, device=device)
                check(L.rtg_splat_backward_camera(*args[:-1], 1 if _VISIBLE_ROWS_ONLY[0] else 0, _ptr(g_cam), _ptr(cam_scratch),
                                                  args[-1]), "rtg_splat_backward_camera")
            elif hook is None and _VISIBLE_ROWS_ONLY[0]:
                check(L.rtg_splat_backward_visible(*args), "rtg_splat_backward_visible")
            elif hook is None:
                check(L.rtg_splat_backward(*args), "rtg_splat_backward")
            else:
                # exchange step between the compositing backward and the per-Gaussian backward (tile-sharded frames)
                check(L.rtg_splat_backward_render(*args), "rtg_splat_backward_render")
                hook(scratch[:P * 16].view(P, 16))
                check(L.rtg_splat_backward_finish(*args), "rtg_splat_backward_finish")
        # same order as the forward's arguments (reference __init__.py:269-279)
        grads = (g_means, g_sh, g_colors, g_opac, g_scales, g_rot, g_cov, None, None)
        if len(ctx.needs_input_grad) == 9:
            return grads
        cam = (slice(0, 16), slice(16, 32), slice(32, 35))
        return grads + tuple(g_cam[c].reshape(s) if n else None for c, s, n in zip(cam, ctx.camera_shapes, ctx.needs_input_grad[9:]))


# Optional list that receives the _Saved state of every forward (see `keep_saved`); None = not kept.
_SAVED_SINK = [None]


class keep_saved:
    """Context manager: while active, every rasterizer forward appends its _Saved state (workspaces, counters, mode) to
    the given list, so that a second pass can replay that forward (features.rasterize_features). Changes nothing else."""

    def __init__(self, sink):
        self.sink, self.prev = sink, None

    def __enter__(self):
        self.prev = _SAVED_SINK[0]
        _SAVED_SINK[0] = self.sink
        return self

    def __exit__(self, *exc):
        _SAVED_SINK[0] = self.prev
        return False


# Optional destination of the dense gradients (see `grad_buffers`); None = allocate per call.
_GRAD_BUFFERS = [None]


class grad_buffers:
    """Context manager: while active, the rasterizer backward writes dL/d{means3D, shs, opacities, scales, rotations} into
    the given tensors (dict by those names; e.g. `parallel.FlatGrads(P, dev).views`) instead of allocating new ones, so a
    following all-reduce over the flat buffer needs no packing copy. The tensors returned to autograd alias them."""

    def __init__(self, buffers):
        self.buffers, self.prev = buffers, None

    def __enter__(self):
        self.prev = _GRAD_BUFFERS[0]
        _GRAD_BUFFERS[0] = self.buffers
        return self

    def __exit__(self, *exc):
        _GRAD_BUFFERS[0] = self.prev
        return False


# When set, the backward leaves the gradient rows of culled Gaussians (radii <= 0) unwritten (see `visible_rows_only`).
_VISIBLE_ROWS_ONLY = [False]


class visible_rows_only:
    """Context manager: while active, the rasterizer backward writes only the gradient rows of Gaussians with radii > 0
    and leaves the others UNSPECIFIED (not zero) -- it skips the zero fill that a dense consumer needs (105 MB of stores
    per 1 M Gaussians). For consumers that mask by `radii` themselves: `mapoptim.MapOptimizer.step(radii=...)`."""

    def __init__(self, enabled=True):
        self.enabled, self.prev = bool(enabled), None

    def __enter__(self):
        self.prev = _VISIBLE_ROWS_ONLY[0]
        _VISIBLE_ROWS_ONLY[0] = self.enabled
        return self

    def __exit__(self, *exc):
        _VISIBLE_ROWS_ONLY[0] = self.prev
        return False


# When set, forwards render antialiased (see `antialiased`).
_ANTIALIASED = [False]


class antialiased:
    """Context manager: while active, rasterizer forwards render antialiased (RTG_VIEW_ANTIALIASED, the 2-D Mip filter of
    Mip-Splatting): each splat keeps its 0.3 px^2 dilation and its opacity is scaled by sqrt(max(det0 / det, 2.5e-5)),
    the ratio of the undilated to the dilated 2-D covariance determinant, so a sub-pixel Gaussian covers its true footprint
    instead of a 0.3 px^2 disc at full opacity. A forward records its mode: its backward (and the pose tangents of
    `tracking`) use that mode whatever the context is by then. Covers GaussianRasterizer, render.Renderer, MapOptimizer,
    tracking.PoseRefiner, tracking.pose_jacobian and parallel.GaussianShard."""

    def __init__(self, enabled=True):
        self.enabled, self.prev = bool(enabled), None

    def __enter__(self):
        self.prev = _ANTIALIASED[0]
        _ANTIALIASED[0] = self.enabled
        return self

    def __exit__(self, *exc):
        _ANTIALIASED[0] = self.prev
        return False


# Optional exchange step of the backward: a callable that receives the (P, 16) fp32 gradient-record tensor after the
# compositing backward and must leave the summed records in place (e.g. `dist.all_reduce`). Set by
# parallel.TileShard.exchange_records(); None = single call, no exchange.
_GRAD_RECORD_HOOK = [None]


def set_grad_record_hook(fn):
    """Install (or, with None, remove) the backward's exchange step; returns the previous hook."""
    prev = _GRAD_RECORD_HOOK[0]
    _GRAD_RECORD_HOOK[0] = fn
    return prev


def rasterize_gaussians(means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, tile_mask, raster_settings):
    """With grad mode on and any of raster_settings.viewmatrix / projmatrix / campos requiring grad, the backward also
    returns their gradients (dL/d of each tensor as stored, rtg_splat_backward_camera); otherwise they are constants. If
    none of the seven Gaussian inputs requires grad either (a frozen map, pose refinement), the backward computes the
    camera gradient alone (rtg_splat_backward_pose) and returns None for the Gaussians."""
    cam = (raster_settings.viewmatrix, raster_settings.projmatrix, raster_settings.campos)
    if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in cam):
        return _RasterizeGaussians.apply(means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, tile_mask,
                                         raster_settings, *cam)
    return _RasterizeGaussians.apply(means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, tile_mask,
                                     raster_settings)


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        with torch.no_grad():
            rs = self.raster_settings
            L = _lib.lib()
            device = positions.device
            pos = _f32_cuda(positions, "positions", device)
            P = pos.size(0)
            present = torch.empty((P,), dtype=torch.bool, device=device)
            vm = _f32_cuda(rs.viewmatrix, "viewmatrix", device)
            pm = _f32_cuda(rs.projmatrix, "projmatrix", device)
            if P > 0:
                check(L.rtg_splat_mark_visible(P, _ptr(pos), _ptr(vm), _ptr(pm), _ptr(present),
                                               C.c_void_p(torch.cuda.current_stream(device).cuda_stream)), "rtg_splat_mark_visible")
        return present

    def forward(self, means3D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None,
                tile_mask=None, normal_w=None):
        raster_settings = self.raster_settings

        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception("Please provide excatly one of either SHs or precomputed colors!")

        if ((scales is None or rotations is None) and cov3D_precomp is None) or (
            (scales is not None or rotations is not None) and cov3D_precomp is not None
        ):
            raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")

        empty = torch.Tensor([])
        if shs is None:
            shs = empty
        if colors_precomp is None:
            colors_precomp = empty
        if scales is None:
            scales = empty
        if rotations is None:
            rotations = empty
        if cov3D_precomp is None:
            cov3D_precomp = empty

        return rasterize_gaussians(means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, tile_mask,
                                   raster_settings)
