"""Frame-to-model projective point-to-plane ICP, API of the reference's SLAM/icp.py.

`ICP` and `IcpTracker` keep the constructor arguments, method names, argument order and return values of
the reference (SLAM/icp.py:16-48,357-452); the arithmetic runs in librtg_splat_b200.so. `IcpTracker.predict_pose`
is ONE cooperative kernel (all levels x all Gauss-Newton iterations: residuals + Jacobians + 27-term reduction +
damped 6x6 solve + exp_se3 + pose update, one grid barrier per iteration, then the point-to-plane loss) that writes
its 72-byte result straight into pinned host memory, and a pyramid is one launch, against ~600 eager ops and >= 45
host synchronisations in the reference. `ICP.icp` (one level) keeps the kernel-per-iteration entry point.
`RgbdIcpTracker` (no counterpart in the reference) adds a photometric term to the same one-launch loop."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import check


def _stream(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr())


_WS = {}
_RES = {}


def _result_buffers(device):
    """(device 18 floats, mapped pinned 18 floats, event) of predict_pose, one set per device."""
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _RES:
        _RES[idx] = (torch.zeros(18, dtype=torch.float32, device=torch.device("cuda", idx)),
                     torch.zeros(18, dtype=torch.float32).pin_memory(), torch.cuda.Event())
    return _RES[idx]



def _workspace(device):
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _WS:
        n = _lib.lib().rtg_icp_workspace_bytes(0, 0)
        _WS[idx] = torch.zeros(n, dtype=torch.uint8, device=torch.device("cuda", idx))
    return _WS[idx]


def _map3(t, name):
    if not t.is_cuda or t.dtype != torch.float32 or t.dim() != 3 or t.shape[-1] != 3:
        raise TypeError(f"{name} must be a CUDA float32 (H, W, 3) tensor")
    return t.contiguous()


def _intrinsics(K):
    """(fx, fy, cx, cy) python floats from a 3x3 tensor / array (one tiny read-back if it lives on the GPU)."""
    if isinstance(K, torch.Tensor):
        K = K.detach().cpu().numpy()
    K = np.asarray(K, dtype=np.float32)
    return float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])


def point2plane_loss(p_t0, p_t1, n_t0, reduce="mean"):
    loss = ((p_t1 - p_t0) * n_t0).sum(dim=-1)
    return (loss * loss).mean() if reduce == "mean" else (loss * loss).sum()


def build_level(depth, pool, fx, fy, cx, cy):
    """One pyramid level: max-pool by `pool`, back-project with the level intrinsics, Sobel normals.
    Returns (vertex, normal), each (H//pool, W//pool, 3)."""
    L = _lib.lib()
    if not depth.is_cuda or depth.dtype != torch.float32:
        raise TypeError("depth must be a CUDA float32 tensor")
    H, W = depth.shape[:2]
    d = depth.contiguous()
    Hs, Ws = H // pool, W // pool
    vertex = torch.empty((Hs, Ws, 3), dtype=torch.float32, device=d.device)
    normal = torch.empty((Hs, Ws, 3), dtype=torch.float32, device=d.device)
    check(L.rtg_icp_build_level(_p(d), H, W, pool, fx, fy, cx, cy, _p(vertex), _p(normal), _p(_workspace(d.device)), _stream(d.device)),
          "rtg_icp_build_level")
    return vertex, normal


def build_pyramids(depth, K, n_levels):
    """build_vertex_pyramid + build_normal_pyramid (SLAM/utils.py:511-527): index 0 is the coarsest level.
    One cooperative launch for all levels (rtg_icp_build_pyramid)."""
    fx, fy, cx, cy = K if isinstance(K, tuple) else _intrinsics(K)
    if not depth.is_cuda or depth.dtype != torch.float32:
        raise TypeError("depth must be a CUDA float32 tensor")
    if n_levels > 4:
        raise ValueError("at most 4 pyramid levels")
    L = _lib.lib()
    d = depth.contiguous()
    H, W = d.shape[:2]
    pools = [1 << (n_levels - 1 - i) for i in range(n_levels)]
    sc = [np.float32(1.0 / p) for p in pools]
    vs = [torch.empty((H // p, W // p, 3), dtype=torch.float32, device=d.device) for p in pools]
    ns = [torch.empty_like(v) for v in vs]
    I32, F32, VP = C.c_int32 * n_levels, C.c_float * n_levels, C.c_void_p * n_levels
    check(L.rtg_icp_build_pyramid(
        _p(d), H, W, n_levels, I32(*pools), F32(*[np.float32(fx) * s for s in sc]), F32(*[np.float32(fy) * s for s in sc]),
        F32(*[np.float32(cx) * s for s in sc]), F32(*[np.float32(cy) * s for s in sc]), VP(*[v.data_ptr() for v in vs]),
        VP(*[n.data_ptr() for n in ns]), _p(_workspace(d.device)), _stream(d.device)), "rtg_icp_build_pyramid")
    return vs, ns


class ICP(torch.nn.Module):
    def __init__(self, max_iter=3, damping=1e-6, distance_threshold=0.2, normal_threshold=20, verbose=False):
        super().__init__()
        self.max_iterations = max_iter
        self.distance_threshold = distance_threshold
        self.normal_threshold = np.cos(np.deg2rad(normal_threshold))
        self.damping = damping
        self.verbose = verbose

    def icp(self, pose10, vertex_t0, vertex_t1, normal_t0, normal_t1, K):
        """Same contract as ICP.icp (SLAM/icp.py:33-48): returns (pose10 (4,4) float32 tensor, valid_ratio tensor)."""
        L = _lib.lib()
        v0, v1 = _map3(vertex_t0, "vertex_t0"), _map3(vertex_t1, "vertex_t1")
        n0, n1 = _map3(normal_t0, "normal_t0"), _map3(normal_t1, "normal_t1")
        device = v0.device
        H, W = v0.shape[:2]
        fx, fy, cx, cy = K if isinstance(K, tuple) else _intrinsics(K)
        pose = pose10.detach().to(device=device, dtype=torch.float32).contiguous().clone()
        valid_ratio = torch.zeros((), dtype=torch.float32, device=device)
        check(L.rtg_icp_solve_level(_p(v0), _p(n0), _p(v1), _p(n1), H, W, fx, fy, cx, cy, float(self.distance_threshold),
                                    float(self.normal_threshold), float(self.damping), int(self.max_iterations), _p(pose),
                                    _p(valid_ratio), _p(_workspace(device)), _stream(device)), "rtg_icp_solve_level")
        return pose, valid_ratio


class IcpTracker:
    def __init__(self, args):
        self.icp_trackers = []
        self.icp_downscales = args.icp_downscales
        self.icp_warmup_frames = args.icp_warmup_frames
        self.icp_use_model_depth = args.icp_use_model_depth
        for iters in args.icp_downscale_iters:
            self.icp_trackers.append(ICP(iters, distance_threshold=args.icp_distance_threshold,
                                         normal_threshold=args.icp_normal_threshold, damping=args.icp_damping,
                                         verbose=args.verbose))
        self.icp_sample_distance_threshold = args.icp_sample_distance_threshold
        self.icp_sample_normal_threshold = args.icp_sample_normal_threshold
        self.icp_fail_threshold = args.icp_fail_threshold
        self.normal_pyramid_t0 = None
        self.vertex_pyramid_t0 = None
        self.verbose = args.verbose
        self.K = None
        self._Kf = None
        self.last_p2ploss = None
        self.last_valid_ratio = None

    def _set_K(self, K):
        self.K = K
        self._Kf = _intrinsics(K)

    def update_curr_status(self, depth_t1, K):
        if self.K is None:
            self._set_K(K)
        self.depth_t1 = depth_t1
        self.vertex_pyramid_t1, self.normal_pyramid_t1 = build_pyramids(depth_t1, self._Kf, len(self.icp_downscales))

    def move_last_status(self):
        self.vertex_pyramid_t0 = self.vertex_pyramid_t1
        self.normal_pyramid_t0 = self.normal_pyramid_t1
        self.last_model_depth = self.depth_t1

    def update_last_status(self, frame, render_depth, frame_depth, render_normal, frame_normal):
        """Fills `render_depth` in place from the measured depth where the model disagrees (SLAM/icp.py:397-415)."""
        L = _lib.lib()
        if not (render_depth.is_contiguous() and render_depth.is_cuda and render_depth.dtype == torch.float32):
            raise TypeError("render_depth must be a contiguous CUDA float32 tensor (it is updated in place)")
        H, W = render_depth.shape[:2]
        fd = frame_depth.contiguous()
        rn, fn = _map3(render_normal, "render_normal"), _map3(frame_normal, "frame_normal")
        check(L.rtg_icp_fill_model_depth(_p(render_depth), _p(fd), _p(rn), _p(fn), H, W, float(self.icp_sample_distance_threshold),
                                         float(self.icp_sample_normal_threshold), _stream(render_depth.device)),
              "rtg_icp_fill_model_depth")
        self.last_model_depth = render_depth

    def predict_pose(self, frame):
        K = frame["K"]
        frame_id = frame["frame_id"]
        if self.vertex_pyramid_t0 is None:
            # the reference sets the identity pose and then subscripts the None pyramid in point2plane_loss
            # (SLAM/icp.py:421-449): same exception type; callers only get here after move_last_status()
            self._set_K(K)
            raise TypeError("'NoneType' object is not subscriptable (predict_pose before move_last_status: no previous frame)")
        L = _lib.lib()
        levels = len(self.icp_downscales)
        if self.icp_use_model_depth and frame_id >= self.icp_warmup_frames:
            self.vertex_pyramid_t0, self.normal_pyramid_t0 = build_pyramids(self.last_model_depth, self._Kf, levels)
        device = self.vertex_pyramid_t1[0].device
        Kf = _intrinsics(K) if K is not self.K else self._Kf
        lv = (_lib.RtgIcpLevel * levels)()
        keep = []
        for level in range(levels):
            s = np.float32(self.icp_downscales[level])
            # argument swap of the reference: "0" inside icp() is the CURRENT frame (SLAM/icp.py:438-441)
            v0, n0 = _map3(self.vertex_pyramid_t1[level], "vertex_t1"), _map3(self.normal_pyramid_t1[level], "normal_t1")
            v1, n1 = _map3(self.vertex_pyramid_t0[level], "vertex_t0"), _map3(self.normal_pyramid_t0[level], "normal_t0")
            keep += [v0, n0, v1, n1]
            trk = self.icp_trackers[level]
            e = lv[level]
            e.vertex0, e.normal0, e.vertex1, e.normal1 = v0.data_ptr(), n0.data_ptr(), v1.data_ptr(), n1.data_ptr()
            e.H, e.W = v0.shape[0], v0.shape[1]
            e.fx, e.fy, e.cx, e.cy = (float(np.float32(k) * s) for k in Kf)
            e.iters = int(trk.max_iterations)
        t0 = self.icp_trackers[0]  # thresholds are shared by all levels (IcpTracker.__init__)
        out, pinned, event = _result_buffers(device)
        v_t0, v_t1, n_t0 = keep[-2], keep[-4], keep[-1]
        H, W = v_t0.shape[:2]
        stream = torch.cuda.current_stream(device)
        check(L.rtg_icp_predict_pose(lv, levels, float(t0.distance_threshold), float(t0.normal_threshold), float(t0.damping), None,
                                     _p(v_t0), _p(v_t1), _p(n_t0), H, W, _p(out), C.c_void_p(pinned.data_ptr()),
                                     _p(_workspace(device)), C.c_void_p(stream.cuda_stream)), "rtg_icp_predict_pose")
        event.record(stream)
        event.synchronize()  # the only wait of the solve; the kernel wrote the 18 floats into pinned host memory itself
        host = pinned.numpy().copy()
        pose_t1_t0 = host[:16].reshape(4, 4).astype(np.float32)
        self.last_p2ploss, self.last_valid_ratio = float(host[16]), float(host[17])
        if self.verbose:
            print(self.last_p2ploss, self.last_valid_ratio)
        tracking_success = not (self.last_p2ploss > self.icp_fail_threshold)
        return pose_t1_t0, tracking_success


# ---------------------------------------------------------------------------------------------------- RGB-D tracking
_RES_RGBD = {}


def _result_buffers_rgbd(device):
    """(device 20 floats, mapped pinned 20 floats, event) of RgbdIcpTracker.predict_pose, one set per device."""
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _RES_RGBD:
        _RES_RGBD[idx] = (torch.zeros(20, dtype=torch.float32, device=torch.device("cuda", idx)),
                          torch.zeros(20, dtype=torch.float32).pin_memory(), torch.cuda.Event())
    return _RES_RGBD[idx]


def _color_layout(color, H, W):
    """True for (H, W, 3), False for (3, H, W); TypeError / ValueError before any CUDA work otherwise."""
    if not isinstance(color, torch.Tensor) or not color.is_cuda or color.dtype != torch.float32:
        raise TypeError("color must be a CUDA float32 tensor, (H, W, 3) or (3, H, W)")
    if color.dim() == 3 and tuple(color.shape) == (H, W, 3):
        return True
    if color.dim() == 3 and tuple(color.shape) == (3, H, W):
        return False
    raise ValueError(f"color must be (H, W, 3) or (3, H, W) with (H, W) = ({H}, {W}) of the depth; got {tuple(color.shape)}")


def build_intensity_pyramid(color, n_levels):
    """Intensity pyramid of the photometric ICP term, index 0 the coarsest level like build_pyramids: level i has
    pool p = 2**(n_levels-1-i) and (H//p, W//p) pixels, each the mean of Y = 0.299 R + 0.587 G + 0.114 B over the p x p
    block whose depth maximum build_pyramids takes. `color`: CUDA float32, (H, W, 3) or (3, H, W). One launch."""
    if not isinstance(color, torch.Tensor) or color.dim() != 3:
        raise TypeError("color must be a CUDA float32 tensor, (H, W, 3) or (3, H, W)")
    if not 1 <= n_levels <= 4:
        raise ValueError("1 to 4 pyramid levels")
    H, W = (color.shape[0], color.shape[1]) if color.shape[-1] == 3 else (color.shape[1], color.shape[2])
    channels_last = _color_layout(color, H, W)
    c = color.contiguous()
    pools = [1 << (n_levels - 1 - i) for i in range(n_levels)]
    out = [torch.empty((H // p, W // p), dtype=torch.float32, device=c.device) for p in pools]
    I32, VP = C.c_int32 * n_levels, C.c_void_p * n_levels
    check(_lib.lib().rtg_icp_build_intensity_pyramid(_p(c), H, W, 1 if channels_last else 0, n_levels, I32(*pools),
                                                     VP(*[o.data_ptr() for o in out]), _stream(c.device)),
          "rtg_icp_build_intensity_pyramid")
    return out


class RgbdIcpTracker(IcpTracker):
    """IcpTracker with a photometric term in the same Gauss-Newton loop (RGB-D odometry as in ElasticFusion / DVO).

    Per pixel with a valid point-to-plane row, r = I_prev(u, v) - I_curr[q] at the projection the geometric row
    computes, bilinear in the previous frame's level intensity; H = sum_geo J^T J + photometric_weight * sum_photo J^T J
    (and g alike). `photometric_weight` is in m^2 per squared intensity unit; the default 0.01 = (2 mm / 0.02)^2 is the
    ratio of sensor depth noise to intensity noise. Frames without colour, or a weight of 0, track exactly as IcpTracker.
    In frame-to-model mode the model depth is IcpTracker's and the model intensity is the previous frame's measured one
    (the render is made at that frame's tracked pose, so it shares its pixel grid)."""

    def __init__(self, args, photometric_weight=0.01):
        w = float(photometric_weight)
        if not (w >= 0.0 and np.isfinite(w)):
            raise ValueError("photometric_weight must be finite and >= 0")
        super().__init__(args)
        self.photometric_weight = w
        self.intensity_pyramid_t0 = None
        self.intensity_pyramid_t1 = None
        self.last_photometric_ratio = None
        self.last_photometric_rmse = None

    def update_curr_status(self, depth_t1, K, color_t1=None):
        if color_t1 is not None:  # checked before any CUDA work
            if not isinstance(depth_t1, torch.Tensor):
                raise TypeError("depth_t1 must be a CUDA float32 tensor")
            _color_layout(color_t1, depth_t1.shape[0], depth_t1.shape[1])
        super().update_curr_status(depth_t1, K)
        self.intensity_pyramid_t1 = None if color_t1 is None else build_intensity_pyramid(color_t1, len(self.icp_downscales))

    def move_last_status(self):
        super().move_last_status()
        self.intensity_pyramid_t0 = self.intensity_pyramid_t1

    def predict_pose(self, frame):
        if (self.vertex_pyramid_t0 is None or self.intensity_pyramid_t0 is None or self.intensity_pyramid_t1 is None
                or not self.photometric_weight > 0.0):
            self.last_photometric_ratio, self.last_photometric_rmse = 0.0, 0.0
            return super().predict_pose(frame)
        K = frame["K"]
        frame_id = frame["frame_id"]
        L = _lib.lib()
        levels = len(self.icp_downscales)
        if self.icp_use_model_depth and frame_id >= self.icp_warmup_frames:
            self.vertex_pyramid_t0, self.normal_pyramid_t0 = build_pyramids(self.last_model_depth, self._Kf, levels)
        device = self.vertex_pyramid_t1[0].device
        Kf = _intrinsics(K) if K is not self.K else self._Kf
        lv = (_lib.RtgIcpLevel * levels)()
        VP = C.c_void_p * levels
        i0 = VP(*[self.intensity_pyramid_t1[level].data_ptr() for level in range(levels)])
        i1 = VP(*[self.intensity_pyramid_t0[level].data_ptr() for level in range(levels)])
        keep = []
        for level in range(levels):
            s = np.float32(self.icp_downscales[level])
            # "0" inside the solve is the CURRENT frame, as in IcpTracker.predict_pose
            v0, n0 = _map3(self.vertex_pyramid_t1[level], "vertex_t1"), _map3(self.normal_pyramid_t1[level], "normal_t1")
            v1, n1 = _map3(self.vertex_pyramid_t0[level], "vertex_t0"), _map3(self.normal_pyramid_t0[level], "normal_t0")
            if (tuple(self.intensity_pyramid_t1[level].shape) != tuple(v0.shape[:2])
                    or tuple(self.intensity_pyramid_t0[level].shape) != tuple(v1.shape[:2])):
                raise ValueError("colour and depth of a frame must have the same size")
            keep += [v0, n0, v1, n1]
            trk = self.icp_trackers[level]
            e = lv[level]
            e.vertex0, e.normal0, e.vertex1, e.normal1 = v0.data_ptr(), n0.data_ptr(), v1.data_ptr(), n1.data_ptr()
            e.H, e.W = v0.shape[0], v0.shape[1]
            e.fx, e.fy, e.cx, e.cy = (float(np.float32(k) * s) for k in Kf)
            e.iters = int(trk.max_iterations)
        t0 = self.icp_trackers[0]
        out, pinned, event = _result_buffers_rgbd(device)
        v_t0, v_t1, n_t0 = keep[-2], keep[-4], keep[-1]
        H, W = v_t0.shape[:2]
        stream = torch.cuda.current_stream(device)
        check(L.rtg_icp_predict_pose_rgbd(lv, i0, i1, levels, float(t0.distance_threshold), float(t0.normal_threshold),
                                          float(t0.damping), self.photometric_weight, None, _p(v_t0), _p(v_t1), _p(n_t0), H, W,
                                          _p(out), C.c_void_p(pinned.data_ptr()), _p(_workspace(device)),
                                          C.c_void_p(stream.cuda_stream)), "rtg_icp_predict_pose_rgbd")
        event.record(stream)
        event.synchronize()  # the kernel wrote the 20 floats into pinned host memory itself
        host = pinned.numpy().copy()
        pose_t1_t0 = host[:16].reshape(4, 4).astype(np.float32)
        self.last_p2ploss, self.last_valid_ratio = float(host[16]), float(host[17])
        self.last_photometric_ratio, self.last_photometric_rmse = float(host[18]), float(host[19])
        if self.verbose:
            print(self.last_p2ploss, self.last_valid_ratio, self.last_photometric_ratio, self.last_photometric_rmse)
        tracking_success = not (self.last_p2ploss > self.icp_fail_threshold)
        return pose_t1_t0, tracking_success
