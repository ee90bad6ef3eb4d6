"""Render-based camera tracking against a frozen map: photometric + geometric pose refinement.

`PoseRefiner.refine` minimises the fused L1 colour + depth loss of a render against a measured frame over the camera
pose, as MonoGS- and SplaTAM-style trackers do. Per iteration it runs four pieces of native work and builds no pose
arithmetic in torch:
  1. the rasterizer forward (`rasterize_gaussians`) with the refiner's own viewmatrix / projmatrix / campos tensors
     requiring grad and the map detached;
  2. `loss.l1_color_depth_loss` (rtg_loss_l1);
  3. `loss.backward()`: no Gaussian input requires grad, so the rasterizer runs rtg_splat_backward_pose, which computes
     the camera gradient and nothing per Gaussian;
  4. rtg_pose_adam_step: the gradient of a left twist xi = (rho, phi) of W2C at zero, one Adam step on it, W2C <- exp(xi^)
     W2C (the pose is kept in double on the device), the three camera tensors rewritten in place, xi reset to zero.

No value is read back to the host inside the loop. What remains is the rasterizer's own capacity bookkeeping: the first
forward of a (P, H, W) shape waits for its scan kernel (and re-runs on a binning overflow), and every backward waits for
its forward's scan-kernel event before it launches -- so the host runs at most about one iteration ahead of the GPU. A
later iteration whose pose needs more binning capacity than the buffer holds is rendered empty; its backward raises
`rasterizer.CapacityOverflow` before any work, with the capacity already raised, and the refiner renders that iteration
again (the pose and Adam's state are untouched by the failed attempt).

`PoseRefiner.refine_gn` minimises the squared colour + depth residuals over the same pixels by damped Gauss-Newton: per
iteration the forward, then rtg_splat_pose_gn_step, which computes the forward-mode tangents of the render along the six
twist directions, forms and solves the 6x6 normal equations and updates the pose, all on the device. `pose_jacobian`
returns those tangent images themselves. Optionally it runs coarse to fine over an image pyramid (`downsample_frame`,
`level_camera`) and weighs each residual by the Huber loss (rtg_splat_pose_gn_step_robust).

Both refiners can estimate the frame's exposure with the pose (`exposure=`): the camera's pixel values are modelled as
e^a C + b of the map's radiance C, one gain and one offset per frame (`apply_exposure`), so that auto-exposure is not
explained by a pose change. `refine_gn` then solves for eight unknowns per step (rtg_splat_pose_gn_step_exposure); `refine`
takes the loss under the exposure (rtg_loss_l1_exposure) and one more Adam step on (a, b).

When to track with either (every frame, after ICP, on keyframes only) is SLAM policy and is left to the caller."""
from __future__ import annotations

import contextlib
import ctypes as C
import math
import types

import torch

from . import _lib, rasterizer
from ._lib import RtgPoseAdam, RtgPoseGN, check
from .loss import frame_targets, l1_color_depth_loss
from .optim import FusedAdam
from .rasterizer import CapacityOverflow, GaussianRasterizationSettings, _forward_native, _make_view, rasterize_gaussians
from .render import Renderer


def _native_args(rs, saved, ins, dev):
    """(view, P, M, the six Gaussian inputs, the three workspaces, R_cap, counters) of one rasterizer forward, the head of
    both tangent entry points' argument lists. The view struct holds the settings' camera tensors by pointer."""
    means3D, sh, colors_precomp, scales, rotations, cov3D_precomp = ins
    view, keep = _make_view(rs, dev, saved.antialiased)
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    return (C.byref(view), int(means3D.shape[0]), int(sh.shape[1]) if sh is not None else 0, p(means3D), p(sh), p(colors_precomp),
            p(scales), p(rotations), p(cov3D_precomp), C.c_void_p(saved.geom), C.c_void_p(saved.img), C.c_void_p(saved.bin),
            saved.r_cap, C.c_void_p(saved.counters))


def _check_depth(depth):
    if depth not in ("hit", "expected"):
        raise ValueError('depth must be "hit" or "expected"')


def pose_jacobian(raster_settings, means3D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                  cov3D_precomp=None, tile_mask=None, depth="hit"):
    """One rasterizer forward at the settings' camera and the forward-mode tangents of its render along the six directions
    of a left twist xi = (rho, phi) of the pose (rtg_splat_pose_tangents). Returns (outputs, J): the forward's eight outputs
    as GaussianRasterizer returns them, and J (6, 4, H, W) float32, J[k] = d(colour r, g, b, depth) / d xi_k. Inputs as
    GaussianRasterizer takes them; nothing is differentiated by autograd.
    `depth="expected"` (rtg_splat_pose_tangents_expected): channel 3 of J is the tangent of the alpha-blended depth
    D = sum w z / sum w of the forward's blend weights w = alpha T (0 where sum w = 0), and a third value is returned:
    `expected` (2, H, W) float32 = (D, sum w), the map the tangents were replayed from."""
    _check_depth(depth)
    with torch.no_grad():
        dev = means3D.device
        st = rasterizer._state(dev)
        for attempt in range(2):
            outs, saved, ins = _forward_native(raster_settings, means3D, shs, colors_precomp, opacities, scales, rotations,
                                               cov3D_precomp, tile_mask)
            st.read(saved.pending, block=True)
            if not saved.pending.overflow:
                break
            if attempt:
                raise CapacityOverflow("pose_jacobian: the render overflowed the binning buffer twice")
        L = _lib.lib()
        H, W = int(raster_settings.image_height), int(raster_settings.image_width)
        P = int(means3D.shape[0])
        scratch = torch.empty((int(L.rtg_splat_pose_gn_scratch_bytes(P, H, W)),), dtype=torch.uint8, device=dev)
        J = torch.empty((6, 4, H, W), dtype=torch.float32, device=dev)
        if depth == "expected":
            expected = torch.empty((2, H, W), dtype=torch.float32, device=dev)
            check(L.rtg_splat_pose_tangents_expected(*_native_args(raster_settings, saved, ins, dev), C.c_void_p(scratch.data_ptr()),
                                                     C.c_void_p(J.data_ptr()), C.c_void_p(expected.data_ptr()),
                                                     C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                  "rtg_splat_pose_tangents_expected")
            return outs, J, expected
        check(L.rtg_splat_pose_tangents(*_native_args(raster_settings, saved, ins, dev), C.c_void_p(outs[3].data_ptr()),
                                        C.c_void_p(scratch.data_ptr()), C.c_void_p(J.data_ptr()),
                                        C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "rtg_splat_pose_tangents")
        return outs, J


def apply_exposure(image, exposure):
    """`image` seen under the exposure (a, b): e^a image + b. `exposure`: a pair of floats or a 2-element tensor."""
    a, b = exposure[0], exposure[1]
    return (torch.exp(a) if torch.is_tensor(a) else math.exp(a)) * image + b


def _exposure_pair(exposure, dev, dtype):
    """A fresh (2,) tensor (a, b) on `dev` from a pair of floats or a 2-element tensor."""
    if torch.is_tensor(exposure):
        t = exposure.detach().to(device=dev, dtype=dtype).reshape(-1).clone()
    else:
        t = torch.tensor([float(x) for x in exposure], dtype=dtype, device=dev)
    if t.numel() != 2:
        raise ValueError("exposure must hold two numbers (a, b)")
    return t


def level_camera(camera, s):
    """The camera of pyramid level `s` (an integer >= 1) of `camera`, for images made by `downsample_frame`: the
    Camera-like object PoseRefiner reads (world_view_transform, projection_matrix, FoVx, FoVy, image_height, image_width,
    cx, cy). The rasterizer samples integer pixel coordinates (pixel = fx x / z + cx, fx = W / (2 tanfovx)), so coarse
    pixel i looks along the ray of the fine block centre s i + (s - 1) / 2: with W_s = W // s,
      fx_s = fx / s,  tanfovx_s = tanfovx s W_s / W,  cx_s = (cx - (s - 1) / 2) / s,
    projection_matrix[0][0] scaled by W / (s W_s) (float64; the z rows unchanged), and likewise in y with H, H_s, cy.
    The pose is shared with `camera`."""
    s = int(s)
    W, H = int(camera.image_width), int(camera.image_height)
    if s < 1 or W // s < 1 or H // s < 1:
        raise ValueError(f"there is no level {s} of a {W}x{H} camera")
    Ws, Hs = W // s, H // s
    projection = camera.projection_matrix.detach().to(torch.float64).clone()
    projection[0, 0] *= W / (s * Ws)
    projection[1, 1] *= H / (s * Hs)
    return types.SimpleNamespace(
        world_view_transform=camera.world_view_transform, projection_matrix=projection,
        FoVx=2 * math.atan(math.tan(camera.FoVx * 0.5) * s * Ws / W), FoVy=2 * math.atan(math.tan(camera.FoVy * 0.5) * s * Hs / H),
        image_width=Ws, image_height=Hs, cx=(camera.cx - (s - 1) / 2) / s, cy=(camera.cy - (s - 1) / 2) / s)


def downsample_frame(gt_color, gt_depth, s, render_mask=None, tile_mask=None):
    """Level `s` (>= 2) of a measured frame, in one launch of rtg_frame_downsample. gt_depth (H, W) or (1, H, W) float32
    sets the size; gt_color (3, H, W) or (H, W, 3) float32; render_mask (H, W), any dtype, nonzero = selected; tile_mask
    the rasterizer's int32 (ceil(H/16), ceil(W/16)) tile mask. All on one CUDA device. Returns (color (3, H_s, W_s),
    depth (H_s, W_s), mask (H_s, W_s) uint8 or None, tile_mask (ceil(H_s/16), ceil(W_s/16)) int32 or None) with
    H_s = H // s, W_s = W // s: colour is the block mean, depth the block mean where all s^2 depths are > 0 (else 0), the
    render mask set where all s^2 pixels are set, a coarse tile set where any of its s x s fine tiles is set."""
    s = int(s)
    if s < 2:
        raise ValueError("s must be >= 2")
    H, W = int(gt_depth.shape[-2]), int(gt_depth.shape[-1])
    gt_color, gt_depth, mask, channels_last = frame_targets(gt_color, gt_depth, render_mask, H, W)
    dev = gt_depth.device
    Hs, Ws = H // s, W // s
    color = torch.empty((3, Hs, Ws), dtype=torch.float32, device=dev)
    depth = torch.empty((Hs, Ws), dtype=torch.float32, device=dev)
    mask_out = None if mask is None else torch.empty_like(depth, dtype=torch.uint8)
    tmask = tmask_out = None
    if tile_mask is not None:
        if not tile_mask.is_cuda or tile_mask.dtype != torch.int32:
            raise TypeError("tile_mask must be a CUDA int32 tensor")
        if tile_mask.numel() != ((H + 15) // 16) * ((W + 15) // 16):
            raise ValueError(f"tile_mask must have {(H + 15) // 16}x{(W + 15) // 16} entries")
        tmask = tile_mask.contiguous()
        tmask_out = torch.empty(((Hs + 15) // 16, (Ws + 15) // 16), dtype=torch.int32, device=dev)
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    check(_lib.lib().rtg_frame_downsample(p(gt_color), p(gt_depth), p(mask), p(tmask), H, W, s, channels_last, p(color), p(depth),
                                          p(mask_out), p(tmask_out), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
          "rtg_frame_downsample")
    return color, depth, mask_out, tmask_out


def camera_tensors(pose, projection):
    """The three camera tensors the rasterizer reads, as rtg_pose_adam_step writes them: viewmatrix = W2C^T, projmatrix =
    viewmatrix @ projection and campos = -R^T t, float32 and contiguous, from the double W2C `pose` (4, 4) and the float32
    `projection` (4, 4)."""
    view = pose.t().float().contiguous()
    proj = (pose.t() @ projection.double()).float().contiguous()
    campos = (-(pose[:3, :3].t() @ pose[:3, 3])).float().contiguous()
    return view, proj, campos


class PoseRefiner:
    """Refines a world-to-camera pose against a frozen Gaussian map. `args` is the bag `render.Renderer` takes."""

    def __init__(self, args):
        self._renderer = Renderer(args)  # rasterizer settings exactly as Renderer.render makes them

    def _settings(self, camera, dev, view, proj, campos):
        """Rasterizer settings at `camera`'s image size and intrinsics over the three camera tensors."""
        r = self._renderer
        return GaussianRasterizationSettings(
            image_height=int(camera.image_height), image_width=int(camera.image_width),
            tanfovx=math.tan(camera.FoVx * 0.5), tanfovy=math.tan(camera.FoVy * 0.5), bg=r.bg_color.to(dev),
            scale_modifier=r.scaling_modifier, viewmatrix=view, projmatrix=proj, sh_degree=r.active_sh_degree, campos=campos,
            opaque_threshold=r.renderer_opaque_threshold, depth_threshold=r.renderer_depth_threshold,
            normal_threshold=r.renderer_normal_threshold, color_sigma=r.color_sigma, prefiltered=False, debug=False,
            cx=camera.cx, cy=camera.cy, T_threshold=0.0001)

    def _setup(self, camera, gaussian_data, requires_grad):
        """The double pose W2C, the projection, the three camera tensors the rasterizer reads (rewritten in place by the
        device pose steps), the rasterizer settings over them and the detached map."""
        dev = gaussian_data["xyz"].device
        vm0 = camera.world_view_transform.detach().to(device=dev, dtype=torch.float64)
        pose = vm0.t().contiguous()                                   # W2C, row-major, double
        projection = camera.projection_matrix.detach().to(device=dev, dtype=torch.float32).contiguous()
        view, proj, campos = (t.requires_grad_(requires_grad) for t in camera_tensors(pose, projection))
        rs = self._settings(camera, dev, view, proj, campos)
        g = {k: gaussian_data[k].detach() for k in ("xyz", "opacity", "shs", "scales", "rotations")}
        return dev, pose, projection, view, proj, campos, rs, g

    def refine_gn(self, camera, gaussian_data, gt_color, gt_depth, iters, damping=1e-4, color_weight=0.8, depth_weight=1.0,
                  render_mask=None, tile_mask=None, depth_error_max=0.1, scales=(1,), robust=None, color_delta=0.1,
                  depth_delta=0.05, exposure=None, coarse_antialias=False, depth="hit", min_coverage=0.5):
        """Gauss-Newton refinement of the pose on the squared colour + depth residuals (rtg_splat_pose_gn_step): per
        iteration the rasterizer forward, then the forward-mode tangents of the render along the six twist directions, the
        normal equations over rtg_loss_l1's pixel selection, the damped solve (H + damping * trace(H) * I) and
        W2C <- exp(xi^) W2C, all on the device. No autograd is involved and nothing is read back inside the loop, except
        that each iteration waits for its forward's scan kernel: an iteration whose render overflowed the binning buffer is
        rendered again (with the capacity raised), keeping the pose refined so far.

        Arguments as in `refine`; `damping` scales the trace added to the diagonal.
        `scales`: the image pyramid, decreasing and ending in 1, e.g. (4, 2, 1). Level s renders at `level_camera(camera,
        s)` against `downsample_frame(...)` of the targets and masks (made once per call); level 1 uses the caller's
        tensors. The pose carries over from level to level on the device. `iters`: one count for every level, or one per
        entry of `scales`. A level whose selection is empty leaves the pose as it is and the next level goes on from it.
        `robust`: None (squared residuals) or "huber" (rtg_splat_pose_gn_step_robust: Huber loss with thresholds
        `color_delta` in colour units and `depth_delta` in map units, minimised by reweighted least squares).
        The defaults (one level, no robust loss) run one rtg_splat_pose_gn_step per iteration and nothing else.
        `exposure`: None, or the starting exposure (a0, b0) of the frame (a pair of floats or a 2-element tensor; (0, 0)
        for none, the previous frame's estimate when tracking a sequence). The colour residual becomes e^a C + b - C^ and
        each step solves for (rho, phi, a, b) (rtg_splat_pose_gn_step_exposure: the pose diagonals damped as above, the
        exposure diagonals scaled by 1 + damping), with any `scales` and `robust`. A block mean is linear, so (a, b) of the
        frame is (a, b) of every level and carries over as the pose does. A third value is then returned: the estimate,
        a (2,) float64 CUDA tensor.
        `coarse_antialias`: True renders the levels s >= 2 antialiased (`rasterizer.antialiased`): a map of sub-pixel
        surfels then renders at a coarse level close to the block mean of its fine render, which a plain render is not.
        Level 1 renders in the mode of the caller's context.
        `depth`: "hit" (the default) takes the depth residual on the opaque-surfel depth of the pixel's hit Gaussian, as
        above. "expected" (rtg_splat_pose_gn_step_expected) takes it on the alpha-blended depth D = sum w z / sum w of the
        forward's blend weights w = alpha T, over the pixels of the render mask with coverage sum w >= `min_coverage` (in
        (0, 1]), a measured depth and D - gt_depth < depth_error_max; the colour rows, weights, Huber rule and exposure are
        unchanged. It combines with `scales`, `coarse_antialias`, `robust` and `exposure`.

        Returns (W2C, report): the refined pose, a (4, 4) float64 CUDA tensor, and the finest level's last step's report,
        a float64 CUDA tensor [E, E_colour, E_depth, N_c, N_d, |rho|, |phi|, status] (E evaluated before that step; status
        0 ok, 1 singular system, 2 no selected pixel, 3 overflowed forward -- the pose is then left unchanged)."""
        scales = tuple(int(x) for x in scales)
        if not scales or scales[-1] != 1 or any(a <= b for a, b in zip(scales, scales[1:])):
            raise ValueError("scales must be decreasing and end in 1")
        level_iters = [int(i) for i in iters] if isinstance(iters, (list, tuple)) else [int(iters)] * len(scales)
        if len(level_iters) != len(scales):
            raise ValueError("iters must be an int or one count per entry of scales")
        if min(level_iters) < 1:
            raise ValueError("iters must be >= 1")
        if robust not in (None, "huber"):
            raise ValueError('robust must be None or "huber"')
        _check_depth(depth)
        min_coverage = float(min_coverage)
        if not 0.0 < min_coverage <= 1.0:
            raise ValueError("min_coverage must be in (0, 1]")
        dev, pose, projection, view, proj, campos, rs, g = self._setup(camera, gaussian_data, requires_grad=False)
        H, W = int(rs.image_height), int(rs.image_width)
        gt_color, gt_depth, mask, channels_last = frame_targets(gt_color, gt_depth, render_mask, H, W)
        P = int(g["xyz"].shape[0])
        L = _lib.lib()
        scratch_bytes = L.rtg_splat_pose_gn_scratch_bytes if exposure is None else L.rtg_splat_pose_gn_exposure_scratch_bytes
        scratch = torch.empty((int(scratch_bytes(P, H, W)),), dtype=torch.uint8, device=dev)  # the finest level's
        report = torch.zeros(_lib.RTG_POSE_GN_REPORT_LEN, dtype=torch.float64, device=dev)

        def state(projection, gt_color, gt_depth, mask, channels_last):
            s = RtgPoseGN()
            s.pose, s.projection, s.viewmatrix, s.projmatrix, s.campos = (t.data_ptr() for t in (pose, projection, view, proj, campos))
            s.gt_color, s.gt_depth = gt_color.data_ptr(), gt_depth.data_ptr()
            s.render_mask = None if mask is None else mask.data_ptr()
            s.scratch, s.report = scratch.data_ptr(), report.data_ptr()
            s.color_weight, s.depth_weight, s.depth_error_max, s.damping = (float(color_weight), float(depth_weight),
                                                                              float(depth_error_max), float(damping))
            s.gt_channels_last = channels_last
            return s

        # per level: settings, projection, the step's state and the tile mask (the tensors are kept alive by `levels`)
        levels = []
        for sc in scales:
            if sc == 1:
                levels.append((rs, projection, state(projection, gt_color, gt_depth, mask, channels_last), tile_mask, None))
                continue
            cam = level_camera(camera, sc)
            lproj = cam.projection_matrix.to(device=dev, dtype=torch.float32).contiguous()
            targets = downsample_frame(gt_color, gt_depth.view(H, W), sc, mask, tile_mask)
            levels.append((self._settings(cam, dev, view, proj, campos), lproj, state(lproj, *targets[:3], 0), targets[3], targets))
        r = _lib.RtgPoseRobust()
        if robust is not None:
            r.kernel, r.color_delta, r.depth_delta = _lib.RTG_ROBUST_HUBER, float(color_delta), float(depth_delta)
        if exposure is not None:
            ab = _exposure_pair(exposure, dev, torch.float64)
            ex = _lib.RtgPoseExposure()
            ex.ab = ab.data_ptr()
        if depth == "expected":  # one entry point for every combination
            step = L.rtg_splat_pose_gn_step_expected
            extra = (C.byref(r), None if exposure is None else C.byref(ex), min_coverage)
        elif exposure is not None:
            step, extra = L.rtg_splat_pose_gn_step_exposure, (C.byref(r), C.byref(ex))
        elif robust is None:
            step, extra = L.rtg_splat_pose_gn_step, ()
        else:
            step, extra = L.rtg_splat_pose_gn_step_robust, (C.byref(r),)
        st = rasterizer._state(dev)
        for sc, (lrs, lproj, s, ltm, _), n in zip(scales, levels, level_iters):
            if len(levels) > 1:  # this level's projmatrix from the pose, on the device
                proj.copy_((pose.t() @ lproj.double()).float())
            mode = rasterizer.antialiased(True) if coarse_antialias and sc >= 2 else contextlib.nullcontext()
            for _ in range(n):
                for attempt in range(2):
                    with mode:
                        outs, saved, ins = _forward_native(lrs, g["xyz"], g["shs"], None, g["opacity"], g["scales"],
                                                           g["rotations"], None, ltm)
                    st.read(saved.pending, block=True)  # this forward's scan kernel; the capacity is raised on an overflow
                    if not saved.pending.overflow:
                        break
                    if attempt:
                        raise CapacityOverflow("PoseRefiner.refine_gn: the render overflowed the binning buffer twice")
                s.render, s.depth, s.hit_depth = outs[0].data_ptr(), outs[1].data_ptr(), outs[3].data_ptr()
                check(step(*_native_args(lrs, saved, ins, dev), C.byref(s), *extra,
                           C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), step.__name__)
        return (pose, report) if exposure is None else (pose, report, ab)

    def refine(self, camera, gaussian_data, gt_color, gt_depth, iters, lr_rot, lr_trans, color_weight=0.8, depth_weight=1.0,
               render_mask=None, tile_mask=None, exposure=None, lr_exposure=0.01):
        """`camera`: a reference-Camera-like object (world_view_transform, projection_matrix, FoVx, FoVy, image_height,
        image_width, cx, cy); its pose is the starting point and is not modified. `gaussian_data`: the dict Renderer.render
        takes (xyz, opacity, shs, scales, rotations); it is not differentiated. gt_color (H,W,3) or (3,H,W), gt_depth
        (H,W); render_mask (H,W) selects the colour / depth pixels of the loss, tile_mask the rendered 16x16 tiles.
        Adam (betas 0.9, 0.999, eps 1e-8) starts from zero moments on every call; lr_rot (radians) and lr_trans (map
        units) are its step sizes.
        `exposure`: None, or the starting exposure (a0, b0) of the frame as in `refine_gn`. The loss is then taken under
        it (l1_color_depth_loss(..., exposure=)), and (a, b) takes its own Adam step of size `lr_exposure` per iteration
        (optim.FusedAdam, one more launch; the pose step is unchanged). A third value is then returned: the estimate, a
        (2,) float32 CUDA tensor.

        Returns (W2C, parts): the refined world-to-camera pose, a (4, 4) float64 CUDA tensor, and the loss parts of the
        last iteration's render, [loss, colour L1, depth L1, n_depth] (l1_color_depth_loss; evaluated before its step)."""
        iters = int(iters)
        if iters < 1:
            raise ValueError("iters must be >= 1")
        dev, pose, projection, view, proj, campos, rs, g = self._setup(camera, gaussian_data, requires_grad=True)
        exp_avg = torch.zeros(6, dtype=torch.float32, device=dev)
        exp_avg_sq = torch.zeros(6, dtype=torch.float32, device=dev)

        st = RtgPoseAdam()
        st.pose, st.exp_avg, st.exp_avg_sq = pose.data_ptr(), exp_avg.data_ptr(), exp_avg_sq.data_ptr()
        st.projection, st.viewmatrix, st.projmatrix, st.campos = (t.data_ptr() for t in (projection, view, proj, campos))
        st.lr_trans, st.lr_rot = float(lr_trans), float(lr_rot)
        st.beta1, st.beta2, st.eps = 0.9, 0.999, 1e-8
        L = _lib.lib()
        parts = None
        ab = adam_ab = None
        if exposure is not None:
            ab = _exposure_pair(exposure, dev, torch.float32).requires_grad_(True)
            adam_ab = FusedAdam([ab], lr=float(lr_exposure), betas=(0.9, 0.999), eps=1e-8)
        with torch.enable_grad():
            for it in range(iters):
                for attempt in range(2):
                    out = rasterize_gaussians(g["xyz"], g["shs"], None, g["opacity"], g["scales"], g["rotations"], None,
                                              tile_mask, rs)
                    loss, parts = l1_color_depth_loss({"render": out[0], "depth": out[1], "depth_index_map": out[3]},
                                                      gt_color, gt_depth, render_mask, color_weight, depth_weight, exposure=ab)
                    try:
                        loss.backward()
                        break
                    except CapacityOverflow:  # this render was empty; the capacity has been raised: render it again
                        if attempt:
                            raise
                        if ab is not None:
                            ab.grad = None  # the empty render's exposure gradient is not this iteration's
                st.dL_dviewmatrix, st.dL_dprojmatrix, st.dL_dcampos = (
                    t.grad.data_ptr() if t.grad is not None else None for t in (view, proj, campos))
                st.step = it + 1
                check(L.rtg_pose_adam_step(C.byref(st), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                      "rtg_pose_adam_step")
                view.grad = proj.grad = campos.grad = None
                if ab is not None:
                    adam_ab.step()
                    ab.grad = None
        return (pose, parts) if exposure is None else (pose, parts, ab.detach())
