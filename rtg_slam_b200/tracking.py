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
returns those tangent images themselves.

When to track with either (every frame, after ICP, on keyframes only) is SLAM policy and is left to the caller."""
from __future__ import annotations

import ctypes as C
import math

import torch

from . import _lib, rasterizer
from ._lib import RtgPoseAdam, RtgPoseGN, check
from .loss import l1_color_depth_loss
from .rasterizer import CapacityOverflow, GaussianRasterizationSettings, _forward_native, _make_view, rasterize_gaussians
from .render import Renderer


def _native_args(rs, saved, ins, dev):
    """(view, P, M, the six Gaussian inputs, the three workspaces, R_cap, counters) of one rasterizer forward, the head of
    both tangent entry points' argument lists. The view struct holds the settings' camera tensors by pointer."""
    means3D, sh, colors_precomp, scales, rotations, cov3D_precomp = ins
    view, keep = _make_view(rs, dev)
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    return (C.byref(view), int(means3D.shape[0]), int(sh.shape[1]) if sh is not None else 0, p(means3D), p(sh), p(colors_precomp),
            p(scales), p(rotations), p(cov3D_precomp), C.c_void_p(saved.geom), C.c_void_p(saved.img), C.c_void_p(saved.bin),
            saved.r_cap, C.c_void_p(saved.counters))


def pose_jacobian(raster_settings, means3D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                  cov3D_precomp=None, tile_mask=None):
    """One rasterizer forward at the settings' camera and the forward-mode tangents of its render along the six directions
    of a left twist xi = (rho, phi) of the pose (rtg_splat_pose_tangents). Returns (outputs, J): the forward's eight outputs
    as GaussianRasterizer returns them, and J (6, 4, H, W) float32, J[k] = d(colour r, g, b, depth) / d xi_k. Inputs as
    GaussianRasterizer takes them; nothing is differentiated by autograd."""
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
        check(L.rtg_splat_pose_tangents(*_native_args(raster_settings, saved, ins, dev), C.c_void_p(outs[3].data_ptr()),
                                        C.c_void_p(scratch.data_ptr()), C.c_void_p(J.data_ptr()),
                                        C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "rtg_splat_pose_tangents")
        return outs, J


class PoseRefiner:
    """Refines a world-to-camera pose against a frozen Gaussian map. `args` is the bag `render.Renderer` takes."""

    def __init__(self, args):
        self._renderer = Renderer(args)  # rasterizer settings exactly as Renderer.render makes them

    def _setup(self, camera, gaussian_data, requires_grad):
        """The double pose W2C, the projection, the three camera tensors the rasterizer reads (rewritten in place by the
        device pose steps), the rasterizer settings over them and the detached map."""
        r = self._renderer
        dev = gaussian_data["xyz"].device
        vm0 = camera.world_view_transform.detach().to(device=dev, dtype=torch.float64)
        pose = vm0.t().contiguous()                                   # W2C, row-major, double
        projection = camera.projection_matrix.detach().to(device=dev, dtype=torch.float32).contiguous()
        view = pose.t().float().contiguous().requires_grad_(requires_grad)
        proj = (pose.t() @ projection.double()).float().contiguous().requires_grad_(requires_grad)
        campos = (-(pose[:3, :3].t() @ pose[:3, 3])).float().contiguous().requires_grad_(requires_grad)
        rs = GaussianRasterizationSettings(
            image_height=int(camera.image_height), image_width=int(camera.image_width),
            tanfovx=math.tan(camera.FoVx * 0.5), tanfovy=math.tan(camera.FoVy * 0.5), bg=r.bg_color.to(dev),
            scale_modifier=r.scaling_modifier, viewmatrix=view, projmatrix=proj, sh_degree=r.active_sh_degree, campos=campos,
            opaque_threshold=r.renderer_opaque_threshold, depth_threshold=r.renderer_depth_threshold,
            normal_threshold=r.renderer_normal_threshold, color_sigma=r.color_sigma, prefiltered=False, debug=False,
            cx=camera.cx, cy=camera.cy, T_threshold=0.0001)
        g = {k: gaussian_data[k].detach() for k in ("xyz", "opacity", "shs", "scales", "rotations")}
        return dev, pose, projection, view, proj, campos, rs, g

    def refine_gn(self, camera, gaussian_data, gt_color, gt_depth, iters, damping=1e-4, color_weight=0.8, depth_weight=1.0,
                  render_mask=None, tile_mask=None, depth_error_max=0.1):
        """Gauss-Newton refinement of the pose on the squared colour + depth residuals (rtg_splat_pose_gn_step): per
        iteration the rasterizer forward, then the forward-mode tangents of the render along the six twist directions, the
        normal equations over rtg_loss_l1's pixel selection, the damped solve (H + damping * trace(H) * I) and
        W2C <- exp(xi^) W2C, all on the device. No autograd is involved and nothing is read back inside the loop, except
        that each iteration waits for its forward's scan kernel: an iteration whose render overflowed the binning buffer is
        rendered again (with the capacity raised), keeping the pose refined so far.

        Arguments as in `refine`; `damping` scales the trace added to the diagonal. Returns (W2C, report): the refined pose,
        a (4, 4) float64 CUDA tensor, and the last step's report, a float64 CUDA tensor [E, E_colour, E_depth, N_c, N_d,
        |rho|, |phi|, status] (E evaluated before that step; status 0 ok, 1 singular system, 2 no selected pixel,
        3 overflowed forward -- the pose is then left unchanged)."""
        iters = int(iters)
        if iters < 1:
            raise ValueError("iters must be >= 1")
        dev, pose, projection, view, proj, campos, rs, g = self._setup(camera, gaussian_data, requires_grad=False)
        H, W = int(rs.image_height), int(rs.image_width)
        gt_color, gt_depth = gt_color.detach().contiguous(), gt_depth.detach().contiguous()
        if gt_color.shape == (H, W, 3):
            channels_last = 1
        elif gt_color.shape == (3, H, W):
            channels_last = 0
        else:
            raise ValueError("gt_color must be (H,W,3) or (3,H,W)")
        if gt_depth.numel() != H * W:
            raise ValueError("gt_depth must have H*W elements")
        for name, t in (("gt_color", gt_color), ("gt_depth", gt_depth)):
            if not t.is_cuda or t.dtype != torch.float32:
                raise TypeError(f"{name} must be a CUDA float32 tensor")
        mask = None
        if render_mask is not None:
            mask = render_mask.detach().to(torch.uint8).contiguous()
            if mask.numel() != H * W:
                raise ValueError("render_mask must have H*W elements")
        P = int(g["xyz"].shape[0])
        L = _lib.lib()
        scratch = torch.empty((int(L.rtg_splat_pose_gn_scratch_bytes(P, H, W)),), dtype=torch.uint8, device=dev)
        report = torch.zeros(_lib.RTG_POSE_GN_REPORT_LEN, dtype=torch.float64, device=dev)
        s = RtgPoseGN()
        s.pose, s.projection, s.viewmatrix, s.projmatrix, s.campos = (t.data_ptr() for t in (pose, projection, view, proj, campos))
        s.gt_color, s.gt_depth = gt_color.data_ptr(), gt_depth.data_ptr()
        s.render_mask = None if mask is None else mask.data_ptr()
        s.scratch, s.report = scratch.data_ptr(), report.data_ptr()
        s.color_weight, s.depth_weight, s.depth_error_max, s.damping = (float(color_weight), float(depth_weight),
                                                                          float(depth_error_max), float(damping))
        s.gt_channels_last = channels_last
        st = rasterizer._state(dev)
        for _ in range(iters):
            for attempt in range(2):
                outs, saved, ins = _forward_native(rs, g["xyz"], g["shs"], None, g["opacity"], g["scales"], g["rotations"], None,
                                                   tile_mask)
                st.read(saved.pending, block=True)  # this forward's scan kernel; the capacity is raised on an overflow
                if not saved.pending.overflow:
                    break
                if attempt:
                    raise CapacityOverflow("PoseRefiner.refine_gn: the render overflowed the binning buffer twice")
            s.render, s.depth, s.hit_depth = outs[0].data_ptr(), outs[1].data_ptr(), outs[3].data_ptr()
            check(L.rtg_splat_pose_gn_step(*_native_args(rs, saved, ins, dev), C.byref(s),
                                           C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "rtg_splat_pose_gn_step")
        return pose, report

    def refine(self, camera, gaussian_data, gt_color, gt_depth, iters, lr_rot, lr_trans, color_weight=0.8, depth_weight=1.0,
               render_mask=None, tile_mask=None):
        """`camera`: a reference-Camera-like object (world_view_transform, projection_matrix, FoVx, FoVy, image_height,
        image_width, cx, cy); its pose is the starting point and is not modified. `gaussian_data`: the dict Renderer.render
        takes (xyz, opacity, shs, scales, rotations); it is not differentiated. gt_color (H,W,3) or (3,H,W), gt_depth
        (H,W); render_mask (H,W) selects the colour / depth pixels of the loss, tile_mask the rendered 16x16 tiles.
        Adam (betas 0.9, 0.999, eps 1e-8) starts from zero moments on every call; lr_rot (radians) and lr_trans (map
        units) are its step sizes.

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
        with torch.enable_grad():
            for it in range(iters):
                for attempt in range(2):
                    out = rasterize_gaussians(g["xyz"], g["shs"], None, g["opacity"], g["scales"], g["rotations"], None,
                                              tile_mask, rs)
                    loss, parts = l1_color_depth_loss({"render": out[0], "depth": out[1], "depth_index_map": out[3]},
                                                      gt_color, gt_depth, render_mask, color_weight, depth_weight)
                    try:
                        loss.backward()
                        break
                    except CapacityOverflow:  # this render was empty; the capacity has been raised: render it again
                        if attempt:
                            raise
                st.dL_dviewmatrix, st.dL_dprojmatrix, st.dL_dcampos = (
                    t.grad.data_ptr() if t.grad is not None else None for t in (view, proj, campos))
                st.step = it + 1
                check(L.rtg_pose_adam_step(C.byref(st), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                      "rtg_pose_adam_step")
                view.grad = proj.grad = campos.grad = None
        return pose, parts
