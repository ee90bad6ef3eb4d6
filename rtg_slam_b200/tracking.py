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

When to track with it (every frame, after ICP, on keyframes only) is SLAM policy and is left to the caller."""
from __future__ import annotations

import ctypes as C
import math

import torch

from . import _lib
from ._lib import RtgPoseAdam, check
from .loss import l1_color_depth_loss
from .rasterizer import CapacityOverflow, GaussianRasterizationSettings, rasterize_gaussians
from .render import Renderer


class PoseRefiner:
    """Refines a world-to-camera pose against a frozen Gaussian map. `args` is the bag `render.Renderer` takes."""

    def __init__(self, args):
        self._renderer = Renderer(args)  # rasterizer settings exactly as Renderer.render makes them

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
        r = self._renderer
        dev = gaussian_data["xyz"].device
        iters = int(iters)
        if iters < 1:
            raise ValueError("iters must be >= 1")
        vm0 = camera.world_view_transform.detach().to(device=dev, dtype=torch.float64)
        pose = vm0.t().contiguous()                                   # W2C, row-major, double
        projection = camera.projection_matrix.detach().to(device=dev, dtype=torch.float32).contiguous()
        view = pose.t().float().contiguous().requires_grad_(True)
        proj = (pose.t() @ projection.double()).float().contiguous().requires_grad_(True)
        campos = (-(pose[:3, :3].t() @ pose[:3, 3])).float().contiguous().requires_grad_(True)
        exp_avg = torch.zeros(6, dtype=torch.float32, device=dev)
        exp_avg_sq = torch.zeros(6, dtype=torch.float32, device=dev)

        rs = GaussianRasterizationSettings(
            image_height=int(camera.image_height), image_width=int(camera.image_width),
            tanfovx=math.tan(camera.FoVx * 0.5), tanfovy=math.tan(camera.FoVy * 0.5), bg=r.bg_color.to(dev),
            scale_modifier=r.scaling_modifier, viewmatrix=view, projmatrix=proj, sh_degree=r.active_sh_degree, campos=campos,
            opaque_threshold=r.renderer_opaque_threshold, depth_threshold=r.renderer_depth_threshold,
            normal_threshold=r.renderer_normal_threshold, color_sigma=r.color_sigma, prefiltered=False, debug=False,
            cx=camera.cx, cy=camera.cy, T_threshold=0.0001)
        g = {k: gaussian_data[k].detach() for k in ("xyz", "opacity", "shs", "scales", "rotations")}

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
