"""Keyframe poses and exposures refined together with the map.

`KeyframeTable` holds, per keyframe, what the mapping step needs to move the keyframe's camera and brightness as well as the
Gaussians, as MonoGS-style Gaussian-splatting SLAM systems do:
  - the world-to-camera pose W2C in double on the device, and the three camera tensors the rasterizer reads (viewmatrix,
    projmatrix, campos) as leaves that require grad. `camera(k)` wraps them in the Camera-like object `Renderer.render`
    takes, so the backward of a render at that camera fills their gradients (rtg_splat_backward_camera, also under
    `rasterizer.visible_rows_only()`, whose per-Gaussian rows `mapoptim.MapOptimizer.step` takes);
  - optionally an exposure (a, b) leaf, the affine brightness e^a C + b of `tracking.apply_exposure`, for
    `loss.mapping_loss(..., exposure=table.exposure(k))`;
  - the keyframe's own Adam state: the pose moments (2, 6) with their step count, and a `optim.FusedAdam` over the exposure.

`step(k)` after the backward takes one device pose step (rtg_pose_adam_step) and one exposure step (rtg_adam_step) and
drops the gradients. Which keyframes to refine, when, and at what learning rates is SLAM policy and is left to the caller.

Gauge freedom: with a free map, the map and every pose can move together by one rigid motion, and the map's colours and
every exposure by one affine brightness change, without changing the loss. Fix at least one keyframe's pose (`fix_pose`),
and one keyframe's exposure (`fix_exposure`) if exposures are refined; otherwise the whole solution can slide.
The normal term of the mapping loss compares with a world-space target (`normal_map_w`) that is not rotated with a refined
pose; `normal_weight` is 0 in every shipped configuration."""
from __future__ import annotations

import ctypes as C
import types

import torch

from . import _lib
from ._lib import RtgPoseAdam, check
from .optim import FusedAdam
from .tracking import _exposure_pair, camera_tensors


class KeyframeTable:
    """Per-keyframe camera tensors, exposures and their Adam states. `lr_rot` (radians) and `lr_trans` (map units) are the
    pose step sizes of rtg_pose_adam_step, `lr_exposure` the step size of (a, b); `betas` and `eps` are Adam's for both."""

    def __init__(self, lr_rot, lr_trans, lr_exposure, betas=(0.9, 0.999), eps=1e-8):
        b1, b2 = (float(b) for b in betas)
        if lr_rot < 0 or lr_trans < 0 or lr_exposure < 0 or eps < 0 or not (0.0 <= b1 < 1.0) or not (0.0 <= b2 < 1.0):
            raise ValueError("KeyframeTable: invalid hyper-parameter")
        self.lr_rot, self.lr_trans, self.lr_exposure = float(lr_rot), float(lr_trans), float(lr_exposure)
        self.betas, self.eps = (b1, b2), float(eps)
        self._kf = []

    def __len__(self):
        return len(self._kf)

    def add(self, camera, exposure=None, fix_pose=False, fix_exposure=False):
        """Adds a keyframe and returns its index k. `camera`: a reference-Camera-like object (world_view_transform,
        projection_matrix, FoVx, FoVy, image_height, image_width, cx, cy), as `tracking.PoseRefiner` takes; its pose is the
        starting point and is copied. `exposure`: None (the keyframe has no exposure), or the starting (a, b), a pair of
        floats or a 2-element tensor, e.g. the estimate of `PoseRefiner.refine_gn(exposure=)` or (0, 0). `fix_pose` /
        `fix_exposure`: the pose / exposure is never stepped (its tensors then do not require grad)."""
        vm = camera.world_view_transform.detach()
        dev = vm.device if vm.is_cuda else torch.device("cuda", torch.cuda.current_device())
        pose = vm.to(device=dev, dtype=torch.float64).t().contiguous()          # W2C, row-major, double
        projection = camera.projection_matrix.detach().to(device=dev, dtype=torch.float32).contiguous()
        view, proj, campos = (t.requires_grad_(not fix_pose) for t in camera_tensors(pose, projection))
        ab = adam = None
        if exposure is not None:
            ab = _exposure_pair(exposure, dev, torch.float32).requires_grad_(not fix_exposure)
            if not fix_exposure:
                adam = FusedAdam([ab], lr=self.lr_exposure, betas=self.betas, eps=self.eps)
        cam = types.SimpleNamespace(world_view_transform=view, full_proj_transform=proj, camera_center=campos,
                                    projection_matrix=projection, FoVx=float(camera.FoVx), FoVy=float(camera.FoVy),
                                    image_height=int(camera.image_height), image_width=int(camera.image_width),
                                    cx=float(camera.cx), cy=float(camera.cy))
        self._kf.append(types.SimpleNamespace(pose=pose, projection=projection, view=view, proj=proj, campos=campos, camera=cam,
                                              moments=torch.zeros((2, 6), dtype=torch.float32, device=dev), step=0, exposure=ab,
                                              adam=adam, fix_pose=bool(fix_pose), fix_exposure=bool(fix_exposure)))
        return len(self._kf) - 1

    def camera(self, k):
        """The Camera-like object `Renderer.render` takes for keyframe k: world_view_transform, full_proj_transform and
        camera_center are the keyframe's leaves (rewritten in place by `step` and `set_pose`), with its intrinsics."""
        return self._kf[k].camera

    def exposure(self, k):
        """Keyframe k's (2,) float32 exposure leaf (a, b) for `loss.mapping_loss(..., exposure=)`, or None."""
        return self._kf[k].exposure

    def step_count(self, k):
        """How many pose steps keyframe k has taken since it was added or its pose was last set."""
        return self._kf[k].step

    def moments(self, k):
        """Keyframe k's pose moments (2, 6): exp_avg and exp_avg_sq of rtg_pose_adam_step (rho then phi)."""
        return self._kf[k].moments

    def step(self, k):
        """After a backward through `camera(k)` / `exposure(k)`: one rtg_pose_adam_step of keyframe k's pose from its camera
        gradients (a missing gradient counts as zero) unless the pose is fixed, one FusedAdam step of its exposure unless it is
        fixed or has no gradient, then drops those gradients. Every other keyframe is left as it is."""
        kf = self._kf[k]
        dev = kf.pose.device
        if not kf.fix_pose:
            kf.step += 1
            st = RtgPoseAdam()
            st.pose, st.projection = kf.pose.data_ptr(), kf.projection.data_ptr()
            st.exp_avg, st.exp_avg_sq = kf.moments[0].data_ptr(), kf.moments[1].data_ptr()
            st.viewmatrix, st.projmatrix, st.campos = (t.data_ptr() for t in (kf.view, kf.proj, kf.campos))
            st.dL_dviewmatrix, st.dL_dprojmatrix, st.dL_dcampos = (
                t.grad.data_ptr() if t.grad is not None else None for t in (kf.view, kf.proj, kf.campos))
            st.lr_trans, st.lr_rot = self.lr_trans, self.lr_rot
            st.beta1, st.beta2 = self.betas
            st.eps, st.step = self.eps, kf.step
            check(_lib.lib().rtg_pose_adam_step(C.byref(st), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                  "rtg_pose_adam_step")
        if kf.adam is not None:
            kf.adam.step()
        kf.view.grad = kf.proj.grad = kf.campos.grad = None
        if kf.exposure is not None:
            kf.exposure.grad = None

    def pose(self, k):
        """Keyframe k's refined W2C, a (4, 4) float64 CUDA tensor (the table's own: copy it to keep a snapshot)."""
        return self._kf[k].pose

    def poses(self):
        """Every keyframe's W2C, (K, 4, 4) float64."""
        return torch.stack([kf.pose for kf in self._kf])

    def set_pose(self, k, w2c):
        """Overwrites keyframe k's pose with the W2C `w2c` (4, 4), e.g. after a loop closure, rewrites its camera tensors and
        resets its pose moments and step count."""
        kf = self._kf[k]
        w2c = torch.as_tensor(w2c)
        if w2c.shape != (4, 4):
            raise ValueError("w2c must be (4, 4)")
        with torch.no_grad():
            kf.pose.copy_(w2c.to(device=kf.pose.device, dtype=torch.float64))
            for t, v in zip((kf.view, kf.proj, kf.campos), camera_tensors(kf.pose, kf.projection)):
                t.copy_(v)
            kf.moments.zero_()
        kf.step = 0
