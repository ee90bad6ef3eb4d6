"""Per-Gaussian feature maps: C channels per Gaussian composited with one rasterizer forward's blend weights.

`rasterize_features` renders the frame once through the rasterizer (the eight outputs and their autograd exactly as
GaussianRasterizer gives them) and replays that forward's blending for a (P, C) feature tensor (rtg_splat_features):

    feature_map[c, p] = sum_g w(p, g) features[g, c],     w = alpha T, the forward's colour weight.

By default the weights are held fixed: the feature map's only gradient is dL/dfeatures[g, c] = sum_p w(p, g)
dL/dfeature_map[c, p] (rtg_splat_features_backward); a loss on it moves the features, not the Gaussians or the camera.
With `weight_grad=True` the map is differentiated through its weights as well (rtg_splat_features_backward_geometry):
the loss also reaches the means, opacities, scales and rotations (or cov3D_precomp) and the settings' camera tensors, as
a colour loss does. Expected depth is then the map of F = (z_view, 1): depth = map[0] / map[1]. Semantic logits,
instance embeddings, confidences or any other per-Gaussian quantity of up to RTG_FEATURES_MAX channels render in one call.
No parameter array is read by the replay; there is no background term (T_map holds the remainder).
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib, rasterizer
from ._lib import check

MAX_CHANNELS = _lib.RTG_FEATURES_MAX


def _check_features(features, means3D):
    """TypeError / ValueError before any CUDA work."""
    if not torch.is_tensor(features):
        raise TypeError(f"features must be a torch.Tensor, got {type(features).__name__}")
    if features.dtype != torch.float32:
        raise TypeError(f"features must be float32, got {features.dtype}")
    if not torch.is_tensor(means3D):
        raise TypeError(f"means3D must be a torch.Tensor, got {type(means3D).__name__}")
    if features.dim() != 2 or means3D.dim() < 1 or features.size(0) != means3D.size(0):
        raise ValueError(f"features must have shape (P, C) with P = {means3D.size(0) if means3D.dim() else '?'}, "
                         f"got {tuple(features.shape)}")
    if not 1 <= features.size(1) <= MAX_CHANNELS:
        raise ValueError(f"features must have 1..{MAX_CHANNELS} channels, got {features.size(1)}")
    if not features.is_cuda or not means3D.is_cuda:
        raise TypeError(f"features and means3D must be CUDA tensors, got them on {features.device} and {means3D.device}")
    if features.device != means3D.device:
        raise ValueError(f"features is on {features.device}, means3D on {means3D.device}")


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _render_map(features, saved, raster_settings):
    dev = features.device
    P, Cn = features.shape
    H, W = int(raster_settings.image_height), int(raster_settings.image_width)
    out = torch.empty((Cn, H, W), dtype=torch.float32, device=dev)
    view, keep = rasterizer._make_view(raster_settings, dev, saved.antialiased)
    check(_lib.lib().rtg_splat_features(C.byref(view), P, C.c_void_p(saved.geom), C.c_void_p(saved.img),
                                        C.c_void_p(saved.bin), saved.r_cap, C.c_void_p(saved.counters), Cn,
                                        C.c_void_p(features.data_ptr()), C.c_void_p(out.data_ptr()), _stream(dev)),
          "rtg_splat_features")
    return out


def _check_not_overflowed(saved, dev):
    st = rasterizer._state(dev)
    if not saved.pending.done:  # a forward that did not wait for its count: it has arrived by now
        st.read(saved.pending, block=True)
    if saved.pending.overflow:
        raise rasterizer.CapacityOverflow(
            f"rasterize_features: this frame needed {saved.pending.num_rendered} (Gaussian, tile) instances but its "
            f"binning buffer held {saved.pending.r_cap}; it was rendered empty and has no feature gradient. The capacity "
            "has been raised: render it again (set_capacity_checks('sync') makes every forward check its own count).")


def _feature_grad(g, saved, rs, P, Cn):
    dev = g.device
    grad = torch.empty((P, Cn), dtype=torch.float32, device=dev)
    view, keep = rasterizer._make_view(rs, dev, saved.antialiased)
    check(_lib.lib().rtg_splat_features_backward(C.byref(view), P, C.c_void_p(saved.geom), C.c_void_p(saved.img),
                                                 C.c_void_p(saved.bin), saved.r_cap, C.c_void_p(saved.counters), Cn,
                                                 C.c_void_p(g.data_ptr()), C.c_void_p(grad.data_ptr()), _stream(dev)),
          "rtg_splat_features_backward")
    return grad


class _RenderFeatures(torch.autograd.Function):
    """The feature map of a finished forward (`saved`, its _Saved state); differentiable in `features` only."""

    @staticmethod
    def forward(ctx, features, saved, raster_settings):
        ctx.native, ctx.raster_settings, ctx.shape = saved, raster_settings, tuple(features.shape)
        return _render_map(features, saved, raster_settings)

    @staticmethod
    def backward(ctx, grad_map):
        saved, rs = ctx.native, ctx.raster_settings
        P, Cn = ctx.shape
        _check_not_overflowed(saved, grad_map.device)
        g = grad_map.contiguous()  # feature_map.sum() delivers a stride-0 view
        return _feature_grad(g, saved, rs, P, Cn), None, None


class _RenderFeaturesWeighted(torch.autograd.Function):
    """The feature map of a finished forward, differentiable in `features` and, through its blend weights, in the
    Gaussians' geometry (means3D, opacities, scales, rotations or cov3D_precomp) and -- passed only when one of them
    requires grad, as rasterize_gaussians does -- the settings' viewmatrix / projmatrix / campos. Its gradients add to the
    rasterizer node's own through autograd."""

    @staticmethod
    def forward(ctx, features, saved, raster_settings, radii, means3D, opacities, scales, rotations, cov3D_precomp,
                viewmatrix=None, projmatrix=None, campos=None):
        ctx.native, ctx.raster_settings, ctx.shape = saved, raster_settings, tuple(features.shape)
        ctx.param_shapes = tuple(None if t is None else t.shape for t in (means3D, opacities, scales, rotations, cov3D_precomp))
        ctx.camera_shapes = tuple(None if t is None else t.shape for t in (viewmatrix, projmatrix, campos))
        dev = features.device
        geo = [rasterizer._f32_cuda(t, n, dev) for t, n in ((means3D, "means3D"), (scales, "scales"),
                                                           (rotations, "rotations"), (cov3D_precomp, "cov3D_precomp"))]
        e = torch.empty(0, device=dev)
        ctx.provided = tuple(t is not None for t in geo)
        ctx.save_for_backward(features, radii, *[e if t is None else t for t in geo])
        return _render_map(features, saved, raster_settings)

    @staticmethod
    def backward(ctx, grad_map):
        saved, rs = ctx.native, ctx.raster_settings
        P, Cn = ctx.shape
        dev = grad_map.device
        features, radii, *geo = ctx.saved_tensors
        means3D, scales, rotations, cov3D = [t if has else None for t, has in zip(geo, ctx.provided)]
        needs = ctx.needs_input_grad
        camera = any(needs[9:])  # only present when the settings' camera tensors were passed
        _check_not_overflowed(saved, dev)
        g = grad_map.contiguous()  # feature_map.sum() delivers a stride-0 view
        grad_F = _feature_grad(g, saved, rs, P, Cn) if needs[0] else None
        gaussians = any(needs[4:9])
        if not gaussians and not camera:
            return (grad_F,) + (None,) * (len(needs) - 1)
        if rasterizer._GRAD_RECORD_HOOK[0] is not None:
            raise RuntimeError("rasterize_features: the weight gradient is not available with a gradient-record exchange "
                               "hook (set_grad_record_hook, tile-sharded frames)")
        visible = rasterizer._VISIBLE_ROWS_ONLY[0]
        # the rasterizer's condition for its pose-only pass: a frozen map, only the camera is differentiated
        pose_only = camera and rasterizer._GRAD_BUFFERS[0] is None and not visible and not gaussians
        f32 = dict(dtype=torch.float32, device=dev)
        shapes = ctx.param_shapes
        if pose_only:
            g_means = g_opac = g_scales = g_rot = g_cov = None
        else:
            g_means, g_opac = torch.empty((P, 3), **f32), torch.empty((P, 1), **f32)
            g_scales = torch.empty((P, 3), **f32) if scales is not None else None
            g_rot = torch.empty((P, 4), **f32) if rotations is not None else None
            g_cov = torch.empty((P, 6), **f32) if cov3D is not None else None
        g_cam = torch.zeros((35,), **f32) if camera else None  # (view 16, proj 16, campos 3)
        L = _lib.lib()
        cam_scratch = (torch.empty((int(L.rtg_splat_camera_scratch_bytes(P)),), dtype=torch.uint8, device=dev)
                       if camera else None)
        scratch = rasterizer._state(dev).get_scratch(P)
        ptr = rasterizer._ptr
        view, keep = rasterizer._make_view(rs, dev, saved.antialiased)
        if P > 0:  # no Gaussian: empty gradients and a zero camera gradient
            check(L.rtg_splat_features_backward_geometry(
                C.byref(view), P, ptr(means3D), ptr(scales), ptr(rotations), ptr(cov3D), ptr(radii), C.c_void_p(saved.geom),
                C.c_void_p(saved.img), C.c_void_p(saved.bin), saved.r_cap, C.c_void_p(saved.counters), Cn, ptr(features),
                ptr(g), ptr(scratch), ptr(g_means), ptr(g_opac), ptr(g_scales), ptr(g_rot), ptr(g_cov), 1 if visible else 0,
                ptr(g_cam), ptr(cam_scratch), _stream(dev)), "rtg_splat_features_backward_geometry")
        grads = tuple(None if (t is None or s is None) else t.view(s)
                      for t, s in zip((g_means, g_opac, g_scales, g_rot, g_cov), shapes))
        out = (grad_F, None, None, None) + grads
        if len(needs) == 9:
            return out
        cam = (slice(0, 16), slice(16, 32), slice(32, 35))
        return out + tuple(g_cam[c].reshape(s) if n else None for c, s, n in zip(cam, ctx.camera_shapes, needs[9:]))


def rasterize_features(raster_settings, means3D, opacities, features, shs=None, colors_precomp=None, scales=None,
                       rotations=None, cov3D_precomp=None, tile_mask=None, weight_grad=False):
    """One rasterizer forward and a C-channel map of per-Gaussian `features` composited with its blend weights.

    Inputs as GaussianRasterizer takes them, plus `features`: (P, C) float32 on the Gaussians' device, 1 <= C <= 128.
    Returns (outputs, feature_map):
      outputs      the eight tensors of GaussianRasterizer on the same inputs, with the same autograd (Gaussian, camera
                   and T_map gradients; `antialiased()`, `grad_buffers`, `visible_rows_only` and the capacity checks apply);
      feature_map  (C, H, W) float32, sum_g alpha T features[g, c] over the pairs the forward blends; 0 on masked-out and
                   empty tiles and where the forward overflowed. Its gradient goes to `features` only, unless
                   `weight_grad`.
    weight_grad  (bool) the feature map is also differentiated through its blend weights: its gradient reaches means3D,
                 opacities, scales and rotations (or cov3D_precomp) and -- when one of them requires grad -- the settings'
                 viewmatrix / projmatrix / campos, and autograd adds it to the rasterizer's own gradients. Honours
                 `visible_rows_only()` and the forward's antialiased mode; with only camera tensors requiring grad it
                 computes the camera gradient alone. Not available with a gradient-record exchange hook (RuntimeError).
    An overflowed forward is reported as for the eight outputs (set_capacity_checks); the feature backward of an
    overflowed forward raises CapacityOverflow."""
    if not isinstance(weight_grad, bool):
        raise TypeError(f"weight_grad must be a bool, got {type(weight_grad).__name__}")
    _check_features(features, means3D)
    saved = []
    with rasterizer.keep_saved(saved):
        outputs = rasterizer.GaussianRasterizer(raster_settings)(means3D, opacities, shs=shs, colors_precomp=colors_precomp,
                                                                  scales=scales, rotations=rotations,
                                                                  cov3D_precomp=cov3D_precomp, tile_mask=tile_mask)
    if not weight_grad:
        return outputs, _RenderFeatures.apply(features.contiguous(), saved[-1], raster_settings)
    cam = ()
    rs = raster_settings
    if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in
                                       (rs.viewmatrix, rs.projmatrix, rs.campos)):
        cam = (rs.viewmatrix, rs.projmatrix, rs.campos)
    return outputs, _RenderFeaturesWeighted.apply(features.contiguous(), saved[-1], raster_settings, outputs[7], means3D,
                                                  opacities, scales, rotations, cov3D_precomp, *cam)
