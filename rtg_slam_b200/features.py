"""Per-Gaussian feature maps: C channels per Gaussian composited with one rasterizer forward's blend weights.

`rasterize_features` renders the frame once through the rasterizer (the eight outputs and their autograd exactly as
GaussianRasterizer gives them) and replays that forward's blending for a (P, C) feature tensor (rtg_splat_features):

    feature_map[c, p] = sum_g w(p, g) features[g, c],     w = alpha T, the forward's colour weight.

The weights are held fixed: the feature map's only gradient is dL/dfeatures[g, c] = sum_p w(p, g) dL/dfeature_map[c, p]
(rtg_splat_features_backward); a loss on it moves the features, not the Gaussians or the camera. Semantic logits,
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


class _RenderFeatures(torch.autograd.Function):
    """The feature map of a finished forward (`saved`, its _Saved state); differentiable in `features` only."""

    @staticmethod
    def forward(ctx, features, saved, raster_settings):
        dev = features.device
        P, Cn = features.shape
        H, W = int(raster_settings.image_height), int(raster_settings.image_width)
        out = torch.empty((Cn, H, W), dtype=torch.float32, device=dev)
        view, keep = rasterizer._make_view(raster_settings, dev, saved.antialiased)
        check(_lib.lib().rtg_splat_features(C.byref(view), P, C.c_void_p(saved.geom), C.c_void_p(saved.img),
                                            C.c_void_p(saved.bin), saved.r_cap, C.c_void_p(saved.counters), Cn,
                                            C.c_void_p(features.data_ptr()), C.c_void_p(out.data_ptr()), _stream(dev)),
              "rtg_splat_features")
        ctx.native, ctx.raster_settings, ctx.shape = saved, raster_settings, (P, Cn)
        return out

    @staticmethod
    def backward(ctx, grad_map):
        saved, rs = ctx.native, ctx.raster_settings
        P, Cn = ctx.shape
        dev = grad_map.device
        st = rasterizer._state(dev)
        if not saved.pending.done:  # a forward that did not wait for its count: it has arrived by now
            st.read(saved.pending, block=True)
        if saved.pending.overflow:
            raise rasterizer.CapacityOverflow(
                f"rasterize_features: this frame needed {saved.pending.num_rendered} (Gaussian, tile) instances but its "
                f"binning buffer held {saved.pending.r_cap}; it was rendered empty and has no feature gradient. The capacity "
                "has been raised: render it again (set_capacity_checks('sync') makes every forward check its own count).")
        g = grad_map.contiguous()  # feature_map.sum() delivers a stride-0 view
        grad = torch.empty((P, Cn), dtype=torch.float32, device=dev)
        view, keep = rasterizer._make_view(rs, dev, saved.antialiased)
        check(_lib.lib().rtg_splat_features_backward(C.byref(view), P, C.c_void_p(saved.geom), C.c_void_p(saved.img),
                                                     C.c_void_p(saved.bin), saved.r_cap, C.c_void_p(saved.counters), Cn,
                                                     C.c_void_p(g.data_ptr()), C.c_void_p(grad.data_ptr()), _stream(dev)),
              "rtg_splat_features_backward")
        return grad, None, None


def rasterize_features(raster_settings, means3D, opacities, features, shs=None, colors_precomp=None, scales=None,
                       rotations=None, cov3D_precomp=None, tile_mask=None):
    """One rasterizer forward and a C-channel map of per-Gaussian `features` composited with its blend weights.

    Inputs as GaussianRasterizer takes them, plus `features`: (P, C) float32 on the Gaussians' device, 1 <= C <= 128.
    Returns (outputs, feature_map):
      outputs      the eight tensors of GaussianRasterizer on the same inputs, with the same autograd (Gaussian, camera
                   and T_map gradients; `antialiased()`, `grad_buffers`, `visible_rows_only` and the capacity checks apply);
      feature_map  (C, H, W) float32, sum_g alpha T features[g, c] over the pairs the forward blends; 0 on masked-out and
                   empty tiles and where the forward overflowed. Its gradient goes to `features` only.
    An overflowed forward is reported as for the eight outputs (set_capacity_checks); the feature backward of an
    overflowed forward raises CapacityOverflow."""
    _check_features(features, means3D)
    saved = []
    with rasterizer.keep_saved(saved):
        outputs = rasterizer.GaussianRasterizer(raster_settings)(means3D, opacities, shs=shs, colors_precomp=colors_precomp,
                                                                  scales=scales, rotations=rotations,
                                                                  cov3D_precomp=cov3D_precomp, tile_mask=tile_mask)
    return outputs, _RenderFeatures.apply(features.contiguous(), saved[-1], raster_settings)
