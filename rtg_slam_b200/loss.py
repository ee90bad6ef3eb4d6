"""Fused mapping loss: masked L1 on the rendered colour + L1 on the rendered depth, with gradients.

Drop-in for the colour / depth terms of `Mapping.loss_update` (SLAM/multiprocess/mapper.py:402-431,444-451; `l1_loss` of
utils/loss_utils.py:27-31). The reference evaluates them with ~25 eager kernels (boolean-mask compactions included) and
autograd builds the same number again in the backward; here three kernels produce the loss *and* dL/d(colour), dL/d(depth),
which autograd hands straight to the rasterizer backward. Their sums are added in a fixed order: two calls on the same
inputs give the same bits."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import check

_WS = {}


def _ws(device):
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _WS:
        _WS[idx] = torch.zeros(_lib.lib().rtg_loss_workspace_bytes(), dtype=torch.uint8, device=torch.device("cuda", idx))
    return _WS[idx]


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _exposure_tensor(exposure):
    """`exposure` as the native losses read it: a (2,) CUDA float32 tensor (a, b), contiguous."""
    if not torch.is_tensor(exposure) or not exposure.is_cuda or exposure.dtype != torch.float32 or exposure.shape != (2,):
        raise TypeError("exposure must be a (2,) CUDA float32 tensor")
    return exposure.contiguous()


def frame_targets(gt_color, gt_depth, render_mask, H, W):
    """A measured H x W frame as the native losses and pose steps read it: (gt_color, gt_depth, mask, channels_last).
    gt_color (H,W,3) (channels_last = 1) or (3,H,W) (0) and gt_depth with H*W elements, both CUDA float32, come back
    detached and contiguous; render_mask (H*W elements, any dtype, nonzero = selected) as contiguous uint8 on their device,
    or None."""
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
        if render_mask.numel() != H * W:
            raise ValueError("render_mask must have H*W elements")
        mask = render_mask.detach().to(device=gt_depth.device, dtype=torch.uint8).contiguous()
    return gt_color.detach().contiguous(), gt_depth.detach().contiguous(), mask, channels_last


class _FusedLoss(torch.autograd.Function):
    """The frame loss and its gradients from one native call: rtg_loss_mapping if `mapping` (with the normal term when
    `normal` is given; rtg_loss_mapping_exposure if `exposure` is given too), else rtg_loss_l1_exposure if `exposure` is
    given, else rtg_loss_l1. Returns (loss, parts)."""

    @staticmethod
    def forward(ctx, render, depth, normal, exposure, depth_index, gt_color, gt_depth, gt_normal, render_mask, weights, mapping):
        L = _lib.lib()
        dev = render.device
        for name, t in (("render", render), ("depth", depth)):
            if not t.is_cuda or t.dtype != torch.float32:
                raise TypeError(f"{name} must be a CUDA float32 tensor")
        if depth_index.dtype != torch.int32:
            raise TypeError("depth_index must be int32 (the rasterizer's depth_index_map)")
        _, H, W = render.shape
        render, depth, depth_index = render.contiguous(), depth.contiguous(), depth_index.contiguous()
        gt_color, gt_depth, mask, channels_last = frame_targets(gt_color, gt_depth, render_mask, H, W)
        color_weight, depth_weight, normal_weight, depth_error_max = (float(w) for w in weights)
        g_color, g_depth, g_normal, g_exposure = torch.empty_like(render), torch.empty_like(depth), None, None
        out = torch.empty(8 if mapping else 4, dtype=torch.float32, device=dev)
        frame = (_p(depth_index), _p(gt_color), _p(gt_depth))
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        if exposure is not None:
            exposure = _exposure_tensor(exposure)
            g_exposure = torch.empty(2, dtype=torch.float32, device=dev)
        if mapping:
            if normal is not None:
                normal, gt_normal = normal.contiguous(), gt_normal.contiguous()
                if normal.shape != (3, H, W) or gt_normal.shape != (H, W, 3):
                    raise ValueError("normal must be (3,H,W) and gt_normal (H,W,3)")
                g_normal = torch.empty_like(render)
            head = (_p(render), _p(depth), _p(normal), *frame, _p(gt_normal), _p(mask), H, W, channels_last, color_weight, depth_weight,
                    normal_weight, depth_error_max)
            if exposure is None:
                check(L.rtg_loss_mapping(*head, _p(g_color), _p(g_depth), _p(g_normal), _p(out), _p(_ws(dev)), stream),
                      "rtg_loss_mapping")
            else:
                check(L.rtg_loss_mapping_exposure(*head, _p(exposure), _p(g_color), _p(g_depth), _p(g_normal), _p(g_exposure), _p(out),
                                                  _p(_ws(dev)), stream), "rtg_loss_mapping_exposure")
        elif exposure is None:
            check(L.rtg_loss_l1(_p(render), _p(depth), *frame, _p(mask), H, W, channels_last, color_weight, depth_weight,
                                depth_error_max, _p(g_color), _p(g_depth), _p(out), _p(_ws(dev)), stream), "rtg_loss_l1")
        else:
            check(L.rtg_loss_l1_exposure(_p(render), _p(depth), *frame, _p(mask), H, W, channels_last, color_weight, depth_weight,
                                         depth_error_max, _p(exposure), _p(g_color), _p(g_depth), _p(g_exposure), _p(out),
                                         _p(_ws(dev)), stream), "rtg_loss_l1_exposure")
        ctx.save_for_backward(g_color, g_depth, g_normal, g_exposure)
        ctx.mark_non_differentiable(out)
        return out[0], out

    @staticmethod
    def backward(ctx, grad_loss, _grad_parts):
        grads = tuple(None if g is None else g * grad_loss for g in ctx.saved_tensors)  # render, depth, normal, exposure
        return grads + (None,) * 7


def l1_color_depth_loss(render_output, gt_color, gt_depth, render_mask=None, color_weight=0.8, depth_weight=1.0,
                        depth_error_max=0.1, exposure=None):
    """`render_output` is the dict of Renderer.render. Defaults: color_weight / depth_weight / add_depth_thres of
    configs/base.yaml:76-77,51. Returns (loss, parts) with parts = tensor [loss, colour_l1, depth_l1, n_depth].
    `exposure`: None, or a (2,) CUDA float32 tensor (a, b): the colour residual becomes e^a render + b - gt_color
    (rtg_loss_l1_exposure) and the loss is differentiable with respect to the render and to `exposure`, so that a keyframe
    can be fitted under its camera's brightness without baking it into the map."""
    return _FusedLoss.apply(render_output["render"], render_output["depth"], None, exposure, render_output["depth_index_map"],
                            gt_color, gt_depth, None, render_mask, (color_weight, depth_weight, 0.0, depth_error_max), False)


_SSIM_WS = {}


class _FusedSsim(torch.autograd.Function):
    """1 - ssim(img1, img2) of utils/loss_utils.py:40-100 (11x11 Gaussian window, sigma 1.5, zero padding, mean) and its
    gradient w.r.t. img1 from three kernels (rtg_ssim_loss) instead of five grouped convolutions + ~15 elementwise kernels
    and their autograd twins. img2 (the measured frame) gets no gradient. With `exposure` (a, b) it is
    1 - ssim(e^a img1 + b, img2) (rtg_ssim_loss_exposure), differentiable w.r.t. img1 and the exposure."""

    @staticmethod
    def forward(ctx, img1, img2, exposure):
        L = _lib.lib()
        if img1.dim() != 3 or img1.shape != img2.shape:
            raise ValueError("ssim_loss: img1 and img2 must both be (C,H,W)")
        for name, t in (("img1", img1), ("img2", img2)):
            if not t.is_cuda or t.dtype != torch.float32:
                raise TypeError(f"{name} must be a CUDA float32 tensor")
        dev = img1.device
        Cn, H, W = img1.shape
        a, b = img1.contiguous(), img2.contiguous()
        if exposure is not None:
            exposure = _exposure_tensor(exposure)
        ws_bytes = L.rtg_ssim_workspace_bytes if exposure is None else L.rtg_ssim_exposure_workspace_bytes
        need = int(ws_bytes(Cn, H, W))
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        ws = _SSIM_WS.get(idx)
        if ws is None or ws.numel() < need:
            ws = _SSIM_WS[idx] = torch.empty(need, dtype=torch.uint8, device=dev)
        if ctx.needs_input_grad[1]:
            raise RuntimeError("ssim_loss: the gradient w.r.t. img2 (the measured frame) is not implemented; detach it")
        want_grad = ctx.needs_input_grad[0]
        g = torch.empty_like(a) if want_grad else None
        out = torch.empty(2, dtype=torch.float32, device=dev)
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        g_exposure = None
        if exposure is None:
            check(L.rtg_ssim_loss(_p(a), _p(b), Cn, H, W, _p(g), _p(out), _p(ws), stream), "rtg_ssim_loss")
        else:
            g_exposure = torch.empty(2, dtype=torch.float32, device=dev) if ctx.needs_input_grad[2] else None
            check(L.rtg_ssim_loss_exposure(_p(a), _p(b), Cn, H, W, _p(exposure), _p(g), _p(g_exposure), _p(out), _p(ws), stream),
                  "rtg_ssim_loss_exposure")
        ctx.save_for_backward(g, g_exposure)
        return out[0]

    @staticmethod
    def backward(ctx, grad_loss):
        g, g_exposure = ctx.saved_tensors
        return (None if g is None else g * grad_loss), None, (None if g_exposure is None else g_exposure * grad_loss)


def ssim_loss(img1, img2, exposure=None):
    """`1 - ssim(img1, img2)` as Mapping.loss_update evaluates it (SLAM/multiprocess/mapper.py:411-415, utils/loss_utils.py:50-100);
    img1, img2: (C,H,W) CUDA float32. Differentiable w.r.t. img1.
    `exposure`: None, or a (2,) CUDA float32 tensor (a, b): the term becomes 1 - ssim(e^a img1 + b, img2)
    (rtg_ssim_loss_exposure), differentiable w.r.t. img1 and `exposure`."""
    return _FusedSsim.apply(img1, img2, exposure)


def _ssim_term(img1, img2, window_size=11):
    """TEST REFERENCE, not used by `mapping_loss`: 1 - ssim(img1, img2) with the reference's own torch expressions
    (utils/loss_utils.py:40-100: 11x11 Gaussian window, sigma 1.5, zero padding, mean)."""
    import torch.nn.functional as F
    ch = img1.size(-3)
    x = torch.arange(window_size, dtype=img1.dtype, device=img1.device)
    g = torch.exp(-((x - window_size // 2) ** 2) / float(2 * 1.5 ** 2))
    g = (g / g.sum()).unsqueeze(1)
    window = (g @ g.t()).unsqueeze(0).unsqueeze(0).expand(ch, 1, window_size, window_size).contiguous()
    pad = window_size // 2
    a, b = img1.unsqueeze(0), img2.unsqueeze(0)
    mu1, mu2 = F.conv2d(a, window, padding=pad, groups=ch), F.conv2d(b, window, padding=pad, groups=ch)
    mu1_sq, mu2_sq, mu12 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    s1 = F.conv2d(a * a, window, padding=pad, groups=ch) - mu1_sq
    s2 = F.conv2d(b * b, window, padding=pad, groups=ch) - mu2_sq
    s12 = F.conv2d(a * b, window, padding=pad, groups=ch) - mu12
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    ssim_map = ((2 * mu12 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s1 + s2 + C2))
    return 1 - ssim_map.mean()


def mapping_loss(render_output, image_input, render_mask=None, color_weight=0.8, depth_weight=1.0, normal_weight=0.0, ssim_weight=0.2,
                 depth_error_max=0.1, exposure=None):
    """The image-space part of `Mapping.loss_update` (SLAM/multiprocess/mapper.py:402-451): colour L1 on the render mask,
    depth L1 on the valid mask, cosine normal loss, and -- only without a render mask, as in the reference -- the SSIM
    term. `render_output`: dict of Renderer.render; `image_input`: dict with "color_map" (H,W,3), "depth_map" (H,W[,1]),
    "normal_map" (H,W,3). Colour, depth and normal terms and their gradients come from three fused kernels, the SSIM term
    (which the shipped flows never reach: both call sites pass a render mask) from three more (`ssim_loss`).
    Returns (total_loss, parts): parts is a device tensor {total, colour, depth, n_depth, normal, n_normal, ssim, 0} --
    read it back once with `report_losses` instead of six `.item()` calls (mapper.py:459-466).
    `exposure`: None, or a (2,) CUDA float32 tensor (a, b), e.g. `keyframes.KeyframeTable.exposure(k)`: the colour L1 and the
    SSIM term are taken on e^a render + b (rtg_loss_mapping_exposure, `ssim_loss(..., exposure=)`), so that a keyframe seen
    brighter or darker than the map is fitted without baking its brightness into the map; autograd sums the two terms'
    exposure gradients. The depth and normal terms do not see it."""
    nrm, gtn = render_output.get("normal"), image_input.get("normal_map")
    if not (normal_weight > 0 and nrm is not None and gtn is not None):
        nrm, gtn, normal_weight = None, None, 0.0
    loss, parts = _FusedLoss.apply(render_output["render"], render_output["depth"], nrm, exposure, render_output["depth_index_map"],
                                   image_input["color_map"], image_input["depth_map"], gtn, render_mask,
                                   (color_weight, depth_weight, normal_weight, depth_error_max), True)
    if render_mask is None and ssim_weight > 0:
        gt = image_input["color_map"]
        gt = gt.permute(2, 0, 1) if gt.shape[-1] == 3 and gt.dim() == 3 and gt.shape[0] != 3 else gt
        ssim_l = ssim_loss(render_output["render"], gt, exposure)
        loss = loss + ssim_weight * ssim_l
        parts = parts.clone()
        parts[6] = ssim_l.detach()
        parts[0] = loss.detach()
    return loss, parts


_REPORT = {}


def report_losses(parts, scale_loss=None):
    """The `report_losses` dict of Mapping.loss_update from ONE device->host copy of the 8-float parts tensor (pinned
    buffer + event; the reference issues six blocking `.item()` calls). `scale_loss`: the attach loss tensor, if any."""
    dev = parts.device
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    if idx not in _REPORT:
        _REPORT[idx] = torch.zeros(9, dtype=torch.float32).pin_memory()
    host = _REPORT[idx]
    src = parts if scale_loss is None else torch.cat([parts, scale_loss.detach().reshape(1).to(parts.dtype)])
    host[:src.numel()].copy_(src, non_blocking=True)
    torch.cuda.current_stream(dev).synchronize()
    v = host.tolist()
    return {"total_loss": v[0], "depth_loss": v[2], "ssim_loss": v[6], "normal_loss": v[4], "color_loss": v[1],
            "scale_loss": v[8] if scale_loss is not None else 0.0}
