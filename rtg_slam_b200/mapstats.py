"""Per-frame consumers of the rasterizer's index / transmittance maps (SURVEY.md section 8(f) #2).

Same names and argument meaning as the reference:
* `accumulate_gaussian_error` -- `cuda_utils._C.accumulate_gaussian_error` (submodules/cuda_utils/cuda_utils.cu:17-60),
  called by Mapping.error_gaussians_remove (SLAM/multiprocess/mapper.py:546-559);
* `pixelmask2tilemask`, `transmission2tilemask`, `colorerror2tilemask` -- SLAM/utils.py:681-734, called by
  Mapping.evaluate_render_range (mapper.py:471-508);
plus two fused entry points for that caller: `transmission_masks(T_map)` = (render_mask, tile_mask) in one pass and
`color_error_map(render, gt)`, and `gaussian_contributions`, what every Gaussian adds to a frame (rtg_splat_contributions).
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib, rasterizer
from ._lib import check


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _f32(name, t, n=None):
    if not t.is_cuda or t.dtype != torch.float32:
        raise TypeError(f"{name} must be a CUDA float32 tensor")
    t = t.contiguous()
    if n is not None and t.numel() != n:
        raise ValueError(f"{name} must have {n} elements")
    return t


def accumulate_gaussian_error(H, W, P, screen_color_error, screen_depth_error, screen_normal_error, screen_color_index,
                              screen_depth_index, color_threshold, depth_threshold, normal_threshold, check_max):
    """Returns (gs_color_error, gs_depth_error, gs_normal_error, gs_rescale_counter), each (P, 1) float32."""
    N = int(H) * int(W)
    ce, de, ne = (_f32(n, t, N) for n, t in (("screen_color_error", screen_color_error), ("screen_depth_error", screen_depth_error),
                                             ("screen_normal_error", screen_normal_error)))
    idx = []
    for name, t in (("screen_color_index", screen_color_index), ("screen_depth_index", screen_depth_index)):
        if not t.is_cuda or t.dtype != torch.int32:
            raise TypeError(f"{name} must be a CUDA int32 tensor (the rasterizer's index maps)")
        if t.numel() != N:
            raise ValueError(f"{name} must have {N} elements")
        idx.append(t.contiguous())
    dev = ce.device
    out = [torch.empty((P, 1), dtype=torch.float32, device=dev) for _ in range(4)]
    counters = None if check_max else torch.empty(2 * max(P, 1), dtype=torch.int32, device=dev)
    check(_lib.lib().rtg_accumulate_gaussian_error(int(H), int(W), int(P), _p(ce), _p(de), _p(ne), _p(idx[0]), _p(idx[1]),
                                                   float(color_threshold), float(depth_threshold), float(normal_threshold),
                                                   1 if check_max else 0, _p(out[0]), _p(out[1]), _p(out[2]), _p(out[3]),
                                                   _p(counters), _stream(dev)), "rtg_accumulate_gaussian_error")
    return tuple(out)


def _tile_grid(H, W, stride):
    if stride != 16:
        raise ValueError("only the rasterizer's 16x16 tiles are supported (the reference passes stride=16 everywhere)")
    return (H + 15) // 16, (W + 15) // 16


def _tile_mean(img, ratio, want_mean, want_mask):
    H, W = img.shape[:2]
    img = _f32("image", img, H * W)
    th, tw = _tile_grid(H, W, 16)
    mean = torch.empty((th, tw), dtype=torch.float32, device=img.device) if want_mean else None
    mask = torch.empty((th, tw), dtype=torch.int32, device=img.device) if want_mask else None
    check(_lib.lib().rtg_tile_mean(H, W, _p(img), float(ratio), _p(mean), _p(mask), _stream(img.device)), "rtg_tile_mean")
    return mean, mask


def transmission2tilemask(pixelmask, stride, tile_mask_ratio=0.5):
    """(H,W) bool / numeric mask -> (tiles_y, tiles_x) int32: tiles whose masked fraction (zero padded) exceeds the ratio."""
    _tile_grid(pixelmask.shape[0], pixelmask.shape[1], stride)
    return _tile_mean(pixelmask.float(), tile_mask_ratio, False, True)[1]


def pixelmask2tilemask(pixelmask, stride):
    """Max pooling: tiles with at least one masked pixel (a 0/1 mask: mean > 0)."""
    _tile_grid(pixelmask.shape[0], pixelmask.shape[1], stride)
    return _tile_mean((pixelmask != 0).float(), 0.0, False, True)[1]


def colorerror2tilemask(color_error, stride, top_ratio=0.4):
    """(H,W) float error -> int32 (tiles_y, tiles_x) mask of the int(numel * top_ratio) tiles with the largest mean
    error (torch.topk on the pooled map, as in the reference; the pooling is the native pass). int32 like the
    reference's devI(...) (SLAM/utils.py:733-735): the mapper hands it to Renderer.render as tile_mask."""
    _tile_grid(color_error.shape[0], color_error.shape[1], stride)
    mean, _ = _tile_mean(color_error, 0.0, True, False)
    k = int(mean.numel() * top_ratio)
    _, top = torch.topk(mean.view(-1), k=k)
    mask = torch.zeros(mean.shape, dtype=torch.int32, device=mean.device)
    mask.view(-1)[top] = 1
    return mask


def transmission_masks(T_map, tile_mask_ratio=0.5):
    """render_mask = (T_map != 1) and transmission2tilemask(render_mask, 16, ratio) in one pass (mapper.py:503-505).
    T_map: (1,H,W) or (H,W). Returns (render_mask bool (H,W), tile_mask int32)."""
    H, W = T_map.shape[-2:]
    T = _f32("T_map", T_map, H * W)
    th, tw = _tile_grid(H, W, 16)
    rm = torch.empty((H, W), dtype=torch.uint8, device=T.device)
    tm = torch.empty((th, tw), dtype=torch.int32, device=T.device)
    check(_lib.lib().rtg_transmission_tile_mask(H, W, _p(T), float(tile_mask_ratio), _p(rm), _p(tm), _stream(T.device)),
          "rtg_transmission_tile_mask")
    return rm.view(torch.bool), tm


def color_error_map(render, gt):
    """sum_c |render - gt| with black rendered pixels zeroed (mapper.py:481-487). render, gt: (3,H,W). Returns (H,W)."""
    _, H, W = render.shape
    r, g = _f32("render", render, 3 * H * W), _f32("gt", gt, 3 * H * W)
    out = torch.empty((H, W), dtype=torch.float32, device=r.device)
    check(_lib.lib().rtg_color_error(H, W, _p(r), _p(g), _p(out), _stream(r.device)), "rtg_color_error")
    return out


def gaussian_contributions(raster_settings, means3D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                           cov3D_precomp=None, tile_mask=None, pixel_error=None, out=None):
    """One rasterizer forward and what each Gaussian added to it (rtg_splat_contributions). A pair (pixel p, Gaussian g)
    adds colour when the forward blends it; its weight is w = alpha T, the forward's colour weight. Per Gaussian:
      n_pixels (int32)  the pixels g adds colour to,
      weight (float32)  sum_p w(p, g)  (an importance score; sum_g = sum_p (1 - T_map) over the rendered pixels),
      error (float32)   sum_p w(p, g) pixel_error(p), only with `pixel_error` (H, W) float32: every pixel's error shared
                        among all the Gaussians that blend into it, not only the arg-max of accumulate_gaussian_error.
    Inputs as GaussianRasterizer takes them; the mode of `rasterizer.antialiased()` applies. A forward that overflows its
    binning buffer is rendered again once; a second overflow raises CapacityOverflow. `out`: a dict of such (P,) CUDA
    tensors to add into (for sums over several frames); without it zeroed tensors are allocated.
    Returns (outputs, stats): the forward's eight outputs as GaussianRasterizer returns them and the dict. Nothing is
    differentiated by autograd."""
    with torch.no_grad():
        dev = means3D.device
        st = rasterizer._state(dev)
        P = int(means3D.shape[0])
        H, W = int(raster_settings.image_height), int(raster_settings.image_width)
        pe = None if pixel_error is None else _f32("pixel_error", pixel_error, H * W)
        if pe is not None and pe.device != dev:
            raise ValueError(f"pixel_error is on {pe.device}, expected {dev}")
        want = {"n_pixels": torch.int32, "weight": torch.float32}
        if pe is not None:
            want["error"] = torch.float32
        if out is None:
            stats = {k: torch.zeros((P,), dtype=dt, device=dev) for k, dt in want.items()}
        else:
            if set(out) != set(want):
                raise ValueError(f"out must hold exactly {sorted(want)}")
            for k, dt in want.items():
                t = out[k]
                if not torch.is_tensor(t) or t.dtype != dt or t.device != dev or tuple(t.shape) != (P,) or not t.is_contiguous():
                    raise ValueError(f"out[{k!r}] must be a contiguous ({P},) {dt} tensor on {dev}")
            stats = out
        for attempt in range(2):
            outs, saved, _ = rasterizer._forward_native(raster_settings, means3D, shs, colors_precomp, opacities, scales, rotations,
                                                        cov3D_precomp, tile_mask)
            st.read(saved.pending, block=True)
            if not saved.pending.overflow:
                break
            if attempt:
                raise rasterizer.CapacityOverflow("gaussian_contributions: the render overflowed the binning buffer twice")
        view, keep = rasterizer._make_view(raster_settings, dev, saved.antialiased)
        check(_lib.lib().rtg_splat_contributions(C.byref(view), P, C.c_void_p(saved.geom), C.c_void_p(saved.img),
                                                 C.c_void_p(saved.bin), saved.r_cap, C.c_void_p(saved.counters), _p(pe),
                                                 _p(stats["n_pixels"]), _p(stats["weight"]), _p(stats.get("error")), _stream(dev)),
              "rtg_splat_contributions")
        return outs, stats
