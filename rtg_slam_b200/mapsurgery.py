"""Map surgery on the Gaussian SoA and nearest-neighbour queries (SURVEY.md section 8(f) #4), backed by
librtg_splat_b200.so.

Mirrors, with the reference's names, argument order and return values:

* `distCUDA2(points)` of submodules/simple-knn (spatial.cu:15-30): `(mean squared distance to the 3 nearest other
  points (P,), their indices (P,3) int32)` -- what `GaussianPointCloud.update_geometry` consumes
  (SLAM/gaussian_pointcloud.py:376);
* `knn_points(p1, p2, K=..., return_nn=...)` of pytorch3d.ops as `Mapping.temp_points_filter` and
  `Mapping.gaussians_isolated` call it (SLAM/multiprocess/mapper.py:812-819,903-910): batched `(1,N,3)` inputs, returns
  `(dists (1,N,K) squared, idx (1,N,K) int64, knn (1,N,K,3) or None)`, neighbours sorted by distance;
* `delete` / `remove` / `cat` of `GaussianPointCloud` (SLAM/gaussian_pointcloud.py:195-235,286-304) on a dict of the
  attribute tensors: one mask scan + one gather launch for all attributes and ONE host synchronisation (the new row
  count) instead of one per attribute;
* `transform(params, anchor, old_c2w, new_c2w)` (no reference counterpart): the map follows corrected camera poses --
  every Gaussian moves rigidly, spherical harmonics included, with the correction of the frame that created it.

Ties between equidistant neighbours may be reported with a different (equally near) index than the reference's
Morton-box search or pytorch3d's would pick; distances are exact.
"""
from __future__ import annotations

import ctypes as C
from collections import namedtuple

import numpy as np
import torch

from . import _lib
from ._lib import check

_KNN = namedtuple("KNN", "dists idx knn")

# attribute names of GaussianPointCloud (SLAM/gaussian_pointcloud.py:195-221), in its order
ATTRIBUTES = ("xyz", "features_dc", "features_rest", "scaling", "rotation", "opacity", "normal", "confidence", "add_tick",
              "depth_error_counter", "color_error_counter")


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _points(name, t):
    if not t.is_cuda or t.dtype != torch.float32 or t.dim() != 2 or t.shape[1] != 3:
        raise TypeError(f"{name} must be a CUDA float32 (N, 3) tensor")
    return t.contiguous()


def knn(query, ref, K, skip_self=False, want_mean=False):
    """Exact K nearest `ref` points of every `query` point: (squared distances (N,K) ascending, indices (N,K) int32
    [, mean of the K squared distances (N,)])."""
    q, r = _points("query", query), _points("ref", ref)
    if q.device != r.device:
        raise ValueError("query and ref must live on the same device")
    L = _lib.lib()
    nq, nr = q.shape[0], r.shape[0]
    d2 = torch.empty((nq, K), dtype=torch.float32, device=q.device)
    idx = torch.empty((nq, K), dtype=torch.int32, device=q.device)
    mean = torch.empty((nq,), dtype=torch.float32, device=q.device) if want_mean else None
    ws = torch.empty(L.rtg_knn_workspace_bytes(nr), dtype=torch.uint8, device=q.device)
    check(L.rtg_knn(_p(q), nq, _p(r), nr, int(K), int(bool(skip_self)), _p(d2), _p(idx), _p(mean), _p(ws), _stream(q.device)), "rtg_knn")
    return (d2, idx, mean) if want_mean else (d2, idx)


def distCUDA2(points):
    """simple-knn's distCUDA2: (mean squared distance to the 3 nearest OTHER points, their indices (P,3) int32)."""
    pts = _points("points", points.float())
    _, idx, mean = knn(pts, pts, 3, skip_self=True, want_mean=True)
    return mean, idx


def knn_points(p1, p2, lengths1=None, lengths2=None, norm: int = 2, K: int = 1, version: int = -1, return_nn: bool = False,
               return_sorted: bool = True):
    """pytorch3d.ops.knn_points for the way the reference calls it: batch size 1, L2 norm, no ragged lengths."""
    if norm != 2 or lengths1 is not None or lengths2 is not None:
        raise NotImplementedError("knn_points: only norm=2 without lengths (the reference's call sites)")
    if p1.dim() != 3 or p2.dim() != 3 or p1.shape[0] != 1 or p2.shape[0] != 1:
        raise ValueError("knn_points: expected (1, N, 3) inputs")
    if K > 8:
        raise NotImplementedError("knn_points: K <= 8")
    d2, idx = knn(p1[0], p2[0], K)
    nn = p2[0][idx.long()][None] if return_nn else None
    return _KNN(dists=d2[None], idx=idx.long()[None], knn=nn)


# ----------------------------------------------------------------------------- SoA compaction
_PINNED = {}


def _count_buffer(device):
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _PINNED:
        _PINNED[idx] = (torch.zeros(1, dtype=torch.int32).pin_memory(), torch.cuda.Event())
    return _PINNED[idx]


def compact(mask, tensors, invert=False):
    """Rows of every tensor in `tensors` (all with the same leading dimension, 4-byte dtypes, same device) where `mask` is
    True (or False with invert=True), in order. One scan, one gather launch, one host synchronisation (the row count)."""
    tensors = list(tensors)
    if not mask.is_cuda or mask.dtype != torch.bool or mask.dim() != 1:
        raise TypeError("mask must be a CUDA bool vector")
    P = mask.shape[0]
    dev = mask.device
    if len(tensors) > 16:
        raise ValueError("at most 16 attribute tensors per call")
    ins, words = [], []
    for t in tensors:
        if t.device != dev or t.shape[0] != P or t.element_size() != 4:
            raise TypeError("every attribute must be a 4-byte tensor on the mask's device with one row per mask entry")
        t = t.detach().contiguous()
        ins.append(t)
        words.append(max(1, t[0].numel()) if P > 0 else 1)
    outs = [torch.empty_like(t) for t in ins]
    L = _lib.lib()
    n = len(ins)
    count_dev = torch.empty(1, dtype=torch.int32, device=dev)
    pinned, event = _count_buffer(dev)
    ws = torch.empty(L.rtg_soa_compact_workspace_bytes(P), dtype=torch.uint8, device=dev)
    VP, I32 = C.c_void_p * max(n, 1), C.c_int32 * max(n, 1)
    m8 = mask.contiguous().view(torch.uint8)
    stream = torch.cuda.current_stream(dev)
    check(L.rtg_soa_compact(_p(m8), int(bool(invert)), P, n, VP(*[t.data_ptr() for t in ins]), VP(*[t.data_ptr() for t in outs]),
                            I32(*words), _p(count_dev), C.c_void_p(pinned.data_ptr()), _p(ws), C.c_void_p(stream.cuda_stream)),
          "rtg_soa_compact")
    event.record(stream)
    event.synchronize()  # the new number of rows defines the tensor shapes
    kept = int(pinned[0])
    return [o[:kept] for o in outs], kept


def delete(params: dict, delete_mask):
    """GaussianPointCloud.delete: every attribute keeps the rows with ~delete_mask. Returns the new dict."""
    keys = [k for k in params if isinstance(params[k], torch.Tensor)]
    outs, _ = compact(delete_mask, [params[k] for k in keys], invert=True)
    new = dict(params)
    new.update(dict(zip(keys, outs)))
    return new


def remove(params: dict, remove_mask):
    """GaussianPointCloud.remove: (rows with remove_mask, dict without them)."""
    keys = [k for k in params if isinstance(params[k], torch.Tensor)]
    taken, _ = compact(remove_mask, [params[k] for k in keys])
    return dict(zip(keys, taken)), delete(params, remove_mask)


def cat(params: dict, extra: dict):
    """GaussianPointCloud.cat for the attributes present in both dicts."""
    return {k: torch.cat([params[k], extra[k]]) if k in extra else params[k] for k in params}


# ----------------------------------------------------------------------------- the map follows corrected poses
SH_REST = (0, 3, 8, 15)


def _poses(name, c2w):
    """Host (K,4,4) camera-to-world poses as float64 numpy, checked to be rigid."""
    if isinstance(c2w, torch.Tensor):
        if c2w.is_cuda:
            raise TypeError(f"{name} must be a host array (numpy or CPU tensor)")
        c2w = c2w.detach().numpy()
    a = np.ascontiguousarray(c2w, dtype=np.float64)
    if a.ndim != 3 or a.shape[1:] != (4, 4):
        raise ValueError(f"{name} must have shape (K, 4, 4), got {a.shape}")
    if not np.isfinite(a).all():
        raise ValueError(f"{name} has non-finite entries")
    if not (a[:, 3] == np.array([0.0, 0.0, 0.0, 1.0])).all():
        raise ValueError(f"{name}: the last row of every pose must be (0, 0, 0, 1)")
    R = a[:, :3, :3]
    if len(a) and (np.abs(R @ R.transpose(0, 2, 1) - np.eye(3)).max() > 1e-5 or (np.linalg.det(R) <= 0).any()):
        raise ValueError(f"{name}: every rotation block must be orthonormal (to 1e-5) with det > 0")
    return a


def _rows(name, t, P, shape, dtype=torch.float32):
    """`t` checked to be a contiguous CUDA (P, *shape) tensor of `dtype`; returned detached (same storage)."""
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != dtype:
        raise TypeError(f"{name} must be a CUDA {dtype} tensor")
    if tuple(t.shape) != (P, *shape):
        raise ValueError(f"{name} must have shape {(P, *shape)}, got {tuple(t.shape)}")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous (it is updated in place)")
    return t.detach()


def transform(params: dict, anchor, old_c2w, new_c2w):
    """Moves the map with corrected camera poses, in place: every Gaussian follows the correction
    new_c2w[k] @ inv(old_c2w[k]) of its anchor frame k = anchor[i] (GaussianPointCloud._add_tick).

    `params` holds the raw attribute tensors under the names of `remove()`: "xyz" (P,3) and "rotation" (P,4) are
    required, "normal" (P,3) and "features_rest" (P,M-1,3), M in {1,4,9,16}, are moved when present (the spherical
    harmonics are rotated band by band, so the rendered colour of a surfel does not change when it moves). Everything else
    is left alone. anchor: (P,) or (P,1) int32 on the map's device; -1 = not anchored. old_c2w, new_c2w: host (K,4,4)
    rigid camera-to-world poses (numpy or CPU tensors), validated here and uploaded without a synchronisation. Rows whose
    anchor's two poses are equal are not written. Returns a device int64 tensor (1,): the number of rows whose anchor is
    neither -1 nor in [0, K) (they are left unchanged; with K == 0 that is every anchored row); it is not read back."""
    old, new = _poses("old_c2w", old_c2w), _poses("new_c2w", new_c2w)
    if old.shape != new.shape:
        raise ValueError(f"old_c2w and new_c2w differ in shape: {old.shape} vs {new.shape}")
    xyz = params["xyz"]
    if isinstance(xyz, torch.Tensor) and xyz.is_cuda and xyz.numel() == 0:  # an empty map (GaussianPointCloud's initial state)
        return torch.zeros(1, dtype=torch.int64, device=xyz.device)
    if not isinstance(xyz, torch.Tensor) or xyz.dim() != 2:
        raise TypeError("params['xyz'] must be a (P, 3) CUDA float32 tensor")
    P, K = xyz.shape[0], old.shape[0]
    xyz = _rows("xyz", xyz, P, (3,))
    dev = xyz.device
    rot = _rows("rotation", params["rotation"], P, (4,))
    normal = params.get("normal")
    normal = None if normal is None else _rows("normal", normal, P, (3,))
    rest = params.get("features_rest")
    sh_rest = 0
    if rest is not None:
        if not isinstance(rest, torch.Tensor):
            raise TypeError("features_rest must be a CUDA float32 tensor")
        if rest.dim() != 3 or rest.shape[1] not in SH_REST:
            raise ValueError("features_rest must be (P, M-1, 3) with M in {1, 4, 9, 16}")
        sh_rest = rest.shape[1]
        rest = _rows("features_rest", rest, P, (sh_rest, 3))
    if not isinstance(anchor, torch.Tensor) or not anchor.is_cuda or anchor.dtype != torch.int32:
        raise TypeError("anchor must be a CUDA int32 tensor")
    if tuple(anchor.shape) not in ((P,), (P, 1)):
        raise ValueError(f"anchor must have shape ({P},) or ({P}, 1), got {tuple(anchor.shape)}")
    for name, t in (("rotation", rot), ("normal", normal), ("features_rest", rest), ("anchor", anchor)):
        if t is not None and t.device != dev:
            raise ValueError(f"{name} is not on the device of xyz")
    anchor = anchor.contiguous()
    poses = torch.from_numpy(np.stack([old, new])).pin_memory().to(dev, non_blocking=True)
    n_skipped = torch.empty(1, dtype=torch.int64, device=dev)
    L = _lib.lib()
    ws = torch.empty(max(int(L.rtg_map_transform_workspace_bytes(K)), 16), dtype=torch.uint8, device=dev)
    xf = _lib.RtgMapTransform(P=P, K=K, sh_rest=sh_rest, _pad=0, anchor=anchor.data_ptr(), old_c2w=poses[0].data_ptr(),
                              new_c2w=poses[1].data_ptr(), xyz=xyz.data_ptr(), rotation=rot.data_ptr(),
                              normal=None if normal is None else normal.data_ptr(),
                              features_rest=None if sh_rest == 0 else rest.data_ptr(), n_skipped=n_skipped.data_ptr())
    check(L.rtg_map_transform(C.byref(xf), _p(ws), _stream(dev)), "rtg_map_transform")
    return n_skipped
