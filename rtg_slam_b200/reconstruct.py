"""A surface from the map, and the reconstruction metric (no reference counterpart for the fusion; the metric is
`eval_pcd` of SLAM/eval.py:149-223), backed by librtg_splat_b200.so.

* `TsdfVolume`: a dense truncated-signed-distance grid on the device. `integrate` folds one depth frame (a rendered hit
  depth at a keyframe pose, or a measured depth at a tracked pose) into it; `extract_mesh` runs marching tetrahedra;
  `raycast` renders depth, normal and colour images of that same surface from a pose. All are CUDA kernels of the library
  (rtg_tsdf_integrate / rtg_tsdf_extract_count / rtg_tsdf_extract_emit / rtg_tsdf_raycast); the only host read-back is
  the two mesh sizes.
* `reconstruction_metrics`: accuracy, completion, precision, recall and F-score of a reconstructed point set against
  ground-truth surface points, with eval_pcd's keys and units; nearest neighbours both ways come from `mapsurgery.knn`.
* `sample_surface`: area-weighted points on a triangle mesh, on the device.
* `write_ply`: a binary little-endian PLY of a mesh.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib, mapsurgery
from ._lib import check

MAX_VOXELS = 1 << 31


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _cuda_f32(name, t):
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32:
        raise TypeError(f"{name} must be a CUDA float32 tensor")
    return t


def _points(name, t):
    t = _cuda_f32(name, t)
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError(f"{name} must be (N, 3), got {tuple(t.shape)}")
    return t.detach().contiguous()


class TsdfVolume:
    """Dense voxel grid over an axis-aligned box: voxel (i, j, k) has its centre at origin + voxel_size * (i, j, k),
    dims = (nx, ny, nz) with nx*ny*nz < 2^31, trunc > 0 the truncation distance in map units.

    `tsdf` (initialised to 1), `weight` (0) and, with color=True, `color` (0) are float32 CUDA tensors of shape (nz, ny, nx)
    and (3, nz, ny, nx): x fastest, as the kernels address them. They may be written directly (for example to load a
    grid); `integrate` and `extract_mesh` read them as they are."""

    def __init__(self, origin, voxel_size, dims, trunc, color=False, device=None):
        origin = tuple(float(o) for o in origin)
        dims = tuple(int(d) for d in dims)
        if len(origin) != 3 or len(dims) != 3:
            raise ValueError("origin and dims must have three entries")
        if not np.isfinite(origin).all():
            raise ValueError("origin must be finite")
        if min(dims) < 1 or dims[0] * dims[1] * dims[2] >= MAX_VOXELS:
            raise ValueError(f"dims must be >= 1 with nx*ny*nz < 2^31, got {dims}")
        if not (np.isfinite(voxel_size) and voxel_size > 0 and np.isfinite(trunc) and trunc > 0):
            raise ValueError("voxel_size and trunc must be finite and > 0")
        self.origin, self.voxel_size, self.dims, self.trunc = origin, float(voxel_size), dims, float(trunc)
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        nx, ny, nz = dims
        self.tsdf = torch.ones((nz, ny, nx), dtype=torch.float32, device=dev)
        self.weight = torch.zeros((nz, ny, nx), dtype=torch.float32, device=dev)
        self.color = torch.zeros((3, nz, ny, nx), dtype=torch.float32, device=dev) if color else None

    @property
    def device(self):
        return self.tsdf.device

    def _desc(self):
        for name, t, shape in (("tsdf", self.tsdf, self.dims[::-1]), ("weight", self.weight, self.dims[::-1]),
                               ("color", self.color, (3, *self.dims[::-1]))):
            if t is None:
                continue
            _cuda_f32(f"vol.{name}", t)
            if tuple(t.shape) != tuple(shape) or not t.is_contiguous() or t.device != self.device:
                raise ValueError(f"vol.{name} must stay a contiguous {tuple(shape)} tensor on {self.device}")
        nx, ny, nz = self.dims
        return _lib.RtgTsdfVolume(nx=nx, ny=ny, nz=nz, voxel_size=self.voxel_size, trunc=self.trunc,
                                  origin=(C.c_float * 3)(*self.origin), tsdf=self.tsdf.data_ptr(), weight=self.weight.data_ptr(),
                                  color=None if self.color is None else self.color.data_ptr())

    def integrate(self, depth, w2c, intrinsics, color=None, color_channels_last=False):
        """Folds one frame into the volume (rtg_tsdf_integrate). depth: (H, W) or (1, H, W) float32, 0 = no reading.
        w2c: (4, 4) float64 or float32 CUDA tensor, the world-to-camera pose (as `KeyframeTable.pose(k)` or
        `PoseRefiner` hold it), read on the device. intrinsics: (fx, fy, cx, cy). color: (3, H, W), or (H, W, 3) with
        color_channels_last=True; required exactly when the volume has colour. No host synchronisation."""
        depth = _cuda_f32("depth", depth)
        if depth.dim() == 3 and depth.shape[0] == 1:
            depth = depth[0]
        if depth.dim() != 2:
            raise ValueError(f"depth must be (H, W) or (1, H, W), got {tuple(depth.shape)}")
        H, W = depth.shape
        if not isinstance(w2c, torch.Tensor) or not w2c.is_cuda or w2c.dtype not in (torch.float32, torch.float64):
            raise TypeError("w2c must be a CUDA float32 or float64 tensor")
        if tuple(w2c.shape) != (4, 4):
            raise ValueError(f"w2c must be (4, 4), got {tuple(w2c.shape)}")
        fx, fy, cx, cy = (float(k) for k in intrinsics)
        if (self.color is None) != (color is None):
            raise ValueError("color must be given exactly when the volume was made with color=True")
        if color is not None:
            color = _cuda_f32("color", color)
            want = (H, W, 3) if color_channels_last else (3, H, W)
            if tuple(color.shape) != want:
                raise ValueError(f"color must be {want}, got {tuple(color.shape)}")
            color = color.detach().contiguous()
        for name, t in (("depth", depth), ("w2c", w2c), ("color", color)):
            if t is not None and t.device != self.device:
                raise ValueError(f"{name} is not on the volume's device")
        depth = depth.detach().contiguous()
        w2c = w2c.detach().contiguous()
        vol = self._desc()
        check(_lib.lib().rtg_tsdf_integrate(C.byref(vol), _p(depth), _p(color), H, W, int(bool(color_channels_last)), fx, fy, cx, cy,
                                            _p(w2c), int(w2c.dtype == torch.float64), _stream(self.device)), "rtg_tsdf_integrate")

    def raycast(self, w2c, intrinsics, H, W):
        """Renders the surface `extract_mesh` emits from a camera (rtg_tsdf_raycast): {"depth": (H, W) camera z,
        "normal": (3, H, W) world-space unit normals towards free space, "color": (3, H, W) or None without volume colour},
        float32 on the volume's device, 0 where the pixel's first crossing is a back face or there is none. w2c: (4, 4)
        float64 or float32 CUDA tensor, read on the device; intrinsics: (fx, fy, cx, cy). No host synchronisation.
        As a frame-to-model target for `icp.IcpTracker.update_last_status`: `depth[..., None]` and
        `normal.permute(1, 2, 0)`, with the frame's normals in world space too."""
        H, W = int(H), int(W)
        if H < 1 or W < 1:
            raise ValueError(f"H and W must be >= 1, got ({H}, {W})")
        if not isinstance(w2c, torch.Tensor) or not w2c.is_cuda or w2c.dtype not in (torch.float32, torch.float64):
            raise TypeError("w2c must be a CUDA float32 or float64 tensor")
        if tuple(w2c.shape) != (4, 4):
            raise ValueError(f"w2c must be (4, 4), got {tuple(w2c.shape)}")
        if w2c.device != self.device:
            raise ValueError("w2c is not on the volume's device")
        fx, fy, cx, cy = (float(k) for k in intrinsics)
        w2c = w2c.detach().contiguous()
        vol = self._desc()
        dev = self.device
        depth = torch.empty((H, W), dtype=torch.float32, device=dev)
        normal = torch.empty((3, H, W), dtype=torch.float32, device=dev)
        color = torch.empty((3, H, W), dtype=torch.float32, device=dev) if self.color is not None else None
        check(_lib.lib().rtg_tsdf_raycast(C.byref(vol), _p(w2c), int(w2c.dtype == torch.float64), H, W, fx, fy, cx, cy, _p(depth),
                                          _p(normal), _p(color), _stream(dev)), "rtg_tsdf_raycast")
        return {"depth": depth, "normal": normal, "color": color}

    def extract_mesh(self):
        """Marching tetrahedra on the Kuhn decomposition of the grid: {"vertices": (V, 3) float32 world positions,
        "faces": (F, 3) int32, right-handed with the normal towards free space, "colors": (V, 3) float32 or None}.
        One host read-back: the two sizes."""
        L = _lib.lib()
        nx, ny, nz = self.dims
        ws_bytes = int(L.rtg_tsdf_extract_workspace_bytes(nx, ny, nz))
        if ws_bytes == 0:
            raise ValueError(f"extraction needs 12*nx*ny*nz < 2^32, got dims {self.dims}")
        vol = self._desc()
        dev, stream = self.device, _stream(self.device)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        counts = torch.empty(2, dtype=torch.int32, device=dev)
        check(L.rtg_tsdf_extract_count(C.byref(vol), _p(ws), _p(counts), stream), "rtg_tsdf_extract_count")
        V, F = (int(c) & 0xFFFFFFFF for c in counts.cpu())
        vertices = torch.empty((max(V, 1), 3), dtype=torch.float32, device=dev)
        faces = torch.empty((max(F, 1), 3), dtype=torch.int32, device=dev)
        colors = torch.empty((max(V, 1), 3), dtype=torch.float32, device=dev) if self.color is not None else None
        check(L.rtg_tsdf_extract_emit(C.byref(vol), _p(ws), _p(vertices), _p(colors), _p(faces), stream), "rtg_tsdf_extract_emit")
        return {"vertices": vertices[:V], "faces": faces[:F], "colors": None if colors is None else colors[:V]}


def reconstruction_metrics(rec_points, gt_points, thresholds=(0.03,)):
    """eval_pcd's numbers (SLAM/eval.py:198-223) for reconstructed points against ground-truth surface points, both
    (N, 3) CUDA float32 in map units: "accuracy" (mean distance rec -> gt) and "completion" (mean distance gt -> rec), x100
    (cm for metres), and per threshold t "P (< t)" / "R (< t)" (percentage of rec / gt points closer than t) and
    "F1 (< t)" = 2PR/(P+R) (0 when both are 0). Subsampling the reconstruction, as eval_pcd does, is the caller's choice.
    Nearest neighbours are exact (`mapsurgery.knn`); the result is read back once."""
    rec, gt = _points("rec_points", rec_points), _points("gt_points", gt_points)
    if rec.device != gt.device:
        raise ValueError("rec_points and gt_points must live on the same device")
    if rec.shape[0] == 0 or gt.shape[0] == 0:
        raise ValueError("both point sets must be non-empty")
    thresholds = tuple(float(t) for t in thresholds)
    d_acc = mapsurgery.knn(rec, gt, 1)[0][:, 0].double().sqrt()
    d_comp = mapsurgery.knn(gt, rec, 1)[0][:, 0].double().sqrt()
    parts = [d_acc.mean(), d_comp.mean()]
    for t in thresholds:
        parts += [(d_acc < t).double().mean(), (d_comp < t).double().mean()]
    vals = torch.stack(parts).cpu().tolist()
    out = {"accuracy": vals[0] * 100, "completion": vals[1] * 100}
    Ps, Rs, Fs = {}, {}, {}
    for n, t in enumerate(thresholds):
        P, R = vals[2 + 2 * n] * 100, vals[3 + 2 * n] * 100
        Ps[f"P (< {t})"], Rs[f"R (< {t})"] = P, R
        Fs[f"F1 (< {t})"] = 2 * P * R / (P + R) if P + R > 0 else 0.0
    out.update(Ps)
    out.update(Rs)
    out.update(Fs)
    return out


def sample_surface(vertices, faces, n, seed=0):
    """n points on the mesh (vertices (V, 3) CUDA float32, faces (F, 3) CUDA int32/int64), faces drawn with probability
    proportional to their area and points uniform inside the drawn face; returns (n, 3) float32 on the mesh's device."""
    v = _points("vertices", vertices)
    if not isinstance(faces, torch.Tensor) or not faces.is_cuda or faces.dtype not in (torch.int32, torch.int64):
        raise TypeError("faces must be a CUDA int32 or int64 tensor")
    if faces.dim() != 2 or faces.shape[1] != 3 or faces.shape[0] == 0:
        raise ValueError(f"faces must be (F, 3) with F >= 1, got {tuple(faces.shape)}")
    if faces.device != v.device:
        raise ValueError("faces and vertices must live on the same device")
    f = faces.long()
    a, b, c = v[f[:, 0]].double(), v[f[:, 1]].double(), v[f[:, 2]].double()
    area = torch.linalg.cross(b - a, c - a).norm(dim=1)
    gen = torch.Generator(device=v.device).manual_seed(int(seed))
    pick = torch.multinomial(area, int(n), replacement=True, generator=gen)
    uv = torch.rand((int(n), 2), dtype=torch.float64, device=v.device, generator=gen)
    uv = torch.where(uv.sum(1, keepdim=True) > 1, 1 - uv, uv)   # reflect (u, v) back into the triangle: uniform over it
    a, b, c = a[pick], b[pick], c[pick]
    return (a + uv[:, :1] * (b - a) + uv[:, 1:] * (c - a)).float()


def write_ply(path, vertices, faces, colors=None):
    """Writes a binary little-endian PLY: float x, y, z per vertex, uchar red, green, blue when `colors` (in [0, 1],
    clipped, rounded) is given, and one `uchar int vertex_indices` list per face. Tensors are copied to the host."""
    v = np.ascontiguousarray(torch.as_tensor(vertices).detach().cpu().numpy(), dtype="<f4")
    f = np.ascontiguousarray(torch.as_tensor(faces).detach().cpu().numpy(), dtype="<i4")
    if v.ndim != 2 or v.shape[1] != 3 or f.ndim != 2 or f.shape[1] != 3:
        raise ValueError("vertices must be (V, 3) and faces (F, 3)")
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    header = ["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}",
              "property float x", "property float y", "property float z"]
    if colors is not None:
        c = torch.as_tensor(colors).detach().cpu().numpy()
        if c.shape != v.shape:
            raise ValueError("colors must be (V, 3) like vertices")
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
        header += ["property uchar red", "property uchar green", "property uchar blue"]
    header += [f"element face {len(f)}", "property list uchar int vertex_indices", "end_header"]
    vert = np.empty(len(v), dtype=fields)
    vert["x"], vert["y"], vert["z"] = v[:, 0], v[:, 1], v[:, 2]
    if colors is not None:
        c8 = np.rint(np.clip(c, 0.0, 1.0) * 255.0).astype(np.uint8)
        vert["red"], vert["green"], vert["blue"] = c8[:, 0], c8[:, 1], c8[:, 2]
    face = np.empty(len(f), dtype=[("n", "u1"), ("i", "<i4", (3,))])
    face["n"], face["i"] = 3, f
    with open(path, "wb") as fh:
        fh.write(("\n".join(header) + "\n").encode("ascii"))
        fh.write(vert.tobytes())
        fh.write(face.tobytes())
