"""ctypes front end of oracle/splat_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / `--impl reference`
legs may import this module. See the header of splat_oracle.c for what it restates and
how it is pinned (tests/golden/, produced by the reference's own CUDA code on an H100).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
_LIBS = {}


def build(force: bool = False) -> None:
    want = [os.path.join(HERE, "_build", f"liboracle_{p}.so") for p in ("f32", "f64")]
    src = os.path.join(HERE, "splat_oracle.c")
    if not force and all(os.path.exists(w) and os.path.getmtime(w) >= os.path.getmtime(src) for w in want):
        return
    subprocess.check_call(["make", "-C", HERE, "-s", "-B"])


def _lib(precision: str):
    if precision in _LIBS:
        return _LIBS[precision]
    build()
    lib = C.CDLL(os.path.join(HERE, "_build", f"liboracle_{precision}.so"))
    real = C.c_float if precision == "f32" else C.c_double
    assert lib.oracle_sizeof_real() == C.sizeof(real)
    lib.oracle_forward.restype = C.c_void_p
    lib.oracle_num_rendered.restype = C.c_int64
    lib.oracle_num_rendered.argtypes = [C.c_void_p]
    lib.oracle_free.argtypes = [C.c_void_p]
    _LIBS[precision] = (lib, real)
    return _LIBS[precision]


def _view_struct(real):
    class OracleView(C.Structure):
        _fields_ = [
            ("H", C.c_int32), ("W", C.c_int32),
            ("tanfovx", real), ("tanfovy", real), ("cx", real), ("cy", real),
            ("scale_modifier", real), ("color_sigma", real),
            ("opaque_threshold", real), ("depth_threshold", real), ("normal_threshold", real), ("T_threshold", real),
            ("view", real * 16), ("proj", real * 16), ("campos", real * 3), ("bg", real * 3),
            ("sh_degree", C.c_int32), ("tie_eps", real),
        ]
    return OracleView


DEFAULTS = dict(  # SLAM/render.py:33-49,83-87 + configs/base.yaml:65-68
    scale_modifier=1.0, color_sigma=3.0, opaque_threshold=0.6, depth_threshold=1.0,
    normal_threshold=float(np.cos(np.deg2rad(60.0))), T_threshold=1e-4, sh_degree=3, bg=(0.0, 0.0, 0.0),
)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class OracleRender:
    """One forward evaluation; keeps the state `backward` needs (like the reference's ctx).

    `colors_precomp` (P,3) replaces the SH colour of g["shs"], `cov3D_precomp` (P,6) the covariance of g["scales"] /
    g["rotations"] (GaussianRasterizer's alternative inputs); the replaced entries of `g` are then not read."""

    def __init__(self, cam, g, tile_mask=None, precision="f32", tie_eps=0.0, nthreads=0, colors_precomp=None,
                 cov3D_precomp=None, **settings):
        lib, real = _lib(precision)
        self.lib, self.real, self.precision = lib, real, precision
        dt = np.float32 if precision == "f32" else np.float64
        self.dt = dt
        st = dict(DEFAULTS)
        st.update(settings)
        self.settings = st
        H, W = cam.height, cam.width
        self.H, self.W = H, W
        V = _view_struct(real)()
        V.H, V.W = H, W
        # the reference receives python floats -> C float; replicate the fp32 rounding in f32 mode
        V.tanfovx, V.tanfovy, V.cx, V.cy = cam.tanfovx, cam.tanfovy, cam.cx, cam.cy
        for k in ("scale_modifier", "color_sigma", "opaque_threshold", "depth_threshold", "normal_threshold", "T_threshold"):
            setattr(V, k, float(np.float32(st[k])) if precision == "f64" else st[k])
        if precision == "f64":  # same rounded inputs as the fp32 paths see
            V.tanfovx, V.tanfovy = float(np.float32(cam.tanfovx)), float(np.float32(cam.tanfovy))
            V.cx, V.cy = float(np.float32(cam.cx)), float(np.float32(cam.cy))
        V.view[:] = [float(x) for x in cam.viewmatrix.reshape(-1)]
        V.proj[:] = [float(x) for x in cam.projmatrix.reshape(-1)]
        V.campos[:] = [float(x) for x in cam.campos]
        V.bg[:] = [float(x) for x in st["bg"]]
        V.sh_degree = int(st["sh_degree"])
        V.tie_eps = tie_eps
        self.V = V
        self.P = P = g["xyz"].shape[0]
        arr = lambda a, *shape: None if a is None else np.ascontiguousarray(a, dtype=dt).reshape(P, *shape)
        self.colors_precomp, self.cov3D_precomp = arr(colors_precomp, 3), arr(cov3D_precomp, 6)
        self.means = np.ascontiguousarray(g["xyz"], dtype=dt)
        self.shs = arr(g["shs"], *g["shs"].shape[1:]) if colors_precomp is None else None
        self.M = M = self.shs.shape[1] if self.shs is not None else 0
        self.opac = np.ascontiguousarray(g["opacity"], dtype=dt).reshape(-1)
        self.scales = arr(g["scales"], 3) if cov3D_precomp is None else None
        self.rots = arr(g["rotations"], 4) if cov3D_precomp is None else None
        th, tw = (H + 15) // 16, (W + 15) // 16
        if tile_mask is None:
            tile_mask = np.ones((th, tw), dtype=np.int32)
        self.tile_mask = np.ascontiguousarray(tile_mask, dtype=np.int32)
        assert self.tile_mask.shape == (th, tw)
        self.color = np.empty((3, H, W), dt)
        self.depth = np.empty((1, H, W), dt)
        self.hit_color = np.empty((1, H, W), np.int32)
        self.hit_depth = np.empty((1, H, W), np.int32)
        self.hit_color_weight = np.empty((1, H, W), dt)
        self.hit_depth_weight = np.empty((1, H, W), dt)
        self.T_map = np.empty((1, H, W), dt)
        self.radii = np.empty((P,), np.int32)
        self.tie = np.zeros((H, W), np.uint8)
        self.state = lib.oracle_forward(
            C.byref(V), C.c_int(P), C.c_int(M), _p(self.means), _p(self.shs), _p(self.opac), _p(self.scales), _p(self.rots),
            _p(self.colors_precomp), _p(self.cov3D_precomp), _p(self.tile_mask), _p(self.color), _p(self.depth), _p(self.hit_color), _p(self.hit_depth),
            _p(self.hit_color_weight), _p(self.hit_depth_weight), _p(self.T_map), _p(self.radii),
            _p(self.tie) if tie_eps > 0 else None, C.c_int(nthreads))
        self.num_rendered = int(lib.oracle_num_rendered(self.state))

    def outputs(self):
        return (self.color, self.depth, self.hit_color, self.hit_depth, self.hit_color_weight, self.hit_depth_weight,
                self.T_map, self.radii)

    def geom(self):
        P, dt = self.P, self.dt
        d = dict(depth=np.empty(P, dt), xy=np.empty((P, 2), dt), conic_opacity=np.empty((P, 4), dt), rgb=np.empty((P, 3), dt),
                 clamped=np.empty((P, 3), np.uint8), tiles_touched=np.empty(P, np.int32), cov3D=np.empty((P, 6), dt))
        self.lib.oracle_get_geom(C.c_void_p(self.state), _p(d["depth"]), _p(d["xy"]), _p(d["conic_opacity"]), _p(d["rgb"]),
                                 _p(d["clamped"]), _p(d["tiles_touched"]), _p(d["cov3D"]))
        return d

    def binning(self):
        T = ((self.H + 15) // 16) * ((self.W + 15) // 16)
        pl = np.empty(max(self.num_rendered, 1), np.int32)
        rg = np.empty((T, 2), np.int64)
        self.lib.oracle_get_binning(C.c_void_p(self.state), _p(pl), _p(rg))
        return pl[: self.num_rendered], rg

    def image_state(self):
        N = self.H * self.W
        fT, nc = np.empty(N, self.dt), np.empty(N, np.int32)
        self.lib.oracle_get_image_state(C.c_void_p(self.state), _p(fT), _p(nc))
        return fT.reshape(self.H, self.W), nc.reshape(self.H, self.W)

    def backward(self, dL_dcolor, dL_ddepth, nthreads=0):
        """Returns dict of grads w.r.t. (means3D, shs, opacities, scales, rotations) + the 2-D intermediates. With
        precomputed colours "colors_precomp" (= the intermediate "colors") replaces "shs"; with a precomputed covariance
        "cov3D_precomp" (= the intermediate "cov3D") replaces "scales" and "rotations"."""
        P, M, dt = self.P, self.M, self.dt
        gc = np.ascontiguousarray(dL_dcolor, dtype=dt)
        gd = np.ascontiguousarray(dL_ddepth, dtype=dt)
        out = dict(means3D=np.empty((P, 3), dt), shs=np.empty((P, M, 3), dt), opacities=np.empty((P, 1), dt),
                   scales=np.empty((P, 3), dt), rotations=np.empty((P, 4), dt), means2D=np.empty((P, 3), dt),
                   conic=np.empty((P, 4), dt), colors=np.empty((P, 3), dt), cov3D=np.empty((P, 6), dt))
        self.lib.oracle_backward(C.c_void_p(self.state), _p(gc), _p(gd), _p(self.hit_depth), _p(out["means3D"]), _p(out["shs"]),
                                 _p(out["opacities"]), _p(out["scales"]), _p(out["rotations"]), _p(out["means2D"]),
                                 _p(out["conic"]), _p(out["colors"]), _p(out["cov3D"]), C.c_int(nthreads))
        if self.colors_precomp is not None:
            del out["shs"]
            out["colors_precomp"] = out["colors"]
        if self.cov3D_precomp is not None:
            del out["scales"], out["rotations"]
            out["cov3D_precomp"] = out["cov3D"]
        return out

    def close(self):
        if getattr(self, "state", None):
            self.lib.oracle_free(C.c_void_p(self.state))
            self.state = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
