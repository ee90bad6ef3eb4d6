"""ctypes binding of librtg_splat_b200.so (the C ABI declared in include/rtg_splat_b200.h).

There is no fallback: if the library is missing or a call fails, this raises."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
# RTG_SPLAT_LIB: developer knob for A/B-ing kernel variants built by tools/build_variant.py
LIB_PATH = os.environ.get("RTG_SPLAT_LIB") or os.path.join(HERE, "librtg_splat_b200.so")

RTG_CNT_WORDS = 8
RTG_ADAM_MAX_GROUPS = 8
RTG_FEATURES_MAX = 128  # channels of rtg_splat_features
# bits of RtgSplatView.prefiltered (a flags word)
RTG_VIEW_PREFILTERED, RTG_VIEW_ANTIALIASED = 1, 2


class RtgSplatView(C.Structure):
    _fields_ = [
        ("image_height", C.c_int32), ("image_width", C.c_int32),
        ("tanfovx", C.c_float), ("tanfovy", C.c_float),
        ("cx", C.c_float), ("cy", C.c_float),
        ("scale_modifier", C.c_float), ("color_sigma", C.c_float),
        ("opaque_threshold", C.c_float), ("depth_threshold", C.c_float),
        ("normal_threshold", C.c_float), ("T_threshold", C.c_float),
        ("sh_degree", C.c_int32), ("prefiltered", C.c_int32),
        ("viewmatrix", C.c_void_p), ("projmatrix", C.c_void_p), ("campos", C.c_void_p), ("bg", C.c_void_p),
    ]


class RtgAdamGroup(C.Structure):
    _fields_ = [
        ("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p),
        ("numel", C.c_int64), ("lr", C.c_float), ("_pad", C.c_float),
    ]


class RtgMapStep(C.Structure):
    """include/rtg_splat_b200.h: RtgMapStep (field order is the ABI)."""
    _fields_ = ([("P", C.c_int32), ("step", C.c_int32)]
                + [(n, C.c_void_p) for n in ("xyz", "sh", "opacity_raw", "scaling_raw", "rotation_raw",
                                             "m_xyz", "m_sh", "m_opacity", "m_scaling", "m_rotation",
                                             "v_xyz", "v_sh", "v_opacity", "v_scaling", "v_rotation",
                                             "g_means3D", "g_sh", "g_opacity", "g_scales", "g_rotations",
                                             "radii", "attach_mask", "xyz0", "scaling0", "rotation0")]
                + [("attach_weight", C.c_float), ("attach_count", C.c_int32)]
                + [(n, C.c_float) for n in ("lr_xyz", "lr_f_dc", "lr_f_rest", "lr_opacity", "lr_scaling", "lr_rotation",
                                            "beta1", "beta2", "eps")]
                + [(n, C.c_void_p) for n in ("scales_out", "rotations_out", "opacities_out", "normal_out", "confidence")])


class RtgHistoryMerge(C.Structure):
    """include/rtg_splat_b200.h: RtgHistoryMerge (field order is the ABI)."""
    _fields_ = ([("P", C.c_int32), ("max_weight", C.c_float)]
                + [(n, C.c_void_p) for n in ("hist_confidence", "confidence", "hist_xyz", "xyz", "hist_features_dc", "features_dc",
                                             "hist_features_rest", "features_rest", "hist_scaling", "scaling", "hist_rotation",
                                             "rotation_raw")]
                + [(n, C.c_int32) for n in ("features_dc_stride", "features_rest_stride", "features_rest_width", "_pad")])


class RtgPoseAdam(C.Structure):
    """include/rtg_splat_b200.h: RtgPoseAdam (field order is the ABI)."""
    _fields_ = ([(n, C.c_void_p) for n in ("pose", "exp_avg", "exp_avg_sq", "dL_dviewmatrix", "dL_dprojmatrix", "dL_dcampos",
                                           "projection", "viewmatrix", "projmatrix", "campos")]
                + [(n, C.c_float) for n in ("lr_trans", "lr_rot", "beta1", "beta2", "eps")]
                + [("step", C.c_int32)])


class RtgPoseGN(C.Structure):
    """include/rtg_splat_b200.h: RtgPoseGN (field order is the ABI)."""
    _fields_ = ([(n, C.c_void_p) for n in ("pose", "projection", "viewmatrix", "projmatrix", "campos", "render", "depth", "hit_depth",
                                           "gt_color", "gt_depth", "render_mask", "scratch", "report")]
                + [(n, C.c_float) for n in ("color_weight", "depth_weight", "depth_error_max", "damping")]
                + [("gt_channels_last", C.c_int32), ("_pad", C.c_int32)])


RTG_POSE_GN_REPORT_LEN = 8
POSE_GN_STATUS = {0: "ok", 1: "singular", 2: "empty", 3: "overflow"}


class RtgPoseRobust(C.Structure):
    """include/rtg_splat_b200.h: RtgPoseRobust (field order is the ABI)."""
    _fields_ = [("kernel", C.c_int32), ("color_delta", C.c_float), ("depth_delta", C.c_float), ("_pad", C.c_int32)]


RTG_ROBUST_NONE, RTG_ROBUST_HUBER = 0, 1


class RtgPoseExposure(C.Structure):
    """include/rtg_splat_b200.h: RtgPoseExposure (field order is the ABI)."""
    _fields_ = [("ab", C.c_void_p)]


class RtgMapTransform(C.Structure):
    """include/rtg_splat_b200.h: RtgMapTransform (field order is the ABI)."""
    _fields_ = ([(n, C.c_int32) for n in ("P", "K", "sh_rest", "_pad")]
                + [(n, C.c_void_p) for n in ("anchor", "old_c2w", "new_c2w", "xyz", "rotation", "normal", "features_rest",
                                             "n_skipped")])


class RtgTsdfVolume(C.Structure):
    """include/rtg_splat_b200.h: RtgTsdfVolume (field order is the ABI)."""
    _fields_ = ([(n, C.c_int32) for n in ("nx", "ny", "nz")] + [("voxel_size", C.c_float), ("trunc", C.c_float),
                                                               ("origin", C.c_float * 3)]
                + [(n, C.c_void_p) for n in ("tsdf", "weight", "color")])


class RtgIcpLevel(C.Structure):
    _fields_ = [("vertex0", C.c_void_p), ("normal0", C.c_void_p), ("vertex1", C.c_void_p), ("normal1", C.c_void_p),
                ("H", C.c_int32), ("W", C.c_int32), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float),
                ("iters", C.c_int32), ("_pad", C.c_int32)]


# name -> (restype, argtypes); must list every symbol of include/rtg_splat_b200.h
_VP, _I32, _I64, _F = C.c_void_p, C.c_int32, C.c_int64, C.c_float
_BWD_ARGS = [C.POINTER(RtgSplatView), _I32, _I32] + [_VP] * 6 + [_VP, _VP, _VP, _VP, _I64, _VP] + [_VP] * 4 + [_VP] + [_VP] * 8 + [_VP]
SIGNATURES = {
    "rtg_last_error": (C.c_char_p, []),
    "rtg_version": (C.c_int, []),
    "rtg_splat_workspace_bytes": (C.c_int, [_I32, _I32, _I32, _I64, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "rtg_splat_forward": (C.c_int, [C.POINTER(RtgSplatView), _I32, _I32] + [_VP] * 8 + [_VP, _VP, _VP, _I64] + [_VP] * 8 + [_VP, _VP, _VP, _VP]),
    "rtg_splat_backward": (C.c_int, _BWD_ARGS),
    "rtg_splat_backward_visible": (C.c_int, _BWD_ARGS),
    "rtg_splat_backward_render": (C.c_int, _BWD_ARGS),
    "rtg_splat_backward_finish": (C.c_int, _BWD_ARGS),
    "rtg_splat_camera_scratch_bytes": (C.c_size_t, [_I32]),
    "rtg_splat_backward_camera": (C.c_int, _BWD_ARGS[:-1] + [_I32, _VP, _VP, _VP]),
    "rtg_splat_geom_layout": (C.c_int, [_I32] + [C.POINTER(C.c_size_t)] * 4),
    "rtg_splat_forward_preprocess": (C.c_int, [C.POINTER(RtgSplatView), _I32, _I32, _I32, _I32] + [_VP] * 7 + [_VP, _VP, _I64, _VP, _VP]),
    "rtg_splat_forward_render": (C.c_int, [C.POINTER(RtgSplatView), _I32, _VP, _VP, _VP, _VP, _I64] + [_VP] * 7 + [_VP, _VP, _VP, _VP, _I32, _I32, _VP]),
    "rtg_splat_backward_render_shard": (C.c_int, [_I32, _I32] + _BWD_ARGS),
    "rtg_splat_backward_finish_shard": (C.c_int, [_I32, _I32] + _BWD_ARGS),
    # _BWD_ARGS with dL_dT after dL_ddepth (argument 19)
    "rtg_splat_backward_dt": (C.c_int, _BWD_ARGS[:19] + [_VP] + _BWD_ARGS[19:-1] + [_I32, _VP, _VP, _VP]),
    "rtg_splat_backward_render_dt": (C.c_int, [_I32, _I32] + _BWD_ARGS[:19] + [_VP] + _BWD_ARGS[19:]),
    # rtg_splat_backward_dt's arguments up to grad2d_scratch, then dL_dcamera, camera_scratch, stream
    "rtg_splat_backward_pose": (C.c_int, _BWD_ARGS[:19] + [_VP, _VP] + [_VP, _VP, _VP]),
    "rtg_pose_adam_step": (C.c_int, [C.POINTER(RtgPoseAdam), _VP]),
    "rtg_splat_pose_gn_scratch_bytes": (C.c_size_t, [_I32, _I32, _I32]),
    # view, P, M, 6 Gaussian inputs, 3 workspaces, R_cap, counters, then hit_image, scratch, J / the step's state, stream
    "rtg_splat_pose_tangents": (C.c_int, [C.POINTER(RtgSplatView), _I32, _I32] + [_VP] * 6 + [_VP] * 3 + [_I64, _VP] + [_VP] * 4),
    # view, P, the three workspaces, R_cap, counters, pixel_error, n_pixels, weight, error, stream
    "rtg_splat_contributions": (C.c_int, [C.POINTER(RtgSplatView), _I32] + [_VP] * 3 + [_I64, _VP] + [_VP] * 4 + [_VP]),
    # view, P, the three workspaces, R_cap, counters, C, input (features / dL_dout), output, stream
    "rtg_splat_features": (C.c_int, [C.POINTER(RtgSplatView), _I32] + [_VP] * 3 + [_I64, _VP, _I32] + [_VP] * 3),
    "rtg_splat_features_backward": (C.c_int, [C.POINTER(RtgSplatView), _I32] + [_VP] * 3 + [_I64, _VP, _I32] + [_VP] * 3),
    # view, P, means3D, scales, rotations, cov3D_precomp, radii, the three workspaces, R_cap, counters, C, features, dL_dout,
    # grad2d_scratch, five per-Gaussian gradients, visible_rows_only, dL_dcamera, camera_scratch, stream
    "rtg_splat_features_backward_geometry": (C.c_int, [C.POINTER(RtgSplatView), _I32] + [_VP] * 5 + [_VP] * 3 + [_I64, _VP, _I32]
                                             + [_VP] * 3 + [_VP] * 5 + [_I32, _VP, _VP, _VP]),
    "rtg_splat_pose_gn_step": (C.c_int, [C.POINTER(RtgSplatView), _I32, _I32] + [_VP] * 6 + [_VP] * 3 + [_I64, _VP]
                               + [C.POINTER(RtgPoseGN), _VP]),
    "rtg_splat_pose_gn_step_robust": (C.c_int, [C.POINTER(RtgSplatView), _I32, _I32] + [_VP] * 6 + [_VP] * 3 + [_I64, _VP]
                                      + [C.POINTER(RtgPoseGN), C.POINTER(RtgPoseRobust), _VP]),
    "rtg_splat_pose_gn_exposure_scratch_bytes": (C.c_size_t, [_I32, _I32, _I32]),
    "rtg_splat_pose_gn_step_exposure": (C.c_int, [C.POINTER(RtgSplatView), _I32, _I32] + [_VP] * 6 + [_VP] * 3 + [_I64, _VP]
                                        + [C.POINTER(RtgPoseGN), C.POINTER(RtgPoseRobust), C.POINTER(RtgPoseExposure), _VP]),
    # view, P, M, 6 Gaussian inputs, 3 workspaces, R_cap, counters, scratch, J, expected, stream
    "rtg_splat_pose_tangents_expected": (C.c_int, [C.POINTER(RtgSplatView), _I32, _I32] + [_VP] * 6 + [_VP] * 3 + [_I64, _VP]
                                         + [_VP] * 4),
    "rtg_splat_pose_gn_step_expected": (C.c_int, [C.POINTER(RtgSplatView), _I32, _I32] + [_VP] * 6 + [_VP] * 3 + [_I64, _VP]
                                        + [C.POINTER(RtgPoseGN), C.POINTER(RtgPoseRobust), C.POINTER(RtgPoseExposure), _F,
                                           _VP]),
    "rtg_splat_mark_visible": (C.c_int, [_I32, _VP, _VP, _VP, _VP, _VP]),
    "rtg_adam_step": (C.c_int, [C.POINTER(RtgAdamGroup), _I32, _F, _F, _F, _I32, _VP]),
    "rtg_map_adam_step": (C.c_int, [C.POINTER(RtgMapStep), _VP]),
    "rtg_map_activate": (C.c_int, [_I32] + [_VP] * 8),
    "rtg_map_history_merge": (C.c_int, [C.POINTER(RtgHistoryMerge), _VP]),
    "rtg_icp_workspace_bytes": (C.c_size_t, [_I32, _I32]),
    "rtg_icp_build_level": (C.c_int, [_VP, _I32, _I32, _I32, _F, _F, _F, _F, _VP, _VP, _VP, _VP]),
    "rtg_icp_solve_level": (C.c_int, [_VP, _VP, _VP, _VP, _I32, _I32, _F, _F, _F, _F, _F, _F, _F, _I32, _VP, _VP, _VP, _VP]),
    "rtg_icp_build_pyramid": (C.c_int, [_VP, _I32, _I32, _I32, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "rtg_icp_predict_pose": (C.c_int, [_VP, _I32, _F, _F, _F, _VP, _VP, _VP, _VP, _I32, _I32, _VP, _VP, _VP, _VP]),
    # color, H, W, channels_last, n_levels, pools, intensity_out, stream
    "rtg_icp_build_intensity_pyramid": (C.c_int, [_VP, _I32, _I32, _I32, _I32, _VP, _VP, _VP]),
    # levels, intensity0, intensity1, then rtg_icp_predict_pose's arguments with photometric_weight after damping
    "rtg_icp_predict_pose_rgbd": (C.c_int, [_VP, _VP, _VP, _I32, _F, _F, _F, _F, _VP, _VP, _VP, _VP, _I32, _I32, _VP, _VP, _VP,
                                            _VP]),
    "rtg_icp_point2plane_loss": (C.c_int, [_VP, _VP, _VP, _I32, _I32, _VP, _VP, _VP, _VP]),
    "rtg_icp_fill_model_depth": (C.c_int, [_VP, _VP, _VP, _VP, _I32, _I32, _F, _F, _VP]),
    "rtg_loss_workspace_bytes": (C.c_size_t, []),
    "rtg_loss_l1": (C.c_int, [_VP] * 6 + [_I32, _I32, _I32, _F, _F, _F, _VP, _VP, _VP, _VP, _VP]),
    # rtg_loss_l1's arguments with exposure before the gradients and dL_dexposure after them
    "rtg_loss_l1_exposure_workspace_bytes": (C.c_size_t, []),
    "rtg_loss_l1_exposure": (C.c_int, [_VP] * 6 + [_I32, _I32, _I32, _F, _F, _F, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "rtg_loss_mapping": (C.c_int, [_VP] * 8 + [_I32, _I32, _I32, _F, _F, _F, _F, _VP, _VP, _VP, _VP, _VP, _VP]),
    # rtg_loss_mapping's arguments with exposure after depth_error_max and dL_dexposure after dL_dnormal
    "rtg_loss_mapping_exposure": (C.c_int, [_VP] * 8 + [_I32, _I32, _I32, _F, _F, _F, _F, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "rtg_ssim_workspace_bytes": (C.c_size_t, [_I32, _I32, _I32]),
    "rtg_ssim_loss": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _VP, _VP, _VP, _VP]),
    "rtg_ssim_exposure_workspace_bytes": (C.c_size_t, [_I32, _I32, _I32]),
    # img1, img2, C, H, W, exposure, dL_dimg1, dL_dexposure, loss_out, ws, stream
    "rtg_ssim_loss_exposure": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _VP, _VP, _VP, _VP, _VP, _VP]),
    "rtg_normal_map": (C.c_int, [_VP, _VP, _I32, _I32, _VP, _VP]),
    "rtg_frame_preprocess": (C.c_int, [_VP, _I32, _I32, _I32, _I32] + [_F] * 9 + [_VP] * 7),
    # color, depth, render_mask, tile_mask, H, W, scale, color_channels_last, 4 outputs, stream
    "rtg_frame_downsample": (C.c_int, [_VP] * 4 + [_I32] * 4 + [_VP] * 4 + [_VP]),
    "rtg_accumulate_gaussian_error": (C.c_int, [_I32, _I32, _I32] + [_VP] * 5 + [_F, _F, _F, _I32] + [_VP] * 6),
    "rtg_tile_mean": (C.c_int, [_I32, _I32, _VP, _F, _VP, _VP, _VP]),
    "rtg_transmission_tile_mask": (C.c_int, [_I32, _I32, _VP, _F, _VP, _VP, _VP]),
    "rtg_color_error": (C.c_int, [_I32, _I32, _VP, _VP, _VP, _VP]),
    "rtg_soa_compact_workspace_bytes": (C.c_size_t, [_I64]),
    "rtg_soa_compact": (C.c_int, [_VP, _I32, _I64, _I32, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "rtg_knn_workspace_bytes": (C.c_size_t, [_I64]),
    "rtg_knn": (C.c_int, [_VP, _I64, _VP, _I64, _I32, _I32, _VP, _VP, _VP, _VP, _VP]),
    "rtg_map_transform_workspace_bytes": (C.c_size_t, [_I32]),
    "rtg_map_transform": (C.c_int, [C.POINTER(RtgMapTransform), _VP, _VP]),
    # vol, depth, color, H, W, color_channels_last, fx, fy, cx, cy, w2c, w2c_is_double, stream
    "rtg_tsdf_integrate": (C.c_int, [C.POINTER(RtgTsdfVolume), _VP, _VP, _I32, _I32, _I32, _F, _F, _F, _F, _VP, _I32, _VP]),
    # vol, w2c, w2c_is_double, H, W, fx, fy, cx, cy, depth, normal, color, stream
    "rtg_tsdf_raycast": (C.c_int, [C.POINTER(RtgTsdfVolume), _VP, _I32, _I32, _I32, _F, _F, _F, _F, _VP, _VP, _VP, _VP]),
    "rtg_tsdf_extract_workspace_bytes": (C.c_size_t, [_I32, _I32, _I32]),
    "rtg_tsdf_extract_count": (C.c_int, [C.POINTER(RtgTsdfVolume), _VP, _VP, _VP]),
    "rtg_tsdf_extract_emit": (C.c_int, [C.POINTER(RtgTsdfVolume), _VP, _VP, _VP, _VP, _VP]),
    "rtg_profile_enable": (C.c_int, [_I32]),
    "rtg_profile_kernel_count": (C.c_int, []),
    "rtg_profile_kernel_name": (C.c_char_p, [_I32]),
    "rtg_profile_read": (C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_int64), _I32]),
}

_lib = None


class RtgError(RuntimeError):
    pass


def lib():
    """Loads the shared library (building is __graft_entry__.build()'s job, not done implicitly here)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RtgError(
            f"{LIB_PATH} is missing: the sm_90a extension has not been built. Run `python -m rtg_slam_b200.build` "
            "(or __graft_entry__.build()). There is no CPU or PyTorch fallback for this path.")
    h = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(h, name)  # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = h
    return h


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().rtg_last_error()
        raise RtgError(f"{what} failed ({rc}): {msg.decode() if msg else ''}")


def header_symbols():
    """Names of all functions declared in include/rtg_splat_b200.h (used by the ABI test)."""
    import re
    hdr = os.path.join(HERE, "..", "include", "rtg_splat_b200.h")
    txt = open(hdr).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(rtg_[a-z0-9_]+)\s*\(", txt)))


def profile_enable(on: bool) -> None:
    check(lib().rtg_profile_enable(1 if on else 0), "rtg_profile_enable")


def profile_read(reset: bool = True) -> dict:
    """{kernel name: (total ms, launches)} since the last reset (synchronises the device)."""
    L = lib()
    n = L.rtg_profile_kernel_count()
    ms = (C.c_double * n)()
    cnt = (C.c_int64 * n)()
    check(L.rtg_profile_read(ms, cnt, 1 if reset else 0), "rtg_profile_read")
    return {L.rtg_profile_kernel_name(i).decode(): (ms[i], int(cnt[i])) for i in range(n)}
