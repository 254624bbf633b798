"""ctypes binding of include/dfusion.h (libdfusion.so).

This is the only way Python reaches the CUDA kernels: plain pointers and sizes, no torch types cross the
boundary.  torch is used by callers for device memory and streams only.  The loader FAILS LOUDLY when the
library is missing -- there is no CPU fallback in the product path.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_HERE = Path(__file__).resolve().parent
# DF_LIB_VARIANT=<tag> loads libdfusion_<tag>.so instead (instrumented / A-B builds made by tools/build_variant.py; measurement only)
_LIB_PATH = _HERE / (f"libdfusion_{os.environ['DF_LIB_VARIANT']}.so" if os.environ.get("DF_LIB_VARIANT") else "libdfusion.so")
_lib = None
MISSING: list[str] = []


class Volume(C.Structure):
    _fields_ = [("data", C.c_void_p), ("dims", C.c_int * 3), ("voxel_size", C.c_float * 3),
                ("trunc_dist", C.c_float), ("max_weight", C.c_int)]


class Aff3f(C.Structure):
    _fields_ = [("R", C.c_float * 9), ("t", C.c_float * 3)]


class Intr(C.Structure):
    _fields_ = [("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float)]


class ColorCamera(C.Structure):
    """df_color_camera (include/dfusion.h): a colour camera with its own size, intrinsics and pose relative to the depth camera"""
    _fields_ = [("cols", C.c_int), ("rows", C.c_int), ("intr", Intr), ("depth_to_color", Aff3f)]


class Lens(C.Structure):
    """df_lens (include/dfusion.h): lens distortion coefficients in OpenCV's order and the squared normalised radius they hold over"""
    _fields_ = [("k1", C.c_float), ("k2", C.c_float), ("p1", C.c_float), ("p2", C.c_float), ("k3", C.c_float), ("k4", C.c_float),
                ("k5", C.c_float), ("k6", C.c_float), ("r2_max", C.c_float)]

    def coeffs(self) -> tuple:
        return (self.k1, self.k2, self.p1, self.p2, self.k3, self.k4, self.k5, self.k6)


class KinfuParams(C.Structure):
    """df_kinfu_params (include/dfusion.h) == KinFuParams, kinfu.hpp:15-47"""
    _fields_ = [("cols", C.c_int), ("rows", C.c_int), ("intr", Intr),
                ("volume_dims", C.c_int * 3), ("volume_size", C.c_float * 3), ("volume_pose", Aff3f),
                ("bilateral_sigma_depth", C.c_float), ("bilateral_sigma_spatial", C.c_float), ("bilateral_kernel_size", C.c_int),
                ("icp_truncate_depth_dist", C.c_float), ("icp_dist_thres", C.c_float), ("icp_angle_thres", C.c_float),
                ("icp_iter_num", C.c_int * 4),
                ("tsdf_min_camera_movement", C.c_float), ("tsdf_trunc_dist", C.c_float), ("tsdf_max_weight", C.c_int),
                ("raycast_step_factor", C.c_float), ("gradient_delta_factor", C.c_float),
                ("light_pose", C.c_float * 3),
                ("solver_nonlinear_iters", C.c_int), ("solver_linear_iters", C.c_int),
                ("max_nodes", C.c_int), ("node_step", C.c_int), ("cloud_capacity", C.c_int), ("flags", C.c_int),
                ("fusion_weight_scale", C.c_float), ("extend_radius", C.c_float)]


class RelocGate(C.Structure):
    """df_reloc_gate (include/dfusion.h): the ICP's T and ok and the gate's counts"""
    _fields_ = [("T", C.c_float * 12), ("ok", C.c_int), ("n_valid", C.c_int), ("n_in", C.c_int), ("pad", C.c_int), ("sum_sq", C.c_double)]


# include/dfusion.h DF_RELOC_*: the relocaliser's constants
RELOC_FERNS = 500
RELOC_CANDIDATES = 3
RELOC_KEYFRAMES = 512
RELOC_NEAR_MM = 400
RELOC_FAR_MM = 3000
RELOC_SEED = 0x5eedf00d
RELOC_HARVEST_FERNS = 40
RELOC_MIN_VALID = 5000
RELOC_MIN_INLIER_FRAC = 0.1
RELOC_MAX_RMS = 0.03
RELOC_GATE_WS_BYTES = 4096


class RelocMatch(C.Structure):
    """df_reloc_match (include/dfusion.h): the lookup's candidates, the append and the database's count"""
    _fields_ = [("index", C.c_int * RELOC_CANDIDATES), ("dissimilarity", C.c_int * RELOC_CANDIDATES), ("appended", C.c_int), ("count", C.c_int),
                ("pose", (C.c_float * 12) * RELOC_CANDIDATES)]


class F2Params(C.Structure):
    """df_f2_params (include/dfusion.h)"""
    _fields_ = [("reg_lambda", C.c_double), ("tukey_c", C.c_double), ("huber_delta", C.c_double), ("lm_mu", C.c_double),
                ("gn_iters", C.c_int), ("reg_k", C.c_int), ("flags", C.c_int), ("lin_iters", C.c_int)]


_vp, _sz, _i, _f = C.c_void_p, C.c_size_t, C.c_int, C.c_float

# name -> (restype, argtypes); must list every symbol declared in include/dfusion.h
PROTOTYPES = {
    "df_error_string": (C.c_char_p, [_i]),
    "df_version": (_i, []),
    "df_clear_volume": (_i, [Volume, _vp]),
    "df_compute_dists": (_i, [_vp, _sz, _i, _i, Intr, _vp, _sz, _vp]),
    "df_integrate": (_i, [Volume, _vp, _sz, _i, _i, Aff3f, Intr, _vp, _vp]),
    "df_volume_activity_bytes": (_sz, [Volume]),
    "df_integrate_workspace_bytes": (_sz, [_i, _i]),
    "df_integrate_launch_count": (_i, [Volume]),
    "df_integrate_last_kernel": (_i, []),
    "df_integrate_selftest": (_i, [_vp, _vp]),
    "df_integrate_tracked": (_i, [Volume, _vp, _sz, _i, _i, Aff3f, Intr, _vp, _vp, _vp, _vp]),
    "df_raycast_points": (_i, [Volume, Aff3f, C.POINTER(C.c_float), Intr, _i, _i, _f, _f, _vp, _sz, _vp, _sz, _vp]),
    "df_raycast_points_tracked": (_i, [Volume, Aff3f, C.POINTER(C.c_float), Intr, _i, _i, _f, _f, _vp, _sz, _vp, _sz, _vp, _vp]),
    "df_raycast_points_stats_tracked": (_i, [Volume, Aff3f, C.POINTER(C.c_float), Intr, _i, _i, _f, _f, _vp, _sz, _vp, _sz, _vp, _vp, _vp, _vp]),
    "df_raycast_touched_bytes": (_sz, [Volume]),
    "df_raycast_points_stats": (_i, [Volume, Aff3f, C.POINTER(C.c_float), Intr, _i, _i, _f, _f, _vp, _sz, _vp, _sz, _vp, _vp, _vp]),
    "df_project_workspace_bytes": (_sz, [_i, _i]),
    "df_project_and_remove": (_i, [_vp, _sz, _i, _i, Intr, _vp, _sz, _i, _i, _vp, _vp]),
    "df_extract_workspace_bytes": (_sz, [Volume]),
    "df_extract_cloud": (_i, [Volume, Aff3f, _vp, _i, _vp, _vp, _vp]),
    "df_extract_cloud_tracked": (_i, [Volume, Aff3f, _vp, _i, _vp, _vp, _vp, _vp]),
    "df_extract_normals": (_i, [Volume, _vp, _i, _vp, Aff3f, C.POINTER(C.c_float), _f, _vp, _vp]),
    "df_bilateral": (_i, [_vp, _sz, _i, _i, _vp, _sz, _i, _f, _f, _vp]),
    "df_truncate_depth": (_i, [_vp, _sz, _i, _i, _f, _vp]),
    "df_pyr_down": (_i, [_vp, _sz, _i, _i, _vp, _sz, _f, _vp]),
    "df_points_normals": (_i, [Intr, _vp, _sz, _i, _i, _vp, _sz, _vp, _sz, _vp]),
    "df_resize_points_normals": (_i, [_vp, _sz, _vp, _sz, _i, _i, _vp, _sz, _vp, _sz, _vp]),
    "df_render_image": (_i, [_vp, _sz, _vp, _sz, _i, _i, C.POINTER(C.c_float), _vp, _sz, _vp]),
    "df_render_tangent_colors": (_i, [_vp, _sz, _i, _i, _vp, _sz, _vp]),
    "df_render_image_depth": (_i, [_vp, _sz, _vp, _sz, _i, _i, Intr, C.POINTER(C.c_float), _vp, _sz, _vp]),
    "df_normals_mask_depth": (_i, [Intr, _vp, _sz, _i, _i, _vp, _sz, _vp]),
    "df_cloud_to_depth": (_i, [_vp, _sz, _i, _i, _vp, _sz, _vp]),
    "df_resize_depth_normals": (_i, [_vp, _sz, _vp, _sz, _i, _i, _vp, _sz, _vp, _sz, _vp]),
    "df_icp_accumulate": (_i, [_vp, _sz, _vp, _sz, _vp, _sz, _vp, _sz, _i, _i, Intr, Aff3f, _f, _f, _vp, _vp]),
    "df_icp_estimate": (_i, [C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_i), C.POINTER(_i),
                             C.POINTER(_sz), _i, C.POINTER(_i), Intr, _f, _f, _vp, _vp, _vp, _vp]),
    "df_icp_accumulate_depth": (_i, [_vp, _sz, _vp, _sz, _vp, _sz, _vp, _sz, _i, _i, Intr, Aff3f, _f, _f, _vp, _vp]),
    "df_icp_estimate_depth": (_i, [C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_i), C.POINTER(_i),
                                   C.POINTER(_sz), C.POINTER(_sz), _i, C.POINTER(_i), Intr, _f, _f, _vp, _vp, _vp, _vp]),
    "df_icp_solve_step": (_i, [_vp, _i, _vp, _vp, _vp]),
    "df_knn8": (_i, [_vp, _i, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "df_node_grid_bytes": (_sz, [_i]),
    "df_build_node_grid": (_i, [_vp, _i, _vp, _vp]),
    "df_extend_field_workspace_bytes": (_sz, [_i]),
    "df_extend_field": (_i, [_vp, _i, _i, _vp, _vp, _i, _vp, _i, _f, _i, _vp, _vp, _vp]),
    "df_warp": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, Aff3f, _i, _vp, _vp, _vp]),
    "df_integrate_warped_workspace_bytes": (_sz, [_i, _i, _i]),
    "df_integrate_warped_launch_count": (_i, []),
    "df_integrate_warped": (_i, [Volume, _vp, _sz, _i, _i, Aff3f, Aff3f, Intr, _vp, _i, _vp, _f, _vp, _vp, _vp, _vp]),
    "df_integrate_warped_color": (_i, [Volume, _vp, _sz, _i, _i, Aff3f, Aff3f, Intr, _vp, _i, _vp, _f, _vp, _vp, _vp, _vp, _vp, _sz,
                                       C.POINTER(ColorCamera), C.POINTER(Lens), _vp, _sz, _vp]),
    "df_solve_workspace_bytes": (_sz, [_i, _i]),
    "df_solve_knn_buffers": (_i, [_vp, _i, _i, C.POINTER(_vp), C.POINTER(_vp)]),
    "df_solve_normal_system": (_i, [_vp, _i, _i, C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp)]),
    "df_solve_data_term": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "df_solve_f2_workspace_bytes": (_sz, [_i, _i, _i]),
    "df_solve_f2": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, C.POINTER(F2Params), _vp, _vp, _vp]),
    "df_kinfu_set_f2_params": (_i, [_vp, C.POINTER(F2Params)]),
    "df_kinfu_default_params": (None, [C.POINTER(KinfuParams), _i]),
    "df_kinfu_create": (_vp, [C.POINTER(KinfuParams)]),
    "df_kinfu_destroy": (None, [_vp]),
    "df_kinfu_reset": (_i, [_vp]),
    "df_kinfu_process_host": (_i, [_vp, _vp, _sz]),
    "df_kinfu_batch_process_host": (_i, [C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_sz), _i, C.POINTER(_i)]),
    "df_kinfu_process_device": (_i, [_vp, _vp, _sz]),
    "df_kinfu_get_stage_ms": (_i, [_vp, C.POINTER(C.c_float), _i]),
    "df_kinfu_dynamicfusion": (_i, [_vp, _vp, _sz, _vp, _sz]),
    "df_kinfu_get_pose": (_i, [_vp, _i, C.POINTER(C.c_float)]),
    "df_kinfu_get_info": (_i, [_vp, C.POINTER(C.c_longlong), _i]),
    "df_kinfu_get_buffer": (_i, [_vp, _i, C.POINTER(_vp), C.POINTER(_sz), C.POINTER(_i), C.POINTER(_i)]),
    "df_kinfu_set_stream": (_i, [_vp, _vp]),
    "df_kinfu_read_buffer": (_i, [_vp, _i, _vp, _sz]),
    "df_kinfu_join": (_i, [_vp]),
    "df_kinfu_set_overrides": (_i, [_vp, _vp, _sz, _vp, _vp, _i]),
    "df_kinfu_state_digest": (_i, [_vp, C.POINTER(C.c_ulonglong)]),
    "df_volume_brick_count": (_sz, [Volume]),
    "df_volume_pack_workspace_bytes": (_sz, [Volume]),
    "df_volume_pack_count": (_i, [Volume, _vp, _vp, _vp, _vp]),
    "df_volume_pack_emit": (_i, [Volume, _vp, _vp, _vp, _sz, _vp]),
    "df_volume_unpack": (_i, [Volume, _vp, _vp, _sz, _vp, _vp, _vp]),
    "df_kinfu_save": (_i, [_vp, _vp, _sz, C.POINTER(_sz)]),
    "df_kinfu_load": (_i, [_vp, _vp, _sz]),
    "df_kinfu_snapshot_params": (_i, [_vp, _sz, C.POINTER(KinfuParams)]),
    "df_mesh_workspace_bytes": (_sz, [Volume]),
    "df_mesh_count": (_i, [Volume, _vp, _vp, _vp, _vp, _vp, _vp]),
    "df_mesh_emit": (_i, [Volume, _vp, _vp, _vp, _i, _vp]),
    "df_kinfu_mesh": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, C.POINTER(_i), C.POINTER(_i)]),
    "df_raster_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "df_raster_mesh": (_i, [_vp, _i, _i, _vp, _i, Aff3f, Intr, _i, _i, _vp, _sz, _vp, _sz, _vp, _sz, _vp, _vp, _vp]),
    "df_mesh_correspond": (_i, [_vp, _sz, _vp, _sz, _vp, _vp, _i, _i, _vp, _i, Aff3f, _i, _i, _vp, _sz, _f, _vp, _sz, _vp, _sz, _vp]),
    "df_kinfu_render":(_i, [_vp, _i, C.POINTER(C.c_float), _vp, _sz, _vp, _sz, _vp, _sz]),
    "df_integrate_color": (_i, [Volume, _vp, _vp, _sz, _vp, _sz, _i, _i, Aff3f, Intr, _vp, _vp]),
    "df_sample_colors": (_i, [Volume, _vp, Aff3f, _f, _vp, _sz, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "df_mesh_colors": (_i, [_vp, _sz, _vp, _sz, _vp, _i, _i, _vp, _i, Aff3f, _vp, _i, _i, _vp, _sz, _vp]),
    "df_kinfu_process_host_color": (_i, [_vp, _vp, _sz, _vp, _sz]),
    "df_kinfu_process_device_color": (_i, [_vp, _vp, _sz, _vp, _sz]),
    "df_kinfu_mesh_colors": (_i, [_vp, _vp, _i, C.POINTER(_i)]),
    "df_kinfu_render_colors": (_i, [_vp, _i, C.POINTER(C.c_float), _vp, _sz]),
    "df_color_map_dims": (_i, [Intr, ColorCamera, C.POINTER(_i), C.POINTER(_i), C.POINTER(_i)]),
    "df_color_depth_map": (_i, [_vp, _sz, _i, _i, Intr, ColorCamera, _vp, _sz, _vp]),
    "df_integrate_color_camera": (_i, [Volume, _vp, _vp, _sz, _i, _i, Aff3f, Intr, ColorCamera, _vp, _sz, _vp, _sz, _vp, _vp]),
    "df_kinfu_set_color_camera": (_i, [_vp, C.POINTER(ColorCamera)]),
    "df_kinfu_snapshot_color_camera": (_i, [_vp, _sz, C.POINTER(ColorCamera), C.POINTER(_i)]),
    "df_frame_intensity": (_i, [_vp, _sz, C.POINTER(ColorCamera), Intr, _vp, _sz, _vp, _sz, _f, _i, C.POINTER(_i), C.POINTER(_i), C.POINTER(_vp),
                                C.POINTER(_sz), _vp]),
    "df_model_intensity": (_i, [Volume, _vp, Aff3f, _i, C.POINTER(_i), C.POINTER(_i), C.POINTER(_vp), C.POINTER(_sz), C.POINTER(_vp),
                                C.POINTER(_sz), _vp]),
    "df_lens_check": (_i, [Lens]),
    "df_undistort": (_i, [_vp, _sz, _vp, _sz, _vp, _sz, _vp, _sz, _i, _i, Intr, Lens, _vp]),
    "df_color_depth_map_lens": (_i, [_vp, _sz, _i, _i, Intr, ColorCamera, C.POINTER(Lens), _vp, _sz, _vp]),
    "df_integrate_color_camera_lens": (_i, [Volume, _vp, _vp, _sz, _i, _i, Aff3f, Intr, ColorCamera, C.POINTER(Lens), _vp, _sz, _vp, _sz, _vp,
                                            _vp]),
    "df_frame_intensity_lens": (_i, [_vp, _sz, C.POINTER(ColorCamera), C.POINTER(Lens), Intr, _vp, _sz, _vp, _sz, _f, _i, C.POINTER(_i),
                                     C.POINTER(_i), C.POINTER(_vp), C.POINTER(_sz), _vp]),
    "df_kinfu_set_depth_lens": (_i, [_vp, C.POINTER(Lens)]),
    "df_kinfu_set_color_lens": (_i, [_vp, C.POINTER(Lens)]),
    "df_kinfu_snapshot_lenses": (_i, [_vp, _sz, C.POINTER(Lens), C.POINTER(_i), C.POINTER(Lens), C.POINTER(_i)]),
    "df_icp_accumulate_color": (_i, [_vp, _sz, _vp, _sz, _vp, _sz, _vp, _sz, _vp, _sz, _vp, _sz, _i, _i, Intr, Aff3f, _f, _f, _f, _f, _vp, _vp]),
    "df_icp_estimate_color": (_i, [C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_sz),
                                   C.POINTER(_vp), C.POINTER(_sz), C.POINTER(_i), C.POINTER(_i), C.POINTER(_sz), _i, C.POINTER(_i), Intr, _f,
                                   _f, _f, _f, _vp, _vp, _vp, _vp]),
    "df_reloc_fern_table": (_i, [C.c_ulonglong, _i, _i, _i, _vp]),
    "df_fern_encode": (_i, [_vp, _sz, _i, _i, _vp, _i, _vp, _vp]),
    "df_fern_match": (_i, [_vp, _vp, _vp, _i, _vp, _i, _i, Aff3f, _vp, _vp]),
    "df_icp_inliers": (_i, [_vp, _sz, _vp, _sz, _vp, _sz, _vp, _sz, _i, _i, Intr, _vp, _vp, _f, _f, _vp, _vp, _vp]),
    "df_reloc_gate_accepts": (_i, [C.POINTER(RelocGate)]),
    "df_kinfu_get_keyframes": (_i, [_vp, _vp, _vp, _i, C.POINTER(_i)]),
}

# include/dfusion.h DF_COLOR_TRACK_WEIGHT / DF_COLOR_TRACK_MAX_RESIDUAL: the frame loop's photometric weight and residual gate
COLOR_TRACK_WEIGHT = 0.1
COLOR_TRACK_MAX_RESIDUAL = 0.2


def lib_path() -> Path:
    return _LIB_PATH


def load() -> C.CDLL:
    """Load libdfusion.so; raise (never fall back) when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise RuntimeError(
            f"{_LIB_PATH} is missing: build it with `python -m dynamicfusion_b200.build` "
            "(nvcc, sm_90a).  dynamicfusion_b200 has no CPU fallback.")
    lib = C.CDLL(str(_LIB_PATH))
    MISSING.clear()
    for name, (res, args) in PROTOTYPES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:       # header/library mismatch: calling it raises, tests/test_capi.py asserts none
            MISSING.append(name)
            continue
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status: int) -> None:
    if status != 0:
        raise RuntimeError(f"libdfusion: CUDA error {status}: {load().df_error_string(status).decode()}")


def make_aff(R, t) -> Aff3f:
    a = Aff3f()
    flat = [float(v) for row in R for v in row] if hasattr(R[0], "__len__") else [float(v) for v in R]
    for i in range(9):
        a.R[i] = flat[i]
    for i in range(3):
        a.t[i] = float(t[i])
    return a


def make_intr(fx, fy, cx, cy) -> Intr:
    return Intr(float(fx), float(fy), float(cx), float(cy))


def make_color_camera(K, cols: int, rows: int, depth_to_color=None) -> ColorCamera:
    """df_color_camera from intrinsics (fx, fy, cx, cy), the image size and depth_to_color (R, t); None = the identity"""
    if depth_to_color is None:
        depth_to_color = ((1, 0, 0, 0, 1, 0, 0, 0, 1), (0, 0, 0))
    return ColorCamera(int(cols), int(rows), make_intr(*K), make_aff(*depth_to_color))


def default_r2_max(K, cols: int, rows: int) -> float:
    """(1.1 * rho)^2, rho the normalised radius of the image corner farthest from the principal point: a calibration's domain with a margin
    of 10 % for the rays the lens bends outwards"""
    fx, fy, cx, cy = (float(k) for k in K)
    rho2 = max(((u - cx) / fx) ** 2 + ((v - cy) / fy) ** 2 for u in (0.0, float(cols)) for v in (0.0, float(rows)))
    return 1.21 * rho2


def make_lens(coeffs, r2_max=None, K=None, cols: int = 0, rows: int = 0) -> Lens:
    """df_lens from 5 (k1, k2, p1, p2, k3: Brown-Conrady) or 8 (and k4, k5, k6: the rational model) coefficients in OpenCV's order.
    r2_max None: default_r2_max of the camera with intrinsics K (fx, fy, cx, cy) and cols x rows pixels, which must then be given."""
    c = [float(v) for v in coeffs]
    if len(c) not in (5, 8):
        raise ValueError(f"a lens has 5 or 8 coefficients, not {len(c)}")
    c += [0.0] * (8 - len(c))
    if r2_max is None:
        if K is None or cols <= 0 or rows <= 0:
            raise ValueError("make_lens: r2_max None needs the camera's K, cols and rows")
        r2_max = default_r2_max(K, cols, rows)
    return Lens(*c, float(r2_max))


def make_volume(ptr: int, dims, voxel_size, trunc_dist: float, max_weight: int) -> Volume:
    v = Volume()
    v.data = ptr
    for i in range(3):
        v.dims[i] = int(dims[i])
        v.voxel_size[i] = float(voxel_size[i])
    v.trunc_dist = float(trunc_dist)
    v.max_weight = int(max_weight)
    return v


def f9(vals):
    arr = (C.c_float * 9)()
    flat = [float(v) for row in vals for v in row] if hasattr(vals[0], "__len__") else [float(v) for v in vals]
    for i in range(9):
        arr[i] = flat[i]
    return arr
