"""ctypes binding of the colour-tracking oracle (tests/color_track_oracle.c), test infrastructure only."""
from __future__ import annotations

import ctypes as C

import numpy as np

import c_oracle
import color_oracle as co

OCCLUSION = 1.0                                             # DF_COLOR_OCCLUSION


def load() -> C.CDLL:
    vp, i, f, sz = C.c_void_p, C.c_int, C.c_float, C.c_size_t
    return c_oracle.load("color_track_oracle", {
        "ct_intensity_registered": (None, [vp, sz, i, i, vp]),
        "ct_intensity_camera": (None, [vp, sz, i, i, vp, vp, i, vp, sz, f, f, vp, i, i, vp]),
        "ct_intensity_down": (None, [vp, i, vp, i, i]),
        "ct_model_intensity": (None, [vp, vp, vp, vp, vp, i, i, vp, vp]),
        "ct_photo_rows": (C.c_long, [vp, vp, vp, vp, i, i, vp, vp, f, f, vp]),
    })


def luma(r, g, b):
    """the intensity rule on integer R, G, B arrays"""
    Y = (77 * np.asarray(r, np.int64) + 150 * np.asarray(g, np.int64) + 29 * np.asarray(b, np.int64) + 128) >> 8
    return (Y.astype(np.float32) / np.float32(255.0)).astype(np.float32)


def level_sizes(cols, rows, levels):
    """the depth pyramid's level sizes [(cols, rows)]: each half the one before, rounded down"""
    out = [(cols, rows)]
    for _ in range(levels - 1):
        out.append((out[-1][0] // 2, out[-1][1] // 2))
    return out


def intensity_down(src):
    """one pyramid level down: float [rows, cols] -> [rows // 2, cols // 2]"""
    src = np.ascontiguousarray(src, np.float32)
    rows, cols = src.shape[0] // 2, src.shape[1] // 2
    out = np.empty((rows, cols), np.float32)
    load().ct_intensity_down(src.ctypes.data, src.shape[1], out.ctypes.data, cols, rows)
    return out


def frame_intensity(bgra, levels, camera=None, K_depth=None, points=None, color_map=None, trunc_dist=0.0):
    """df_frame_intensity's rule: [float [rows_l, cols_l]] for levels 0..levels-1.  Registered (camera None): bgra is the depth frame's size.
    Through a colour camera: camera = color_camera_oracle.Camera, K_depth the depth intrinsics, points = the level-0 vertex map
    [rows, cols, 4], color_map = the occlusion map (uint32 [map_rows, map_cols]) of the same frame."""
    if camera is None:
        rows, cols = bgra.shape[:2]
        out = np.empty((rows, cols), np.float32)
        load().ct_intensity_registered(bgra.ctypes.data, bgra.strides[0], cols, rows, out.ctypes.data)
    else:
        P = np.ascontiguousarray(points, np.float32)
        rows, cols = P.shape[:2]
        m = np.ascontiguousarray(color_map, np.uint32)
        import color_camera_oracle as cco
        cam4 = camera.k4()
        d2c = co.a12(camera.d2c)
        out = np.empty((rows, cols), np.float32)
        load().ct_intensity_camera(bgra.ctypes.data, bgra.strides[0], camera.cols, camera.rows, cam4.ctypes.data, d2c.ctypes.data,
                                   cco.cell(K_depth, camera),
                                   m.ctypes.data, m.strides[0], OCCLUSION, float(trunc_dist), P.ctypes.data, cols, rows, out.ctypes.data)
    pyr = [out]
    for _ in range(levels - 1):
        pyr.append(intensity_down(pyr[-1]))
    return pyr


def model_intensity(colors, dims, voxel_size, cam2vol, points):
    """df_model_intensity's rule for one level: float [rows, cols, 4] (I, gu, gv, 0) or four NaNs; cam2vol (R, t) applied as written"""
    P = np.ascontiguousarray(points, np.float32)
    rows, cols = P.shape[:2]
    d = np.asarray(dims, np.int32)
    vs = np.asarray(voxel_size, np.float32)
    col = np.ascontiguousarray(colors, np.uint32)
    out = np.empty((rows, cols, 4), np.float32)
    scratch = np.empty(rows * cols, np.float32)
    load().ct_model_intensity(d.ctypes.data, vs.ctypes.data, col.ctypes.data, co.a12(cam2vol).ctypes.data, P.ctypes.data, cols, rows,
                              out.ctypes.data, scratch.ctypes.data)
    return out


def photo_rows(vcurr, icurr, model, match, K_level, T, weight, max_residual):
    """the photometric rows of one level: (rows [rows, cols, 7] float32, NaN where there is none; count)"""
    V = np.ascontiguousarray(vcurr, np.float32)
    I = np.ascontiguousarray(icurr, np.float32)
    M = np.ascontiguousarray(model, np.float32)
    m = np.ascontiguousarray(match, np.int32)
    rows, cols = V.shape[:2]
    out = np.empty((rows, cols, 7), np.float32)
    K = np.asarray(K_level, np.float32)
    n = load().ct_photo_rows(V.ctypes.data, I.ctypes.data, M.ctypes.data, m.ctypes.data, cols, rows, K.ctypes.data, co.a12(T).ctypes.data,
                             float(weight), float(max_residual), out.ctypes.data)
    return out, int(n)
