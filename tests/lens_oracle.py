"""ctypes binding of the lens oracle (tests/lens_oracle.c), test infrastructure only."""
from __future__ import annotations

import ctypes as C

import numpy as np

import c_oracle
import color_oracle as co
import color_camera_oracle as cco


def load() -> C.CDLL:
    vp, i, f, sz = C.c_void_p, C.c_int, C.c_float, C.c_size_t
    return c_oracle.load("lens_oracle", {
        "lens_distort": (i, [vp, f, f, C.POINTER(f), C.POINTER(f)]),
        "lens_undistort": (None, [vp, sz, vp, sz, vp, sz, vp, sz, i, i, vp, vp]),
        "lens_depth_map": (None, [vp, sz, i, i, vp, i, i, vp, vp, vp, vp, sz]),
        "lens_integrate_color_camera": (None, [vp, vp, f, i, vp, vp, sz, i, i, vp, vp, i, i, vp, vp, vp, vp, sz, vp, sz, vp]),
        "lens_frame_intensity": (None, [vp, sz, i, i, vp, vp, vp, vp, vp, sz, f, vp, i, i, vp]),
    })


def lens9(lens):
    """float32 [9] (k1, k2, p1, p2, k3, k4, k5, k6, r2_max) of a capi.Lens or of 9 numbers; None stays None"""
    if lens is None:
        return None
    if hasattr(lens, "coeffs"):
        return np.array(list(lens.coeffs()) + [lens.r2_max], np.float32)
    a = np.asarray(lens, np.float32)
    assert a.shape == (9,)
    return a


def _ptr(a):
    return None if a is None else a.ctypes.data


def distort(x, y, lens):
    """the rule's forward distortion of float32 points: (xd, yd, valid) arrays"""
    L = lens9(lens)
    x, y = np.asarray(x, np.float32).ravel(), np.asarray(y, np.float32).ravel()
    xd, yd, ok = np.empty_like(x), np.empty_like(y), np.zeros(x.shape, bool)
    a, b = C.c_float(), C.c_float()
    lib = load()
    for n in range(x.size):
        ok[n] = bool(lib.lens_distort(L.ctypes.data, float(x[n]), float(y[n]), C.byref(a), C.byref(b)))
        xd[n], yd[n] = a.value, b.value
    return xd, yd, ok


def undistort(depth, K, lens, bgra=None):
    """df_undistort's rule: (depth_out uint16 [rows, cols], bgra_out uint8 [rows, cols, 4] or None); inputs may be strided views"""
    assert depth.dtype == np.uint16 and depth.strides[1] == 2
    rows, cols = depth.shape
    out = np.empty((rows, cols), np.uint16)
    bout = None
    if bgra is not None:
        assert bgra.dtype == np.uint8 and bgra.strides[1:] == (4, 1) and bgra.shape == (rows, cols, 4)
        bout = np.empty((rows, cols, 4), np.uint8)
    k, L = np.asarray(K, np.float32), lens9(lens)
    load().lens_undistort(depth.ctypes.data, depth.strides[0], out.ctypes.data, out.strides[0], _ptr(bgra), 0 if bgra is None else bgra.strides[0],
                          _ptr(bout), 0 if bout is None else bout.strides[0], cols, rows, k.ctypes.data, L.ctypes.data)
    return out, bout


def depth_map(depth, K_depth, cam: cco.Camera, lens):
    """df_color_depth_map_lens' rule: uint32 [map rows, map cols]"""
    assert depth.dtype == np.uint16 and depth.strides[1] == 2
    rows, cols = depth.shape
    mc, mr, _ = cco.map_dims(K_depth, cam)
    out = np.empty((mr, mc), np.uint32)
    k, kc, d2c, L = np.asarray(K_depth, np.float32), cam.k4(), co.a12(cam.d2c), lens9(lens)
    load().lens_depth_map(depth.ctypes.data, depth.strides[0], cols, rows, k.ctypes.data, cam.cols, cam.rows, kc.ctypes.data, d2c.ctypes.data,
                          _ptr(L), out.ctypes.data, out.strides[0])
    return out


def integrate_color_camera(colors, dims, voxel_size, trunc_dist, max_weight, dists, vol2cam, K_depth, cam: cco.Camera, lens, bgra, cmap,
                           activity=None):
    """df_integrate_color_camera_lens' rule: colors (uint32 [Dx*Dy*Dz]) updated IN PLACE and returned"""
    assert colors.dtype == np.uint32 and colors.flags.c_contiguous and colors.size == int(np.prod(dims))
    assert dists.dtype == np.uint16 and dists.strides[1] == 2 and bgra.dtype == np.uint8 and bgra.strides[1:] == (4, 1)
    assert bgra.shape == (cam.rows, cam.cols, 4) and cmap.dtype == np.uint32 and cmap.strides[1] == 4
    rows, cols = dists.shape
    d, vs = np.asarray(dims, np.int32), np.asarray(voxel_size, np.float32)
    k, kc, w, d2c, L = np.asarray(K_depth, np.float32), cam.k4(), co.a12(vol2cam), co.a12(cam.d2c), lens9(lens)
    act = None if activity is None else np.ascontiguousarray(activity, np.uint8)
    load().lens_integrate_color_camera(d.ctypes.data, vs.ctypes.data, float(trunc_dist), int(max_weight), colors.ctypes.data, dists.ctypes.data,
                                       dists.strides[0], cols, rows, w.ctypes.data, k.ctypes.data, cam.cols, cam.rows, kc.ctypes.data,
                                       d2c.ctypes.data, _ptr(L), bgra.ctypes.data, bgra.strides[0], cmap.ctypes.data, cmap.strides[0], _ptr(act))
    return colors


def frame_intensity(bgra, K_depth, cam: cco.Camera, lens, cmap, trunc_dist, points):
    """level 0 of df_frame_intensity_lens through the colour camera: float32 [rows, cols] (NaN = no value); points float32 [rows, cols, 4]"""
    pts = np.ascontiguousarray(points, np.float32)
    rows, cols = pts.shape[:2]
    out = np.empty((rows, cols), np.float32)
    k, kc, d2c, L = np.asarray(K_depth, np.float32), cam.k4(), co.a12(cam.d2c), lens9(lens)
    load().lens_frame_intensity(bgra.ctypes.data, bgra.strides[0], cam.cols, cam.rows, kc.ctypes.data, d2c.ctypes.data, _ptr(L), k.ctypes.data,
                                cmap.ctypes.data, cmap.strides[0], float(trunc_dist), pts.ctypes.data, cols, rows, out.ctypes.data)
    return out
