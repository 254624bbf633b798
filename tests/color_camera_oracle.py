"""ctypes binding of the colour-camera oracle (tests/color_camera_oracle.c), test infrastructure only."""
from __future__ import annotations

import ctypes as C

import numpy as np

import c_oracle
import color_oracle as co

EMPTY = 0xFFFFFFFF


def load() -> C.CDLL:
    vp, i, f, sz = C.c_void_p, C.c_int, C.c_float, C.c_size_t
    return c_oracle.load("color_camera_oracle", {
        "cc_cell": (i, [vp, vp]),
        "cc_depth_map": (None, [vp, sz, i, i, vp, i, i, vp, vp, vp, sz]),
        "cc_integrate_color_camera": (None, [vp, vp, f, i, vp, vp, sz, i, i, vp, vp, i, i, vp, vp, vp, sz, vp, sz, vp]),
    })


class Camera:
    """a colour camera: size, intrinsics (fx, fy, cx, cy) and depth_to_color (R, t) -- df_color_camera's fields"""

    def __init__(self, cols, rows, K, depth_to_color=None):
        self.cols, self.rows = int(cols), int(rows)
        self.K = tuple(float(k) for k in K)
        self.d2c = depth_to_color if depth_to_color is not None else (np.eye(3, dtype=np.float32), np.zeros(3, np.float32))

    def k4(self):
        return np.asarray(self.K, np.float32)


def cell(K_depth, cam: Camera) -> int:
    k, kc = np.asarray(K_depth, np.float32), cam.k4()
    return int(load().cc_cell(k.ctypes.data, kc.ctypes.data))


def map_dims(K_depth, cam: Camera):
    """(map cols, map rows, cell) as df_color_map_dims computes them"""
    c = cell(K_depth, cam)
    return -(-cam.cols // c), -(-cam.rows // c), c


def depth_map(depth, K_depth, cam: Camera):
    """df_color_depth_map's rule: uint32 [map rows, map cols] for a u16 depth image (may be a strided view with padded rows)"""
    assert depth.dtype == np.uint16 and depth.strides[1] == 2
    rows, cols = depth.shape
    mc, mr, _ = map_dims(K_depth, cam)
    out = np.empty((mr, mc), np.uint32)
    k, kc, d2c = np.asarray(K_depth, np.float32), cam.k4(), co.a12(cam.d2c)
    load().cc_depth_map(depth.ctypes.data, depth.strides[0], cols, rows, k.ctypes.data, cam.cols, cam.rows, kc.ctypes.data, d2c.ctypes.data,
                        out.ctypes.data, out.strides[0])
    return out


def integrate_color_camera(colors, dims, voxel_size, trunc_dist, max_weight, dists, vol2cam, K_depth, cam: Camera, bgra, cmap, activity=None):
    """df_integrate_color_camera's rule on the host: colors (uint32 [Dx*Dy*Dz]) is updated IN PLACE and returned.  dists: uint16 [rows, cols]
    fp16 bit patterns of the depth frame; bgra: uint8 [cam.rows, cam.cols, 4]; cmap: uint32 [map rows, map cols] (each may be a strided
    view with padded rows)"""
    assert colors.dtype == np.uint32 and colors.flags.c_contiguous and colors.size == int(np.prod(dims))
    assert dists.dtype == np.uint16 and dists.strides[1] == 2 and bgra.dtype == np.uint8 and bgra.strides[1:] == (4, 1)
    assert bgra.shape == (cam.rows, cam.cols, 4) and cmap.dtype == np.uint32 and cmap.strides[1] == 4
    rows, cols = dists.shape
    d = np.asarray(dims, np.int32)
    vs = np.asarray(voxel_size, np.float32)
    k, kc, w, d2c = np.asarray(K_depth, np.float32), cam.k4(), co.a12(vol2cam), co.a12(cam.d2c)
    act = None if activity is None else np.ascontiguousarray(activity, np.uint8)
    load().cc_integrate_color_camera(d.ctypes.data, vs.ctypes.data, float(trunc_dist), int(max_weight), colors.ctypes.data, dists.ctypes.data,
                                     dists.strides[0], cols, rows, w.ctypes.data, k.ctypes.data, cam.cols, cam.rows, kc.ctypes.data,
                                     d2c.ctypes.data, bgra.ctypes.data, bgra.strides[0], cmap.ctypes.data,
                                     cmap.strides[0], None if act is None else act.ctypes.data)
    return colors
