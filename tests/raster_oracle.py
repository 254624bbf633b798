"""ctypes binding of the rasteriser oracle (tests/raster_oracle.c), test infrastructure only."""
from __future__ import annotations

import ctypes as C

import numpy as np

import c_oracle
import color_oracle as co


def load() -> C.CDLL:
    args = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    return c_oracle.load("raster_oracle", {
        "ro_raster": (C.c_int, args + [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
        "ro_coverage": (C.c_int, args + [C.c_void_p]),
    })


def _inputs(verts, tris, world2cam, K):
    v = np.ascontiguousarray(verts, np.float32)
    assert v.ndim == 2 and v.shape[1] in (3, 4)
    t = np.ascontiguousarray(np.asarray(tris, np.int32).reshape(-1, 3))
    k = np.asarray(K, np.float32).reshape(4)
    return v, t, co.a12(world2cam), k


def raster(verts, tris, world2cam, K, cols, rows):
    """(tri_ids [rows, cols] int32, points [rows, cols, 4] float32, normals [rows, cols, 4] float32, stats [5] uint64) of df_raster_mesh.
    verts: [N, 3|4] float32; tris: [T, 3] int32; world2cam: (R 3x3, t 3); K: (fx, fy, cx, cy)"""
    v, t, w, k = _inputs(verts, tris, world2cam, K)
    ids = np.empty((rows, cols), np.int32)
    pts = np.empty((rows, cols, 4), np.float32)
    nrm = np.empty((rows, cols, 4), np.float32)
    stats = np.zeros(5, np.uint64)
    r = load().ro_raster(v.ctypes.data, len(v), v.shape[1], t.ctypes.data, len(t), w.ctypes.data, k.ctypes.data, cols, rows, ids.ctypes.data,
                         pts.ctypes.data, nrm.ctypes.data, stats.ctypes.data)
    assert r == 0
    return ids, pts, nrm, stats


def coverage(verts, tris, world2cam, K, cols, rows):
    """[rows, cols] int32: how many drawn triangles cover each pixel's sample, without the depth test"""
    v, t, w, k = _inputs(verts, tris, world2cam, K)
    out = np.empty((rows, cols), np.int32)
    assert load().ro_coverage(v.ctypes.data, len(v), v.shape[1], t.ctypes.data, len(t), w.ctypes.data, k.ctypes.data, cols, rows,
                              out.ctypes.data) == 0
    return out
