"""ctypes binding of the correspondence oracle (tests/correspond_oracle.c), test infrastructure only."""
from __future__ import annotations

import ctypes as C

import numpy as np

import c_oracle
import color_oracle as co


def load() -> C.CDLL:
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    return c_oracle.load("correspond_oracle", {
        "co_correspond": (None, [vp, vp, vp, vp, i, i, vp, i, vp, i, i, vp, f, vp, vp]),
        "co_weights": (None, [vp, vp, vp, i, vp, vp, i, vp]),
    })


def correspond(tri_ids, points, verts, src, tris, world2cam, target=None, max_dist=0.0):
    """(source points [rows, cols, 4], source normals [rows, cols, 4]) of df_mesh_correspond; tri_ids / points: a raster_oracle.raster (or
    df_raster_mesh) result for verts / tris / world2cam (R, t); src: the source vertex set, same shape as verts"""
    ids = np.ascontiguousarray(tri_ids, np.int32)
    rows, cols = ids.shape
    P = np.ascontiguousarray(points, np.float32)
    v = np.ascontiguousarray(verts, np.float32)
    s = np.ascontiguousarray(src, np.float32)
    assert v.shape == s.shape and v.shape[1] in (3, 4)
    t = np.ascontiguousarray(np.asarray(tris, np.int32).reshape(-1, 3))
    w = co.a12(world2cam)
    T = None if target is None else np.ascontiguousarray(target, np.float32)
    out_p = np.empty((rows, cols, 4), np.float32)
    out_n = np.empty((rows, cols, 4), np.float32)
    load().co_correspond(ids.ctypes.data, P.ctypes.data, v.ctypes.data, s.ctypes.data, len(v), v.shape[1], t.ctypes.data, len(t), w.ctypes.data,
                         cols, rows, None if T is None else T.ctypes.data, float(max_dist), out_p.ctypes.data, out_n.ctypes.data)
    return out_p, out_n


def weights(tri_ids, points, verts, tris, world2cam):
    """[rows, cols, 3] float32 barycentric weights (b0, b1, b2) of the rule, NaN where there is none"""
    ids = np.ascontiguousarray(tri_ids, np.int32)
    P = np.ascontiguousarray(points, np.float32)
    v = np.ascontiguousarray(verts, np.float32)
    t = np.ascontiguousarray(np.asarray(tris, np.int32).reshape(-1, 3))
    w = co.a12(world2cam)
    out = np.empty(ids.shape + (3,), np.float32)
    load().co_weights(ids.ctypes.data, P.ctypes.data, v.ctypes.data, v.shape[1], t.ctypes.data, w.ctypes.data, ids.size, out.ctypes.data)
    return out
