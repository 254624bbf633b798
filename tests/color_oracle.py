"""ctypes binding of the colour oracle (tests/color_oracle.c), test infrastructure only."""
from __future__ import annotations

import ctypes as C

import numpy as np

import c_oracle


def load() -> C.CDLL:
    vp, i, f, sz = C.c_void_p, C.c_int, C.c_float, C.c_size_t
    return c_oracle.load("color_oracle", {
        "cl_integrate_color": (None, [vp, vp, f, i, vp, vp, sz, vp, sz, i, i, vp, vp, vp]),
        "cl_sample_colors": (None, [vp, vp, vp, vp, f, vp, i, sz, vp]),
        "cl_mesh_colors": (None, [vp, vp, vp, i, i, vp, i, vp, vp, sz, vp, vp]),
        "cl_aff_mul": (None, [vp, vp, vp]),
        "cl_aff_inv": (None, [vp, vp]),
    })


def a12(aff):
    """(R 3x3, t 3) -> 12 float32, R row-major then t"""
    return np.concatenate([np.asarray(aff[0], np.float32).reshape(9), np.asarray(aff[1], np.float32).reshape(3)]).astype(np.float32)


def unpack(a):
    return a[:9].reshape(3, 3).copy(), a[9:].copy()


def aff_mul(A, B):
    """A * B as df_hostmath.h dfh_aff_mul computes it"""
    a, b, out = a12(A), a12(B), np.empty(12, np.float32)
    load().cl_aff_mul(a.ctypes.data, b.ctypes.data, out.ctypes.data)
    return unpack(out)


def aff_inv(A):
    """A^-1 as df_hostmath.h dfh_aff_inv computes it"""
    a, out = a12(A), np.empty(12, np.float32)
    load().cl_aff_inv(a.ctypes.data, out.ctypes.data)
    return unpack(out)


def integrate_color(colors, dims, voxel_size, trunc_dist, max_weight, dists, bgra, vol2cam, intr, activity=None):
    """df_integrate_color's rule on the host: colors (uint32 [Dx*Dy*Dz]) is updated IN PLACE and returned.  dists: uint16 [rows, cols] fp16
    bit patterns, bgra: uint8 [rows, cols, 4] (either may be a strided view with padded rows); vol2cam: (R, t); intr: (fx, fy, cx, cy)"""
    assert colors.dtype == np.uint32 and colors.flags.c_contiguous and colors.size == int(np.prod(dims))
    assert dists.dtype == np.uint16 and dists.strides[1] == 2 and bgra.dtype == np.uint8 and bgra.strides[1:] == (4, 1)
    rows, cols = dists.shape
    assert bgra.shape == (rows, cols, 4)
    d = np.asarray(dims, np.int32)
    vs = np.asarray(voxel_size, np.float32)
    k = np.asarray(intr, np.float32)
    w = a12(vol2cam)
    act = None if activity is None else np.ascontiguousarray(activity, np.uint8)
    load().cl_integrate_color(d.ctypes.data, vs.ctypes.data, float(trunc_dist), int(max_weight), colors.ctypes.data, dists.ctypes.data,
                              dists.strides[0], bgra.ctypes.data, bgra.strides[0], cols, rows, w.ctypes.data, k.ctypes.data,
                              None if act is None else act.ctypes.data)
    return colors


def sample_colors(colors, dims, voxel_size, vol_pose, offset, points):
    """df_sample_colors' rule: uint8 [..., 4] R, G, B, A for points [..., 3 or 4]"""
    P = np.ascontiguousarray(points, np.float32)
    flat = P.reshape(-1, P.shape[-1])
    d = np.asarray(dims, np.int32)
    vs = np.asarray(voxel_size, np.float32)
    out = np.empty(len(flat), np.uint32)
    col = np.ascontiguousarray(colors, np.uint32)
    load().cl_sample_colors(d.ctypes.data, vs.ctypes.data, col.ctypes.data, a12(vol_pose).ctypes.data, float(offset), flat.ctypes.data,
                            flat.shape[1], len(flat), out.ctypes.data)
    return out.view(np.uint8).reshape(P.shape[:-1] + (4,))


def mesh_colors(tri_ids, points, verts, tris, world2cam, vert_rgba, want_weights=False):
    """df_mesh_colors' rule: BGRA uint8 [rows, cols, 4] (and the weights [rows, cols, 3]) for a raster result tri_ids / points of
    verts / tris / world2cam (R, t); vert_rgba: uint8 [N, 4] or uint32 [N]"""
    ids = np.ascontiguousarray(tri_ids, np.int32)
    P = np.ascontiguousarray(points, np.float32)
    v = np.ascontiguousarray(verts, np.float32)
    t = np.ascontiguousarray(np.asarray(tris, np.int32).reshape(-1, 3))
    c = np.ascontiguousarray(vert_rgba).view(np.uint32).reshape(-1)
    assert len(c) == len(v)
    img = np.empty(ids.shape + (4,), np.uint8)
    wts = np.empty(ids.shape + (3,), np.float32) if want_weights else None
    load().cl_mesh_colors(ids.ctypes.data, P.ctypes.data, v.ctypes.data, len(v), v.shape[1], t.ctypes.data, len(t), a12(world2cam).ctypes.data,
                          c.ctypes.data, ids.size, img.ctypes.data, None if wts is None else wts.ctypes.data)
    return (img, wts) if want_weights else img
