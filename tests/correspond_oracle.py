"""ctypes binding of the correspondence oracle (tests/correspond_oracle.c), test infrastructure only.  The C file is compiled on first use
into a fresh temporary directory, so a read-only checkout works too."""
from __future__ import annotations

import ctypes as C
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
SRC = HERE / "correspond_oracle.c"
_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        cc = "/usr/bin/gcc" if Path("/usr/bin/gcc").exists() else (shutil.which("gcc") or "cc")
        out = Path(tempfile.mkdtemp(prefix="correspond_oracle_")) / "libcorrespond_oracle.so"
        subprocess.run([cc, "-std=gnu11", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-shared",
                        "-I", str(HERE.parent / "include"), "-o", str(out), str(SRC), "-lm"], check=True, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT)
        lib = C.CDLL(str(out))
        vp, i, f = C.c_void_p, C.c_int, C.c_float
        lib.co_correspond.restype = None
        lib.co_correspond.argtypes = [vp, vp, vp, vp, i, i, vp, i, vp, i, i, vp, f, vp, vp]
        lib.co_weights.restype = None
        lib.co_weights.argtypes = [vp, vp, vp, i, vp, vp, i, vp]
        lib.co_aff_mul.restype = None
        lib.co_aff_mul.argtypes = [vp, vp, vp]
        lib.co_aff_inv.restype = None
        lib.co_aff_inv.argtypes = [vp, vp]
        _lib = lib
    return _lib


def a12(aff):
    """(R 3x3, t 3) -> 12 float32, R row-major then t"""
    return np.concatenate([np.asarray(aff[0], np.float32).reshape(9), np.asarray(aff[1], np.float32).reshape(3)]).astype(np.float32)


def unpack(a):
    return a[:9].reshape(3, 3).copy(), a[9:].copy()


def aff_mul(A, B):
    """A * B as df_hostmath.h dfh_aff_mul computes it"""
    a, b, out = a12(A), a12(B), np.empty(12, np.float32)
    load().co_aff_mul(a.ctypes.data, b.ctypes.data, out.ctypes.data)
    return unpack(out)


def aff_inv(A):
    """A^-1 as df_hostmath.h dfh_aff_inv computes it"""
    a, out = a12(A), np.empty(12, np.float32)
    load().co_aff_inv(a.ctypes.data, out.ctypes.data)
    return unpack(out)


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
    w = a12(world2cam)
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
    w = a12(world2cam)
    out = np.empty(ids.shape + (3,), np.float32)
    load().co_weights(ids.ctypes.data, P.ctypes.data, v.ctypes.data, v.shape[1], t.ctypes.data, w.ctypes.data, ids.size, out.ctypes.data)
    return out
