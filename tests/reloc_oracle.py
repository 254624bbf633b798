"""ctypes binding of the relocaliser's oracle (tests/reloc_oracle.c), test infrastructure only.  The constants come from capi, which
tests/test_reloc.py pins to include/dfusion.h."""
from __future__ import annotations

import ctypes as C

import numpy as np

import c_oracle
from dynamicfusion_b200 import capi


def load() -> C.CDLL:
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    return c_oracle.load("reloc_oracle", {
        "rc_fern_table": (None, [C.c_uint64, i, i, i, i, i, vp]),
        "rc_encode": (None, [vp, i, i, i, vp, i, vp]),
        "rc_dissimilarity": (i, [vp, vp, i]),
        "rc_match": (i, [vp, vp, i, vp, i, i, i, i, vp, vp]),
        "rc_gate": (None, [vp, vp, vp, vp, i, i, f, f, f, f, vp, f, f, vp, vp]),
        "rc_accepts": (i, [i, i, i, C.c_double, i, f, f]),
    })


def fern_table(seed: int, cols: int, rows: int, n_ferns: int = capi.RELOC_FERNS) -> np.ndarray:
    """int32 [n_ferns, 4, 3] (u, v, theta_mm)"""
    out = np.empty((n_ferns, 4, 3), np.int32)
    load().rc_fern_table(seed, cols, rows, n_ferns, capi.RELOC_NEAR_MM, capi.RELOC_FAR_MM, out.ctypes.data)
    return out


def encode(depth: np.ndarray, table: np.ndarray) -> np.ndarray:
    """the Code rule on a host u16 [rows, cols] image (any row stride)"""
    assert depth.dtype == np.uint16 and depth.strides[1] == 2
    t = np.ascontiguousarray(table, np.int32)
    codes = np.empty(len(t), np.uint8)
    load().rc_encode(depth.ctypes.data, depth.strides[0] // 2, depth.shape[1], depth.shape[0], t.ctypes.data, len(t), codes.ctypes.data)
    return codes


def match(db: np.ndarray, count: int, code: np.ndarray, append: bool, capacity: int = capi.RELOC_KEYFRAMES):
    """the lookup and the harvest on a database db [capacity, F] uint8 holding `count` entries (updated in place on an append):
    (index [K], dissimilarity [K], appended, count after)"""
    assert db.dtype == np.uint8 and db.flags.c_contiguous and db.shape[0] >= capacity
    code = np.ascontiguousarray(code, np.uint8)
    n = C.c_int(count)
    idx = np.empty(capi.RELOC_CANDIDATES, np.int32)
    dis = np.empty(capi.RELOC_CANDIDATES, np.int32)
    add = load().rc_match(db.ctypes.data, C.byref(n), capacity, code.ctypes.data, len(code), capi.RELOC_CANDIDATES, capi.RELOC_HARVEST_FERNS,
                          int(append), idx.ctypes.data, dis.ctypes.data)
    return idx, dis, bool(add), n.value


def gate(vc, nc, vp, np_, K, T12, dist_thres: float, angle_thres: float):
    """the gate's counts in double on dense float32 [rows, cols, 4] maps: (n_valid, n_in, n_ambiguous, sum_sq)"""
    maps = [np.ascontiguousarray(a, np.float32) for a in (vc, nc, vp, np_)]
    T = np.ascontiguousarray(T12, np.float32).reshape(12)
    counts = np.zeros(3, np.int32)
    s = C.c_double()
    rows, cols = maps[0].shape[:2]
    load().rc_gate(*[a.ctypes.data for a in maps], cols, rows, *[float(k) for k in K], T.ctypes.data, dist_thres, angle_thres,
                   counts.ctypes.data, C.byref(s))
    return int(counts[0]), int(counts[1]), int(counts[2]), s.value


def accepts(ok: int, n_valid: int, n_in: int, sum_sq: float) -> bool:
    return bool(load().rc_accepts(ok, n_valid, n_in, sum_sq, capi.RELOC_MIN_VALID, capi.RELOC_MIN_INLIER_FRAC, capi.RELOC_MAX_RMS))
