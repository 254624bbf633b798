"""ctypes/numpy binding of the CPU oracle (oracle/liborc.so).  TEST INFRASTRUCTURE ONLY:
importable from tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg, never from
dynamicfusion_b200/ (tests/test_no_oracle_in_product.py enforces it)."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
LIB = HERE / "liborc.so"
_lib = None


class Volume(C.Structure):
    _fields_ = [("data", C.c_void_p), ("dims", C.c_int * 3), ("voxel_size", C.c_float * 3),
                ("trunc_dist", C.c_float), ("max_weight", C.c_int)]


class Aff3f(C.Structure):
    _fields_ = [("R", C.c_float * 9), ("t", C.c_float * 3)]


class Intr(C.Structure):
    _fields_ = [("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float)]


def build(force: bool = False) -> Path:
    srcs = list(HERE.glob("orc_*.c")) + [HERE / "orc_common.h", HERE / "Makefile"]
    if force or not LIB.exists() or any(s.stat().st_mtime > LIB.stat().st_mtime for s in srcs):
        subprocess.run(["make", "-C", str(HERE), "-B", "liborc.so"], check=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    return LIB


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not LIB.exists():
            build()
        _lib = C.CDLL(str(LIB))
        _lib.orc_integrate.restype = C.c_longlong
        _lib.orc_extract_cloud.restype = C.c_longlong
        _lib.orc_integrate_warped.restype = C.c_longlong
        _lib.orc_icp_accumulate.restype = C.c_longlong
        _lib.orc_icp_accumulate_depth.restype = C.c_longlong
        _lib.orc_icp_rows.restype = C.c_longlong
        _lib.orc_icp_rows_depth.restype = C.c_longlong
        _lib.orc_float2half_rn.restype = C.c_uint16
        _lib.orc_float2half_rn.argtypes = [C.c_float]
        _lib.orc_half2float.restype = C.c_float
        _lib.orc_half2float.argtypes = [C.c_uint16]
        _lib.orc_interpolate.restype = C.c_float
    return _lib


# ------------------------------------------------------------------ reference arm --------------------------------------------------
# oracle/_ref/libkfref.so = the REFERENCE's own kfusion/src/cuda/*.cu kernels compiled for the host (oracle/ref_shim/cudahost),
# exported with the orc_* signatures under the kfref_ prefix.  `with orc.reference(): orc.integrate(...)` runs the reference's
# code instead of the restatement, on the same numpy buffers -- used by tests/ and golden/make_golden.py to pin the oracle.
REF_LIB = HERE / "_ref" / "libkfref.so"
_ref_lib = None
_use_ref = False


def reference_available() -> bool:
    return REF_LIB.exists() and REF_LOCKSTEP_LIB.exists()


def load_ref() -> C.CDLL:
    global _ref_lib
    if _ref_lib is None:
        _ref_lib = C.CDLL(str(REF_LIB))
        _ref_lib.kfref_integrate.restype = C.c_longlong
        _ref_lib.kfref_icp_accumulate.restype = C.c_longlong
    return _ref_lib


# libkfref_usedepth.so = proj_icp.cu compiled with the reference's compile-time USE_DEPTH alternative (internal.hpp:6); it defines the
# same C++ symbols as libkfref.so, hence a library of its own (both are loaded RTLD_LOCAL)
# libkfref_lockstep.so = tsdf_volume.cu once more, under the warp-lock-step executor (oracle/ref_shim/cudahost/lockstep.h): the reference's
# warp-synchronous extract_kernel (tsdf_volume.cu:511-710) really runs, 32 lanes stepped together
REF_LOCKSTEP_LIB = HERE / "_ref" / "libkfref_lockstep.so"
_ref_lockstep_lib = None


def load_ref_lockstep() -> C.CDLL:
    global _ref_lockstep_lib
    if _ref_lockstep_lib is None:
        _ref_lockstep_lib = C.CDLL(str(REF_LOCKSTEP_LIB))
        _ref_lockstep_lib.kfref_extract_cloud.restype = C.c_longlong
    return _ref_lockstep_lib


REF_DEPTH_LIB = HERE / "_ref" / "libkfref_usedepth.so"
_ref_depth_lib = None


def load_ref_usedepth() -> C.CDLL:
    global _ref_depth_lib
    if _ref_depth_lib is None:
        _ref_depth_lib = C.CDLL(str(REF_DEPTH_LIB))
        _ref_depth_lib.kfref_icp_accumulate_depth.restype = C.c_longlong
    return _ref_depth_lib


class reference:
    """context manager: route the wrappers below to the reference's own kernels (libkfref.so)"""

    def __enter__(self):
        global _use_ref
        load_ref()
        self.prev, _use_ref = _use_ref, True
        return self

    def __exit__(self, *exc):
        global _use_ref
        _use_ref = self.prev
        return False


def _fn(name: str):
    if _use_ref and name == "icp_accumulate_depth":
        return load_ref_usedepth().kfref_icp_accumulate_depth
    if _use_ref and name == "extract_cloud":
        return load_ref_lockstep().kfref_extract_cloud
    if _use_ref:
        return getattr(load_ref(), "kfref_" + name)
    return getattr(load(), "orc_" + name)


def aff(R, t) -> Aff3f:
    a = Aff3f()
    R = np.asarray(R, np.float32).reshape(9)
    t = np.asarray(t, np.float32).reshape(3)
    for i in range(9):
        a.R[i] = float(R[i])
    for i in range(3):
        a.t[i] = float(t[i])
    return a


def intr(fx, fy, cx, cy) -> Intr:
    return Intr(float(fx), float(fy), float(cx), float(cy))


def volume(data: np.ndarray, dims, voxel_size, trunc, max_weight) -> Volume:
    assert data.dtype == np.uint32 and data.flags.c_contiguous
    v = Volume()
    v.data = data.ctypes.data
    for i in range(3):
        v.dims[i] = int(dims[i])
        v.voxel_size[i] = float(voxel_size[i])
    v.trunc_dist = float(trunc)
    v.max_weight = int(max_weight)
    return v


def _p(a: np.ndarray):
    assert a.flags.c_contiguous
    return C.c_void_p(a.ctypes.data)


def _f9(R):
    arr = (C.c_float * 9)(*[float(v) for v in np.asarray(R, np.float32).reshape(9)])
    return arr


# ------------------------------------------------------------------ wrappers (numpy in / numpy out) ------------------------------------------
def clear_volume(vol_data, dims, vs, trunc, mw):
    _fn("clear_volume")(volume(vol_data, dims, vs, trunc, mw))


def compute_dists(depth: np.ndarray, K) -> np.ndarray:
    rows, cols = depth.shape
    out = np.empty_like(depth)
    _fn("compute_dists")(_p(depth), C.c_size_t(cols * 2), cols, rows, intr(*K), _p(out), C.c_size_t(cols * 2))
    return out


def integrate(vol_data, dims, vs, trunc, mw, dists, vol2cam, K) -> int:
    rows, cols = dists.shape
    return int(_fn("integrate")(volume(vol_data, dims, vs, trunc, mw), _p(dists), C.c_size_t(cols * 2), cols, rows,
                                    aff(*vol2cam), intr(*K)))


def integrate_warped(vol_data, dims, vs, trunc, mw, depth, vol2world, world2cam, K, nodes, weight_scale) -> int:
    """per-voxel warped integration (orc_fusion.c); depth = u16 millimetres"""
    rows, cols = depth.shape
    nodes = np.ascontiguousarray(nodes, np.float32)
    return int(load().orc_integrate_warped(volume(vol_data, dims, vs, trunc, mw), _p(depth), C.c_size_t(cols * 2), cols, rows,
                                           aff(*vol2world), aff(*world2cam), intr(*K), _p(nodes), len(nodes), C.c_float(weight_scale)))


def extend_field(nodes, cloud, radius, step, max_nodes) -> np.ndarray:
    """orc_extend_field (orc_fusion.c): returns the extended node table"""
    nodes = np.ascontiguousarray(nodes, np.float32)
    M = len(nodes)
    buf = np.zeros((max_nodes, NODE_STRIDE), np.float32)
    buf[:M] = nodes
    c = np.ascontiguousarray(cloud, np.float32)
    Mn = load().orc_extend_field(_p(buf), M, max_nodes, _p(c), C.c_longlong(len(c)), c.shape[1], C.c_float(radius), step)
    return buf[:Mn].copy()


def raycast_points(vol_data, dims, vs, trunc, mw, cam2vol, Rinv, K, cols, rows, step_factor, delta_factor):
    pts = np.empty((rows, cols, 4), np.float32)
    nrm = np.empty((rows, cols, 4), np.float32)
    stats = (C.c_longlong * 3)()
    _fn("raycast_points")(volume(vol_data, dims, vs, trunc, mw), aff(*cam2vol), _f9(Rinv), intr(*K), cols, rows,
                              C.c_float(step_factor), C.c_float(delta_factor), _p(pts), C.c_size_t(cols * 16), _p(nrm),
                              C.c_size_t(cols * 16), stats)
    return pts, nrm, [int(s) for s in stats]


def project_and_remove(dists: np.ndarray, K, points: np.ndarray):
    rows, cols = dists.shape
    prow, pcol = points.shape[:2]
    _fn("project_and_remove")(_p(dists), C.c_size_t(cols * 2), cols, rows, intr(*K), _p(points), C.c_size_t(pcol * 16), pcol, prow)


def extract_cloud(vol_data, dims, vs, trunc, mw, pose, capacity) -> np.ndarray:
    out = np.empty((capacity, 4), np.float32)
    n = int(_fn("extract_cloud")(volume(vol_data, dims, vs, trunc, mw), aff(*pose), _p(out), C.c_longlong(capacity)))
    return out[:n].copy()


def extract_normals(vol_data, dims, vs, trunc, mw, pts, pose, Rinv, delta_factor) -> np.ndarray:
    out = np.empty_like(pts)
    _fn("extract_normals")(volume(vol_data, dims, vs, trunc, mw), _p(pts), C.c_longlong(len(pts)), aff(*pose), _f9(Rinv),
                               C.c_float(delta_factor), _p(out))
    return out


def bilateral(depth, ksz, sigma_spatial, sigma_depth):
    rows, cols = depth.shape
    out = np.empty_like(depth)
    _fn("bilateral")(_p(depth), C.c_size_t(cols * 2), cols, rows, _p(out), C.c_size_t(cols * 2), ksz, C.c_float(sigma_spatial),
                         C.c_float(sigma_depth))
    return out


def truncate_depth(depth, max_dist):
    rows, cols = depth.shape
    _fn("truncate_depth")(_p(depth), C.c_size_t(cols * 2), cols, rows, C.c_float(max_dist))


def pyr_down(depth, sigma_depth):
    rows, cols = depth.shape
    out = np.empty((rows // 2, cols // 2), np.uint16)
    _fn("pyr_down")(_p(depth), C.c_size_t(cols * 2), cols, rows, _p(out), C.c_size_t((cols // 2) * 2), C.c_float(sigma_depth))
    return out


def points_normals(K, depth):
    rows, cols = depth.shape
    pts = np.empty((rows, cols, 4), np.float32)
    nrm = np.empty((rows, cols, 4), np.float32)
    _fn("points_normals")(intr(*K), _p(depth), C.c_size_t(cols * 2), cols, rows, _p(pts), C.c_size_t(cols * 16), _p(nrm), C.c_size_t(cols * 16))
    return pts, nrm


def resize_points_normals(v, n):
    rows, cols = v.shape[:2]
    vd = np.empty((rows // 2, cols // 2, 4), np.float32)
    nd = np.empty((rows // 2, cols // 2, 4), np.float32)
    _fn("resize_points_normals")(_p(v), C.c_size_t(cols * 16), _p(n), C.c_size_t(cols * 16), cols, rows, _p(vd),
                                     C.c_size_t((cols // 2) * 16), _p(nd), C.c_size_t((cols // 2) * 16))
    return vd, nd


def icp_accumulate(vcurr, ncurr, vprev, nprev, K_level, T, dist2, min_cos):
    rows, cols = vcurr.shape[:2]
    out = np.zeros(27, np.float64)
    n = _fn("icp_accumulate")(_p(vcurr), C.c_size_t(cols * 16), _p(ncurr), C.c_size_t(cols * 16), _p(vprev), C.c_size_t(cols * 16),
                                  _p(nprev), C.c_size_t(cols * 16), cols, rows, intr(*K_level), aff(*T), C.c_float(dist2),
                                  C.c_float(min_cos), _p(out))
    return out, int(n)


def icp_accumulate_depth(dcurr, ncurr, dprev, nprev, K_level, T, dist2, min_cos):
    """USE_DEPTH variant: u16 millimetre depth maps in place of the vertex maps"""
    rows, cols = dcurr.shape[:2]
    dcurr, dprev = np.ascontiguousarray(dcurr, np.uint16), np.ascontiguousarray(dprev, np.uint16)
    out = np.zeros(27, np.float64)
    n = _fn("icp_accumulate_depth")(_p(dcurr), C.c_size_t(cols * 2), _p(ncurr), C.c_size_t(cols * 16), _p(dprev), C.c_size_t(cols * 2),
                                        _p(nprev), C.c_size_t(cols * 16), cols, rows, intr(*K_level), aff(*T), C.c_float(dist2),
                                        C.c_float(min_cos), _p(out))
    return out, int(n)


def icp_rows(vcurr, ncurr, vprev, nprev, K_level, T, dist2, min_cos):
    """the per-pixel rule of icp_accumulate: rows [rows, cols, 7] float32 (NaN where rejected), match [rows, cols] int32 (linear
    index of the matched previous pixel, -1 where rejected) and the inlier count"""
    rows, cols = vcurr.shape[:2]
    out = np.empty((rows, cols, 7), np.float32)
    match = np.empty((rows, cols), np.int32)
    n = load().orc_icp_rows(_p(vcurr), C.c_size_t(cols * 16), _p(ncurr), C.c_size_t(cols * 16), _p(vprev), C.c_size_t(cols * 16),
                            _p(nprev), C.c_size_t(cols * 16), cols, rows, intr(*K_level), aff(*T), C.c_float(dist2), C.c_float(min_cos),
                            _p(out), _p(match))
    return out, match, int(n)


def icp_rows_depth(dcurr, ncurr, dprev, nprev, K_level, T, dist2, min_cos):
    """icp_rows for the USE_DEPTH variant"""
    rows, cols = dcurr.shape[:2]
    dcurr, dprev = np.ascontiguousarray(dcurr, np.uint16), np.ascontiguousarray(dprev, np.uint16)
    out = np.empty((rows, cols, 7), np.float32)
    match = np.empty((rows, cols), np.int32)
    n = load().orc_icp_rows_depth(_p(dcurr), C.c_size_t(cols * 2), _p(ncurr), C.c_size_t(cols * 16), _p(dprev), C.c_size_t(cols * 2),
                                  _p(nprev), C.c_size_t(cols * 16), cols, rows, intr(*K_level), aff(*T), C.c_float(dist2),
                                  C.c_float(min_cos), _p(out), _p(match))
    return out, match, int(n)


def icp_estimate_depth(dcurr, ncurr, dprev, nprev, iters, K, dist_thres, angle_thres):
    L = len(dcurr)
    dcurr = [np.ascontiguousarray(x, np.uint16) for x in dcurr]
    dprev = [np.ascontiguousarray(x, np.uint16) for x in dprev]
    arr = lambda xs: (C.c_void_p * L)(*[x.ctypes.data for x in xs])
    cols = (C.c_int * L)(*[x.shape[1] for x in dcurr])
    rows = (C.c_int * L)(*[x.shape[0] for x in dcurr])
    dpitch = (C.c_size_t * L)(*[x.shape[1] * 2 for x in dcurr])
    npitch = (C.c_size_t * L)(*[x.shape[1] * 16 for x in dcurr])
    it = (C.c_int * L)(*iters[:L])
    a = Aff3f()
    ok = load().orc_icp_estimate_depth(arr(dcurr), arr(ncurr), arr(dprev), arr(nprev), cols, rows, dpitch, npitch, L, it, intr(*K),
                                       C.c_float(dist_thres), C.c_float(angle_thres), C.byref(a))
    return bool(ok), (np.array(list(a.R), np.float32).reshape(3, 3), np.array(list(a.t), np.float32))


def icp_solve_update(sums27, T):
    a = aff(*T)
    s = np.ascontiguousarray(sums27, np.float64)
    ok = _fn("icp_solve_update")(_p(s), C.byref(a))
    return bool(ok), (np.array(list(a.R), np.float32).reshape(3, 3), np.array(list(a.t), np.float32))


def icp_estimate(vcurr, ncurr, vprev, nprev, iters, K, dist_thres, angle_thres):
    L = len(vcurr)
    arr = lambda xs: (C.c_void_p * L)(*[x.ctypes.data for x in xs])
    cols = (C.c_int * L)(*[x.shape[1] for x in vcurr])
    rows = (C.c_int * L)(*[x.shape[0] for x in vcurr])
    pitch = (C.c_size_t * L)(*[x.shape[1] * 16 for x in vcurr])
    it = (C.c_int * L)(*iters[:L])
    a = Aff3f()
    ok = _fn("icp_estimate")(arr(vcurr), arr(ncurr), arr(vprev), arr(nprev), cols, rows, pitch, L, it, intr(*K),
                                 C.c_float(dist_thres), C.c_float(angle_thres), C.byref(a))
    return bool(ok), (np.array(list(a.R), np.float32).reshape(3, 3), np.array(list(a.t), np.float32))


NODE_STRIDE = 12


def make_nodes(vertices, weight=3.0) -> np.ndarray:
    """deformation_node defaults (warp_field.cpp:68-80): identity DualQuaternion() = rot (1,0,0,0), dual (1,0,0,0)"""
    v = np.asarray(vertices, np.float32).reshape(-1, 3)
    n = np.zeros((len(v), NODE_STRIDE), np.float32)
    n[:, 0:3] = v
    n[:, 3] = 1.0
    n[:, 7] = 1.0
    n[:, 11] = weight
    return n


def knn8(nodes, queries):
    q = np.ascontiguousarray(queries, np.float32)
    N, stride = q.shape
    idx = np.empty((N, 8), np.int32)
    d2 = np.empty((N, 8), np.float32)
    _fn("knn8")(_p(nodes), len(nodes), _p(q), C.c_longlong(N), stride, _p(idx), _p(d2))
    return idx, d2


def warp(nodes, points, normals, warp_to_live=None, flags=0):
    """in place on float32 (N, stride) arrays"""
    if warp_to_live is None:
        warp_to_live = (np.eye(3, dtype=np.float32), np.zeros(3, np.float32))
    N, stride = points.shape
    _fn("warp")(_p(nodes), len(nodes), _p(points), _p(normals), C.c_longlong(N), stride, aff(*warp_to_live), flags)


def node_translations(nodes) -> np.ndarray:
    out = np.empty((len(nodes), 4), np.float32)
    for i in range(len(nodes)):
        _fn("node_translation")(C.c_void_p(nodes[i].ctypes.data), C.c_void_p(out[i].ctypes.data))
    return out


def solve_data_term(nodes, canon, live, flags=0, lm_iters=5):
    c = np.ascontiguousarray(canon, np.float32)
    l = np.ascontiguousarray(live, np.float32)
    N, stride = c.shape
    stats = np.zeros(4, np.float64)
    _fn("solve_data_term")(_p(nodes), len(nodes), _p(c), _p(l), C.c_longlong(N), stride, flags, lm_iters, _p(stats))
    return stats


# ------------------------------------------------------------------ SURVEY 8f(2): robust data term + regularisation over 6-DoF increments
class F2Params(C.Structure):
    """orc_f2_params (oracle/orc_reg.c) == df_f2_params (include/dfusion.h)"""
    _fields_ = [("reg_lambda", C.c_double), ("tukey_c", C.c_double), ("huber_delta", C.c_double), ("lm_mu", C.c_double),
                ("gn_iters", C.c_int), ("reg_k", C.c_int), ("flags", C.c_int), ("lin_iters", C.c_int)]


F2_TWIST, F2_TUKEY, F2_HUBER = 1, 2, 4


def f2_params(reg_lambda=0.0, tukey_c=0.01, huber_delta=1e-4, lm_mu=1e-4, gn_iters=3, reg_k=4, flags=0, lin_iters=200) -> F2Params:
    return F2Params(reg_lambda, tukey_c, huber_delta, lm_mu, gn_iters, reg_k, flags, lin_iters)


def solve_f2(nodes: np.ndarray, canon: np.ndarray, live: np.ndarray, prm: F2Params) -> np.ndarray:
    """orc_solve_f2: nodes [M, 12] float32 updated in place; returns the 16 stats"""
    c = np.ascontiguousarray(canon, np.float32)
    l = np.ascontiguousarray(live, np.float32)
    assert nodes.dtype == np.float32 and nodes.flags.c_contiguous and c.shape == l.shape
    stats = np.zeros(16, np.float64)
    load().orc_solve_f2(_p(nodes), len(nodes), _p(c), _p(l), C.c_longlong(len(c)), c.shape[1], C.byref(prm), _p(stats))
    return stats


def f2_edges(nodes: np.ndarray, reg_k: int) -> np.ndarray:
    e = np.empty((len(nodes), reg_k), np.int32)
    load().orc_f2_edges(_p(nodes), len(nodes), reg_k, _p(e))
    return e
