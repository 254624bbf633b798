"""ctypes binding of the mesh oracle (tests/mesh_oracle.c), test infrastructure only."""
from __future__ import annotations

import ctypes as C

import numpy as np

import c_oracle


class _Volume(C.Structure):
    _fields_ = [("data", C.c_void_p), ("dims", C.c_int * 3)]


def load() -> C.CDLL:
    return c_oracle.load("mesh_oracle", {
        "mo_vertex_map": (C.c_longlong, [_Volume, C.c_void_p]),
        "mo_mesh": (C.c_longlong, [_Volume, C.c_longlong, C.c_void_p, C.c_longlong]),
    })


def _vol(vol_data: np.ndarray, dims) -> _Volume:
    assert vol_data.dtype == np.uint32 and vol_data.flags.c_contiguous and vol_data.size == int(np.prod(dims))
    v = _Volume()
    v.data = vol_data.ctypes.data
    for i in range(3):
        v.dims[i] = int(dims[i])
    return v


def vertex_map(vol_data: np.ndarray, dims) -> np.ndarray:
    """[Dz, Dy, Dx, 3] cloud index of the point each voxel emits on each axis, -1 where none"""
    out = np.empty(int(np.prod(dims)) * 3, np.int32)
    load().mo_vertex_map(_vol(vol_data, dims), out.ctypes.data)
    return out.reshape(dims[2], dims[1], dims[0], 3)


def mesh(vol_data: np.ndarray, dims, cloud_count: int) -> np.ndarray | None:
    """the [T, 3] int32 triangles over a cloud of cloud_count points, None when the volume holds another number of points"""
    v = _vol(vol_data, dims)
    n = int(load().mo_mesh(v, cloud_count, None, 0))
    if n < 0:
        return None
    out = np.empty((n, 3), np.int32)
    load().mo_mesh(v, cloud_count, out.ctypes.data, n)
    return out
