"""ctypes binding of the warped colour oracle (tests/warped_color_oracle.c, over oracle/orc_fusion.c's warped fusion), test infrastructure
only."""
from __future__ import annotations

import ctypes as C

import numpy as np

import c_oracle
import color_oracle as co
import color_camera_oracle as cco
import lens_oracle as lo


def load() -> C.CDLL:
    from oracle import orc
    C.CDLL(str(orc.build()), mode=C.RTLD_GLOBAL)          # the warp this oracle's copy of orc_fusion.c calls
    vp, i, f, sz, ll = C.c_void_p, C.c_int, C.c_float, C.c_size_t, C.c_longlong
    return c_oracle.load("warped_color_oracle", {
        "wc_integrate_warped_records": (ll, [orc.Volume, vp, sz, i, i, orc.Aff3f, orc.Aff3f, orc.Intr, vp, i, f, vp, vp]),
        "wc_fuse": (ll, [ll, vp, vp, f, i, vp, vp, sz, vp, i, i, vp, vp, vp, vp, sz]),
    })


def integrate_warped(vol_data, dims, vs, trunc, mw, depth, vol2world, world2cam, K, nodes, weight_scale):
    """orc_integrate_warped's rule on vol_data (uint32, updated IN PLACE) with the per-voxel records of the voxels it wrote:
    (voxels written, rec float32 [nvox, 6] = tx, ty, tz, u, v, rho, hit bool [nvox])"""
    from oracle import orc
    lib = load()
    rows, cols = depth.shape
    nvox = int(np.prod(dims))
    rec = np.zeros((nvox, 6), np.float32)
    hit = np.zeros(nvox, np.uint8)
    nodes = np.ascontiguousarray(nodes, np.float32)
    depth = np.ascontiguousarray(depth, np.uint16)
    n = lib.wc_integrate_warped_records(orc.volume(vol_data, dims, vs, trunc, mw), depth.ctypes.data, cols * 2, cols, rows, orc.aff(*vol2world),
                                        orc.aff(*world2cam), orc.intr(*K), nodes.ctypes.data, len(nodes), float(weight_scale), rec.ctypes.data,
                                        hit.ctypes.data)
    return int(n), rec, hit.astype(bool)


def fuse(colors, rec, hit, trunc, mw, bgra, K_depth=None, cam: cco.Camera | None = None, lens=None, cmap=None):
    """the colour side of df_integrate_warped_color over integrate_warped's records: colors (uint32 [nvox]) updated IN PLACE; returns the
    voxels coloured.  cam None: bgra registered to the depth; else the colour camera's image, its lens (None, 9 floats or a capi.Lens) and
    cmap (df_color_depth_map_lens of the frame)"""
    assert colors.dtype == np.uint32 and colors.flags.c_contiguous and bgra.dtype == np.uint8 and bgra.strides[1:] == (4, 1)
    h = np.ascontiguousarray(hit, np.uint8)
    rec = np.ascontiguousarray(rec, np.float32)
    k = kc = d2c = L = None
    ccols = crows = 0
    if cam is not None:
        k, kc, d2c, L = np.asarray(K_depth, np.float32), cam.k4(), co.a12(cam.d2c), lo.lens9(lens)
        ccols, crows = cam.cols, cam.rows
    p = lambda a: None if a is None else a.ctypes.data  # noqa: E731
    return int(load().wc_fuse(colors.size, rec.ctypes.data, h.ctypes.data, float(trunc), int(mw), colors.ctypes.data, bgra.ctypes.data,
                              bgra.strides[0], p(k), ccols, crows, p(kc), p(d2c), p(L), p(cmap), 0 if cmap is None else cmap.strides[0]))
