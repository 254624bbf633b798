"""Colour under per-voxel warped fusion on the CPU (df_integrate_warped_color's rule, include/dfusion.h): tests/warped_color_oracle.c over the
per-voxel records of oracle/orc_fusion.c.  The oracle's TSDF side is orc_integrate_warped's bit for bit; on a fronto-parallel wall the
coloured voxels are exactly the band around the wall inside the frustum, each with its own pixel; a field that moves every voxel by t moves
the coloured set by -t; the colour camera's occlusion test accepts and rejects as stated; the zero lens is no lens."""
import ctypes as C

import numpy as np
import pytest

import color_camera_oracle as cco
import lens_oracle as lo
import warped_color_oracle as wco

DIM, VS = 64, 1.0 / 64                       # a power-of-two voxel: every voxel centre and the shifts below are exact in float
TRUNC, MAXW = 0.04, 64
COLS, ROWS, K = 160, 120, (200.0, 200.0, 80.0, 60.0)
POSE = (np.eye(3, dtype=np.float32), np.array([-0.5, -0.5, 0.5], np.float32))
CAM = (np.eye(3, dtype=np.float32), np.zeros(3, np.float32))


def _wall(mm=1000):
    return np.full((ROWS, COLS), mm, np.uint16)


def _pixel_image():
    """BGRA whose pixel (u, v) encodes u and v: B = u, G = v, R = 7"""
    u, v = np.meshgrid(np.arange(COLS), np.arange(ROWS))
    img = np.zeros((ROWS, COLS, 4), np.uint8)
    img[..., 0], img[..., 1], img[..., 2] = u, v, 7
    return img


def _nodes(orc, shift=(0.0, 0.0, 0.0)):
    """8 nodes with a weight so large that every blend weight is 1.0f, each translated by shift / 8: every voxel moves by exactly shift"""
    v = np.array([[x, y, z] for x in (-0.2, 0.2) for y in (-0.2, 0.2) for z in (0.9, 1.1)], np.float32)
    nodes = orc.make_nodes(v, weight=1e4)
    for n in nodes:
        orc.load().orc_node_encode_translation(C.c_void_p(n.ctypes.data), C.c_float(shift[0] / 8), C.c_float(shift[1] / 8), C.c_float(shift[2] / 8))
    return nodes


def _run(orc, nodes, depth=None, weight_scale=0.0):
    vol = np.zeros(DIM ** 3, np.uint32)
    n, rec, hit = wco.integrate_warped(vol, (DIM,) * 3, (VS,) * 3, TRUNC, MAXW, _wall() if depth is None else depth, POSE, CAM, K, nodes,
                                       weight_scale)
    return vol, n, rec, hit


def test_tsdf_side_is_orc_integrate_warped(orc):
    rng = np.random.default_rng(5)
    v = np.concatenate([rng.uniform(-0.45, 0.45, (60, 2)), rng.uniform(0.95, 1.05, (60, 1))], axis=1).astype(np.float32)
    nodes = orc.make_nodes(v, weight=0.05)
    for n in nodes:
        t = rng.uniform(-0.01, 0.01, 3)
        orc.load().orc_node_encode_translation(C.c_void_p(n.ctypes.data), C.c_float(t[0]), C.c_float(t[1]), C.c_float(t[2]))
    depth = (1000 + 60 * np.sin(np.arange(COLS) / 9.0)[None, :] + np.zeros((ROWS, 1))).astype(np.uint16)
    depth[:10] = 0
    for ws in (0.0, 100.0):
        vol, n, rec, hit = _run(orc, nodes, depth, ws)
        ref = np.zeros(DIM ** 3, np.uint32)
        n_ref = orc.integrate_warped(ref, (DIM,) * 3, (VS,) * 3, TRUNC, MAXW, depth, POSE, CAM, K, nodes, ws)
        assert n == n_ref > 10000 and np.array_equal(vol, ref)
        assert int(hit.sum()) == n


def test_wall_band_inside_frustum(orc):
    vol, n, rec, hit = _run(orc, _nodes(orc))
    colors = np.zeros(DIM ** 3, np.uint32)
    n_col = wco.fuse(colors, rec, hit, TRUNC, MAXW, _pixel_image())
    z, y, x = np.meshgrid(np.arange(DIM), np.arange(DIM), np.arange(DIM), indexing="ij")
    X, Y, Z = (x * VS - 0.5).ravel(), (y * VS - 0.5).ravel(), (z * VS + 0.5).ravel()     # exact: the field is the identity here
    u, v = K[0] * X / Z + K[2], K[1] * Y / Z + K[3]
    inside = (u >= 0) & (v >= 0) & (u < COLS) & (v < ROWS)
    band = np.abs(np.float32(1.0) - Z.astype(np.float32)) <= np.float32(0.5) * np.float32(TRUNC)
    # pixels within 1e-4 of a pixel edge may round either way in float: leave them out of the exact comparison
    safe = (np.abs(u - np.round(u)) > 1e-4) & (np.abs(v - np.round(v)) > 1e-4)
    coloured = (colors >> 24) != 0
    assert n_col == int(coloured.sum()) > 1000
    assert np.array_equal(coloured[safe], (inside & band)[safe])
    c = colors[coloured & safe]
    assert np.array_equal(c & 0xff, np.full(c.shape, 7))                          # R = byte 2 of the BGRA pixel
    assert np.array_equal((c >> 8) & 0xff, np.floor(v[coloured & safe]).astype(np.uint32))   # G = v
    assert np.array_equal((c >> 16) & 0xff, np.floor(u[coloured & safe]).astype(np.uint32))  # B = u
    assert np.all(c >> 24 == 1)


def test_translated_field_moves_the_coloured_set(orc):
    img = _pixel_image()
    out = []
    for shift in ((0, 0, 0), (3, -2, 4)):
        vol, n, rec, hit = _run(orc, _nodes(orc, tuple(np.float32(s * VS) for s in shift)))
        colors = np.zeros(DIM ** 3, np.uint32)
        wco.fuse(colors, rec, hit, TRUNC, MAXW, img)
        out.append(colors.reshape(DIM, DIM, DIM))
    c0, ct = out
    # voxel x under the shifted field lands where voxel x + t lands under the identity field: same sample, same word
    sx, sy, sz = 3, -2, 4
    a = ct[max(0, -sz):DIM - max(0, sz), max(0, -sy):DIM - max(0, sy), max(0, -sx):DIM - max(0, sx)]
    b = c0[max(0, sz):DIM - max(0, -sz), max(0, sy):DIM - max(0, -sy), max(0, sx):DIM - max(0, -sx)]
    assert np.count_nonzero(b >> 24) > 1000 and np.array_equal(a, b)


def test_color_camera_occlusion(orc):
    vol, n, rec, hit = _run(orc, _nodes(orc))
    img = _pixel_image()
    reg = np.zeros(DIM ** 3, np.uint32)
    wco.fuse(reg, rec, hit, TRUNC, MAXW, img)
    cam = cco.Camera(COLS, ROWS, K, CAM)                  # the depth camera's twin: a voxel reaches the same pixel as registered
    open_map = lo.depth_map(_wall(), K, cam, None)
    got = np.zeros(DIM ** 3, np.uint32)
    wco.fuse(got, rec, hit, TRUNC, MAXW, img, K, cam, None, open_map)
    # accepted: every band voxel is within DF_COLOR_OCCLUSION * trunc of the wall (a few cells that no reprojected depth pixel lands in
    # stay empty and reject, and the fma chain of depth_to_color can move a pixel across an edge: most, not all, words are the registered ones)
    n_reg = np.count_nonzero(reg >> 24)
    assert np.count_nonzero((got == reg) & (reg != 0)) >= 0.95 * n_reg > 1000
    near = _wall()
    near[:, : COLS // 2] = 800                            # something 20 cm nearer covers the left half of the colour image
    occl = np.zeros(DIM ** 3, np.uint32)
    wco.fuse(occl, rec, hit, TRUNC, MAXW, img, K, cam, None, lo.depth_map(near, K, cam, None))
    cell = cco.cell(K, cam)
    left = ((reg >> 16) & 0xff) < (COLS // 2 // cell) * cell   # the pixel's map cell lies under the occluder
    assert np.count_nonzero(reg[left] >> 24) > 100 and np.all(occl[left] == 0)
    assert np.array_equal(occl[~left], got[~left])       # the rest is what the open map gave


def test_zero_lens_is_no_lens(orc):
    vol, n, rec, hit = _run(orc, _nodes(orc))
    img = _pixel_image()
    cam = cco.Camera(COLS, ROWS, (190.0, 195.0, 81.0, 58.5), (np.eye(3, dtype=np.float32), np.array([0.02, 0.0, 0.0], np.float32)))
    cmap = lo.depth_map(_wall(), K, cam, None)
    a, b = np.zeros(DIM ** 3, np.uint32), np.zeros(DIM ** 3, np.uint32)
    na = wco.fuse(a, rec, hit, TRUNC, MAXW, img, K, cam, None, cmap)
    nb = wco.fuse(b, rec, hit, TRUNC, MAXW, img, K, cam, np.array([0] * 8 + [4.0], np.float32), cmap)
    assert na == nb > 1000 and np.array_equal(a, b)
    c = np.zeros(DIM ** 3, np.uint32)
    nc = wco.fuse(c, rec, hit, TRUNC, MAXW, img, K, cam, np.array([0.1, -0.02, 0, 0, 0, 0, 0, 0, 4.0], np.float32), cmap)
    assert nc > 1000 and not np.array_equal(a, c)
