"""CPU checks of the colour feature: the three rules of include/dfusion.h as tests/color_oracle.c states them (closed forms on small scenes),
the synthetic RGB-D scene, the coloured PLY export and the version-2 snapshot checks of df_kinfu_snapshot_params (host code)."""
import struct

import numpy as np
import pytest

import color_oracle as co
import snapshot_model as sm
from scenes import BAND, COLS, DIMS, K, ROWS, TRUNC, VOL2CAM, VS, constant_image, plane_dists, word
from snapshot_model import lib  # noqa: F401  (a fixture)


def voxel_sdf(dists):
    """float64 model of the rule's sdf per voxel (NaN where the rule skips the voxel before the band test)"""
    z, y, x = np.meshgrid(np.arange(DIMS[2]), np.arange(DIMS[1]), np.arange(DIMS[0]), indexing="ij")
    vc = np.stack([x * VS[0], y * VS[1], z * VS[2]], -1).astype(np.float64) + VOL2CAM[1].astype(np.float64)
    u = K[0] * vc[..., 0] / vc[..., 2] + K[2]
    v = K[1] * vc[..., 1] / vc[..., 2] + K[3]
    ok = (u >= 0) & (v >= 0) & (u < COLS) & (v < ROWS) & (vc[..., 2] > 0)
    Dp = dists.view(np.float16).astype(np.float64)[np.clip(v.astype(int), 0, ROWS - 1), np.clip(u.astype(int), 0, COLS - 1)]
    sdf = Dp - np.linalg.norm(vc, axis=-1)
    return np.where(ok & (Dp != 0), sdf, np.nan).reshape(-1)


def integrate(colors, img, dists=None, activity=None, max_weight=64):
    return co.integrate_color(colors, DIMS, VS, TRUNC, max_weight, plane_dists() if dists is None else dists, img, VOL2CAM, K, activity)


def test_plane_colours_exactly_the_band():
    dists = plane_dists()
    colors = integrate(np.zeros(np.prod(DIMS), np.uint32), constant_image((10, 20, 30)), dists)
    sdf = voxel_sdf(dists)
    with np.errstate(invalid="ignore"):
        surely_in, surely_out = np.abs(sdf) < BAND - 1e-5, ~(np.abs(sdf) < BAND + 1e-5)
    assert surely_in.sum() > 1000
    assert np.all(colors[surely_in] == word(30, 20, 10, 1))             # the image is B, G, R; the voxel R, G, B, W
    assert np.all(colors[surely_out] == 0)
    assert set(np.unique(colors)) == {0, word(30, 20, 10, 1)}


def test_weight_counts_frames_up_to_the_cap():
    colors = np.zeros(np.prod(DIMS), np.uint32)
    img = constant_image((1, 2, 3))
    for k in range(1, 6):
        integrate(colors, img, max_weight=3)
        assert set(np.unique(colors >> 24)) == {0, min(k, 3)}
    colors[:] = 0
    for _ in range(3):
        integrate(colors, img, max_weight=1000)                         # the weight byte caps at 255
    assert (colors >> 24).max() == 3


def test_running_average_closed_form():
    colors = np.zeros(np.prod(DIMS), np.uint32)
    seq = [(0, 0, 0)] * 2 + [(255, 101, 7)] * 5
    c, W = np.zeros(3, np.int64), 0
    for bgr in seq:
        integrate(colors, constant_image(bgr), max_weight=4)
        s = np.array(bgr[::-1], np.int64)
        c = (c * W + s + ((W + 1) >> 1)) // (W + 1)
        W = min(W + 1, 4)
        assert set(np.unique(colors)) == {0, word(int(c[0]), int(c[1]), int(c[2]), W)}
    # two colours, W below the cap: the rounded mean
    colors[:] = 0
    integrate(colors, constant_image((0, 0, 10)))
    integrate(colors, constant_image((0, 0, 13)))
    assert set(np.unique(colors)) == {0, word(12, 0, 0, 2)}             # (10 + 13 + 1) // 2


def test_activity_byte_zero_suppresses_its_stretch():
    full = integrate(np.zeros(np.prod(DIMS), np.uint32), constant_image((9, 9, 9)))
    nstretch = (np.prod(DIMS) + 1023) // 1024
    act = np.ones(nstretch, np.uint8)
    touched = np.unique(np.flatnonzero(full) // 1024)
    off = touched[len(touched) // 2]
    act[off] = 0
    part = integrate(np.zeros(np.prod(DIMS), np.uint32), constant_image((9, 9, 9)), activity=act)
    sl = slice(off * 1024, (off + 1) * 1024)
    assert full[sl].any() and not part[sl].any()
    part[sl] = full[sl]
    assert np.array_equal(part, full)


# ------------------------------------------------------------------------------------------------------------------------- sampler
POSE = (np.eye(3, dtype=np.float32), np.array([-0.32, -0.24, 0.5], np.float32))


def grid_points(g, offset):
    """world points whose grid coordinate is g (float64 model): p = pose * ((g + offset) * vs)"""
    return ((np.asarray(g, np.float64) + offset) * np.array(VS) + POSE[1].astype(np.float64)).astype(np.float32)


def test_sampler_constant_and_ramp():
    rng = np.random.default_rng(1)
    g = rng.uniform(1.0, np.array(DIMS) - 2.0, (500, 3))
    colors = np.full(np.prod(DIMS), word(40, 50, 60, 3), np.uint32)
    out = co.sample_colors(colors, DIMS, VS, POSE, 0.0, grid_points(g, 0.0))
    assert np.all(out == (40, 50, 60, 255))
    z, y, x = np.meshgrid(np.arange(DIMS[2]), np.arange(DIMS[1]), np.arange(DIMS[0]), indexing="ij")
    ramp = ((2 * x + 10) | ((3 * y + 20) << 8) | ((4 * z + 30) << 16) | (1 << 24)).astype(np.uint32).reshape(-1)
    out = co.sample_colors(ramp, DIMS, VS, POSE, 0.0, grid_points(g, 0.0)).astype(np.float64)
    want = np.stack([2 * g[:, 0] + 10, 3 * g[:, 1] + 20, 4 * g[:, 2] + 30], -1)
    assert np.abs(out[:, :3] - want).max() <= 1.0 and np.all(out[:, 3] == 255)


def test_sampler_leaves_out_uncoloured_corners():
    colors = np.zeros(np.prod(DIMS), np.uint32)
    idx = lambda x, y, z: x + DIMS[0] * (y + DIMS[1] * z)
    colors[idx(5, 6, 7)] = word(100, 0, 0, 1)
    colors[idx(6, 6, 7)] = word(200, 0, 0, 1)
    out = co.sample_colors(colors, DIMS, VS, POSE, 0.0, grid_points([[5.25, 6.5, 7.5]], 0.0))
    assert tuple(out[0]) == (125, 0, 0, 255)                            # 0.75 * 100 + 0.25 * 200 over the two coloured corners only
    out = co.sample_colors(colors, DIMS, VS, POSE, 0.0, grid_points([[10.5, 6.5, 7.5]], 0.0))
    assert tuple(out[0]) == (0, 0, 0, 0)                                # no coloured corner


def test_sampler_nan_and_outside_give_zero():
    colors = np.full(np.prod(DIMS), word(1, 2, 3, 1), np.uint32)
    pts = grid_points([[-0.5, 3, 3], [3, 3, DIMS[2] - 0.5], [3, DIMS[1] - 1, 3], [3, 3, 3]], 0.0)
    pts = np.concatenate([pts, [[np.nan, 0, 0], [0.0, np.nan, 0.7]]]).astype(np.float32)
    out = co.sample_colors(colors, DIMS, VS, POSE, 0.0, pts)
    assert np.array_equal(out.view(np.uint32).reshape(-1) != 0, [False, False, False, True, False, False])


def test_sampler_offset_joins_the_two_voxel_conventions():
    rng = np.random.default_rng(2)
    colors = (rng.integers(0, 2 ** 24, np.prod(DIMS)).astype(np.uint32) | np.uint32(1 << 24))
    g = rng.uniform(1.0, np.array(DIMS) - 2.0, (300, 3))
    g[:, 0] = np.floor(g[:, 0])                                         # cloud points lie on voxel edges
    raycast = co.sample_colors(colors, DIMS, VS, POSE, 0.0, grid_points(g, 0.0))
    cloud = co.sample_colors(colors, DIMS, VS, POSE, 0.5, grid_points(g, 0.5))
    assert np.abs(raycast.astype(int) - cloud.astype(int)).max() <= 1  # the same physical sample up to float rounding of g
    shifted = co.sample_colors(colors, DIMS, VS, POSE, 0.0, grid_points(g, 0.5))
    assert np.abs(raycast.astype(int) - shifted.astype(int)).max() > 20  # forgetting the offset is visible


# --------------------------------------------------------------------------------------------------------------------- mesh colours
def one_triangle_view():
    verts = np.array([[-0.5, -0.5, 1.0], [0.5, -0.5, 1.2], [0.0, 0.6, 0.9]], np.float32)
    tris = np.array([[0, 1, 2]], np.int32)
    rows, cols = 24, 32
    ids = np.full((rows, cols), -1, np.int32)
    pts = np.full((rows, cols, 4), np.nan, np.float32)
    rng = np.random.default_rng(4)
    for j in range(rows):
        for i in range(cols):
            b = rng.dirichlet([1, 1, 1])
            if (i + j) % 3:
                ids[j, i] = 0
                pts[j, i, :3] = b @ verts
                pts[j, i, 3] = 0
    return verts, tris, ids, pts, (np.eye(3, dtype=np.float32), np.zeros(3, np.float32))


def test_mesh_colours_rule():
    verts, tris, ids, pts, cam = one_triangle_view()
    drawn = ids >= 0
    rgba = np.array([[10, 20, 30, 255]] * 3, np.uint8)
    img, w = co.mesh_colors(ids, pts, verts, tris, cam, rgba, want_weights=True)
    assert np.abs(w[drawn].sum(-1) - 1).max() < 1e-5 and np.isnan(w[~drawn]).all()
    assert np.all(img[drawn] == (30, 20, 10, 0)) and not img[~drawn].any()   # one colour in, that colour out; B, G, R, 0
    rgba = np.array([[200, 0, 0, 255], [0, 200, 0, 255], [0, 0, 200, 255]], np.uint8)
    img = co.mesh_colors(ids, pts, verts, tris, cam, rgba)
    want = np.rint(np.clip(w[drawn], 0, 1) * 200)
    assert np.abs(img[drawn][:, [2, 1, 0]].astype(int) - want).max() <= 1
    rgba[1] = 0                                                         # vertex 1 has no colour: left out, the rest renormalised
    img = co.mesh_colors(ids, pts, verts, tris, cam, rgba)
    keep = drawn & (w[..., 0] + w[..., 2] > 1e-3)
    want = 200 * w[keep][:, [0, 2]] / (w[keep][:, [0]] + w[keep][:, [2]])
    assert np.abs(img[keep][:, [2, 0]].astype(int) - want).max() <= 1 and not img[keep][:, 1].any()
    assert not co.mesh_colors(ids, pts, verts, tris, cam, np.zeros((3, 4), np.uint8)).any()


# --------------------------------------------------------------------------------------------------------------------- synthetic scene
def test_umbrella_rgbd_matches_depth_and_texture():
    from dynamicfusion_b200 import synth
    for t in (0, 9):
        depth, bgra = synth.umbrella_rgbd(t, cols=160, rows=120, K=synth.scaled_K(160, 120))
        assert np.array_equal(depth, synth.umbrella_depth(t, cols=160, rows=120, K=synth.scaled_K(160, 120)))
        assert bgra.shape == (120, 160, 4) and bgra.dtype == np.uint8 and np.all(bgra[..., 3] == 255)
        s, which, pts = synth._umbrella_hits(t, 160, 120, synth.scaled_K(160, 120), 1.3, True, None)
        for k, name in enumerate(("cap", "wall", "sphere")):
            m = which == k
            assert m.any()
            assert np.array_equal(synth.umbrella_texture(pts[m], name), bgra[m][:, 2::-1])
    cap = synth.umbrella_texture(np.array([[0.0, 0.0, 0.9], [0.05, 0.0, 0.9]]))
    assert tuple(cap[0]) == (128, 128, 128) and cap[1, 0] == 228         # a fixed function of the material coordinates


# ----------------------------------------------------------------------------------------------------------------------------- PLY
def test_save_ply_with_colours(tmp_path):
    from dynamicfusion_b200.host import save_ply
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [np.nan, 0, 0]], np.float32)
    n = np.array([[0, 0, 1]] * 3 + [[np.nan] * 3], np.float32)
    f = np.array([[0, 1, 2]], np.int32)
    c = np.array([[255, 0, 0, 255], [0, 255, 0, 255], [1, 2, 3, 255], [0, 0, 0, 0]], np.uint8)
    path = tmp_path / "m.ply"
    assert save_ply(path, v, n, f, colors=c) == 4
    raw = path.read_bytes()
    head, body = raw.split(b"end_header\n", 1)
    lines = head.decode().splitlines()
    assert lines[3:13] == ["element vertex 4", "property float x", "property float y", "property float z", "property float nx", "property float ny",
                           "property float nz", "property uchar red", "property uchar green", "property uchar blue"]
    rec = np.frombuffer(body[:4 * 27], np.dtype([("f", "<f4", (6,)), ("c", "u1", (3,))]))
    assert np.array_equal(rec["c"], c[:, :3]) and np.array_equal(rec["f"][:3, :3], v[:3])
    assert body[4 * 27:] == b"\x03" + f.tobytes()
    plain = tmp_path / "p.ply"
    save_ply(plain, v, n, f)
    assert b"red" not in plain.read_bytes()                             # without colours the file is what it was
    assert save_ply(tmp_path / "c.ply", v, colors=c) == 3               # a cloud drops its NaN point together with its colour
    with pytest.raises(ValueError):
        save_ply(path, v, n, f, colors=c[:2])


# ------------------------------------------------------------------------------------------------------------------------- snapshots
def test_snapshot_version_2_checks(lib):
    from dynamicfusion_b200 import capi
    from dynamicfusion_b200.kinfu import COLOR
    p1, p2 = sm.small_params(capi, lib, 0), sm.small_params(capi, lib, COLOR)
    dims = tuple(p2.volume_dims)
    v1 = sm.v1_body(capi, lib, p1)
    st, out = sm.read_params(lib, capi, sm.header(v1) + v1)
    assert st == 0 and bytes(out) == bytes(p1)                          # a version-1 byte string is still accepted
    length, cls, payload, rgba = sm.color_sections(dims)
    body = sm.v1_body(capi, lib, p2) + length + cls + payload + rgba
    snap = sm.header(body, version=2) + body
    st, out = sm.read_params(lib, capi, snap)
    assert st == 0 and bytes(out) == bytes(p2) and out.flags & COLOR

    def rejected(b, version=2):
        return sm.read_params(lib, capi, sm.header(b, version=version) + b)[0] != 0
    assert rejected(body, version=1)                                    # the version must match the colour flag
    assert rejected(v1, version=2)
    assert rejected(body, version=3)
    assert rejected(body[:-4])                                          # a colour word short
    assert rejected(body + b"\0\0\0\0")
    assert rejected(sm.v1_body(capi, lib, p2))                          # the colour sections missing altogether
    bad = bytearray(cls); bad[5] = 3
    assert rejected(sm.v1_body(capi, lib, p2) + length + bytes(bad) + payload + rgba)
    swap = bytearray(cls); swap[list(cls).index(1)] = 2                 # classes that imply another payload length
    assert rejected(sm.v1_body(capi, lib, p2) + length + bytes(swap) + payload + rgba)
    assert rejected(sm.v1_body(capi, lib, p2) + struct.pack("<Q", 4 * 512) + cls + payload[4:] + rgba)
    assert rejected(sm.v1_body(capi, lib, p2) + struct.pack("<Q", 2 ** 62) + cls + payload + rgba)
    corrupt = bytearray(snap); corrupt[-10] ^= 1                        # the checksum covers the colour sections
    assert sm.read_params(lib, capi, bytes(corrupt))[0] != 0


def test_cpp_colour_export_builds():
    from pathlib import Path
    from dynamicfusion_b200 import build
    root = Path(__file__).resolve().parents[1]
    exe = build.build_cpp_program(root / "tests" / "cpp" / "color_export.cpp", root / "tests" / "cpp" / "_build" / "color_export")
    assert exe.exists()
