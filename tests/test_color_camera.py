"""CPU checks of the colour camera (df_color_camera): df_color_map_dims' cell rule, the occlusion map and the occlusion test as
tests/color_camera_oracle.c states them (hand-built cases), the version-3 snapshot checks of df_kinfu_snapshot_params /
df_kinfu_snapshot_color_camera (host code) and the synthetic scene seen from a colour camera."""
import ctypes as C
import struct

import numpy as np
import pytest

import color_camera_oracle as cco
import color_oracle as co
import snapshot_model as sm
from scenes import COLS, DIMS, K, ROWS, TRUNC, VOL2CAM, VS, constant_image, plane_dists
from snapshot_model import lib  # noqa: F401  (a fixture)

IDENTITY = (np.eye(3, dtype=np.float32), np.zeros(3, np.float32))


def f32_bits(x):
    return int(np.float32(x).view(np.uint32))


# ------------------------------------------------------------------------------------------------------------------------- cells
@pytest.mark.parametrize("Kd,Kc,want", [((570.342, 570.342, 320, 240), (1620, 1620, 959.5, 539.5), 3),      # colour larger
                                        ((570.342, 570.342, 320, 240), (285.171, 285.171, 159.5, 119.5), 1),  # smaller: never below 1
                                        ((570.342, 570.342, 320, 240), (1081.37, 1081.37, 959.5, 539.5), 2),  # Kinect v2 class
                                        ((365.0, 365.0, 256, 212), (1081.37, 1081.37, 959.5, 539.5), 3),
                                        ((500.0, 500.0, 320, 240), (1000.0, 1000.0, 320, 240), 2),            # an exact ratio is not rounded up
                                        ((500.0, 400.0, 320, 240), (600.0, 1300.0, 320, 240), 4)])            # the larger of the two axes
def test_cell_rule(lib, Kd, Kc, want):
    from dynamicfusion_b200 import capi
    cam = cco.Camera(1919, 1081, Kc)
    assert cco.cell(Kd, cam) == want
    mc, mr, cell = C.c_int(), C.c_int(), C.c_int()
    assert lib.df_color_map_dims(capi.make_intr(*Kd), capi.make_color_camera(Kc, 1919, 1081), C.byref(mc), C.byref(mr), C.byref(cell)) == 0
    assert (mc.value, mr.value, cell.value) == cco.map_dims(Kd, cam) == (-(-1919 // want), -(-1081 // want), want)


def test_map_dims_refuses_invalid_cameras(lib):
    from dynamicfusion_b200 import capi
    Kd = capi.make_intr(570.342, 570.342, 320, 240)
    good = ((1081.0, 1081.0, 959.5, 539.5), 1920, 1080, ((1, 0, 0, 0, 1, 0, 0, 0, 1), (0.052, 0, 0)))
    mc = C.c_int(-7)
    assert lib.df_color_map_dims(Kd, capi.make_color_camera(*good), C.byref(mc), None, None) == 0 and mc.value == 960   # cell 2
    bad = [((0.0, 1081.0, 959.5, 539.5), 1920, 1080), ((1081.0, -1.0, 959.5, 539.5), 1920, 1080), ((float("nan"), 1081.0, 959.5, 539.5), 1920, 1080),
           ((1081.0, 1081.0, float("inf"), 539.5), 1920, 1080), ((1081.0, 1081.0, 959.5, 539.5), 0, 1080), ((1081.0, 1081.0, 959.5, 539.5), 1920, 16385)]
    for K_, c_, r_ in bad:
        mc.value = -7
        assert lib.df_color_map_dims(Kd, capi.make_color_camera(K_, c_, r_, good[3]), C.byref(mc), None, None) != 0 and mc.value == -7
    cam = capi.make_color_camera(*good)
    cam.depth_to_color.t[2] = float("nan")
    assert lib.df_color_map_dims(Kd, cam, C.byref(mc), None, None) != 0
    assert lib.df_color_map_dims(capi.make_intr(0.0, 570.0, 320, 240), capi.make_color_camera(*good), C.byref(mc), None, None) != 0


# ------------------------------------------------------------------------------------------------------------------------- the map
KD = (100.0, 100.0, 8.0, 6.0)                # a 16 x 12 depth camera
DC, DR = 16, 12


def test_map_of_an_empty_frame_is_empty():
    m = cco.depth_map(np.zeros((DR, DC), np.uint16), KD, cco.Camera(40, 30, (200.0, 200.0, 20.0, 15.0)))
    assert m.shape == (15, 20) and np.all(m == cco.EMPTY)


def test_map_splats_the_nearest_depth():
    cam = cco.Camera(DC, DR, KD, (np.eye(3, dtype=np.float32), np.array([0.05, 0.0, 0.0], np.float32)))   # 5 cm baseline along x
    depth = np.zeros((DR, DC), np.uint16)
    depth[6, 8] = 1000                                                  # the principal ray at 1 m: lands at u = 8 + 100 * 0.05 = 13
    m = cco.depth_map(depth, KD, cam)
    assert cco.cell(KD, cam) == 1
    assert m[6, 13] == f32_bits(np.float32(1000) * np.float32(0.001)) and (m != cco.EMPTY).sum() == 1
    depth[6, 8] = 500                                                   # at 0.5 m the baseline moves it twice as far: u = 18, outside
    assert np.all(cco.depth_map(depth, KD, cam) == cco.EMPTY)
    # two depth pixels into one colour pixel: the nearer wins, whichever comes first; equal depths tie on the same word
    cam0 = cco.Camera(DC, DR, KD, IDENTITY)
    wide = cco.Camera(DC // 2, DR // 2, (50.0, 50.0, 4.0, 3.0), IDENTITY)  # half the resolution: 2 x 2 depth pixels per colour pixel
    depth = np.zeros((DR, DC), np.uint16)
    depth[6, 8], depth[6, 9] = 1200, 900
    m = cco.depth_map(depth, KD, wide)
    assert m[3, 4] == f32_bits(np.float32(900) * np.float32(0.001)) and (m != cco.EMPTY).sum() == 1
    depth[6, 8], depth[6, 9] = 900, 1200
    assert np.array_equal(cco.depth_map(depth, KD, wide), m)
    depth[6, 9] = 900
    assert np.array_equal(cco.depth_map(depth, KD, wide), m)
    # a colour camera of 3x the focal length: cells of 3 x 3 colour pixels
    tele = cco.Camera(48, 36, (300.0, 300.0, 24.0, 18.0), IDENTITY)
    assert cco.map_dims(KD, tele) == (16, 12, 3)
    depth = np.full((DR, DC), 800, np.uint16)
    m = cco.depth_map(depth, KD, tele)
    full = m != cco.EMPTY
    assert np.all(m[full] == f32_bits(np.float32(800) * np.float32(0.001))) and full.mean() > 0.7 and cco.map_dims(KD, cam0)[2] == 1
    near = np.zeros_like(full)                                          # a cell the frame covers and misses has a covered neighbour
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            near |= np.roll(np.roll(full, dy, 0), dx, 1)
    assert near[1:-1, 1:-1].all()


def test_points_behind_the_colour_camera_are_skipped():
    depth = np.full((DR, DC), 1000, np.uint16)
    ahead = cco.Camera(DC, DR, KD, (np.eye(3, dtype=np.float32), np.array([0.0, 0.0, -1.5], np.float32)))   # 1.5 m in front of the depth camera
    assert np.all(cco.depth_map(depth, KD, ahead) == cco.EMPTY)
    near = cco.Camera(DC, DR, KD, (np.eye(3, dtype=np.float32), np.array([0.0, 0.0, -0.5], np.float32)))
    m = cco.depth_map(depth, KD, near)
    seen = m[m != cco.EMPTY]
    assert len(seen) > 0 and np.all(seen == f32_bits(np.float32(1.0) - np.float32(0.5)))
    flip = cco.Camera(DC, DR, KD, (np.diag([1, 1, -1]).astype(np.float32), np.zeros(3, np.float32)))        # looking backwards
    assert np.all(cco.depth_map(depth, KD, flip) == cco.EMPTY)


# ------------------------------------------------------------------------------------------------------------------- occlusion
ID_CAM = cco.Camera(COLS, ROWS, K, IDENTITY)


def camera_integrate(img, cmap, cam=ID_CAM, dists=None, colors=None):
    colors = np.zeros(np.prod(DIMS), np.uint32) if colors is None else colors
    return cco.integrate_color_camera(colors, DIMS, VS, TRUNC, 64, plane_dists() if dists is None else dists, VOL2CAM, K, cam, img, cmap)


def constant_map(z, cam=ID_CAM):
    mc, mr, _ = cco.map_dims(K, cam)
    return np.full((mr, mc), f32_bits(z) if z is not None else cco.EMPTY, np.uint32)


def voxel_z():
    z, y, x = np.meshgrid(np.arange(DIMS[2]), np.arange(DIMS[1]), np.arange(DIMS[0]), indexing="ij")
    return (z * VS[2] + VOL2CAM[1][2]).reshape(-1).astype(np.float64)


def test_identity_camera_with_an_unblocked_map_is_the_registered_rule():
    img = constant_image((10, 20, 30))
    reg = co.integrate_color(np.zeros(np.prod(DIMS), np.uint32), DIMS, VS, TRUNC, 64, plane_dists(), img, VOL2CAM, K)
    assert (reg != 0).sum() > 1000
    assert np.array_equal(camera_integrate(img, constant_map(0.7)), reg)
    rng = np.random.default_rng(5)
    noisy = rng.integers(0, 256, (ROWS, COLS, 4), np.uint8)            # the sample is the same pixel of the same image
    reg = co.integrate_color(np.zeros(np.prod(DIMS), np.uint32), DIMS, VS, TRUNC, 64, plane_dists(), noisy, VOL2CAM, K)
    assert np.array_equal(camera_integrate(noisy, constant_map(0.7)), reg)


def test_occlusion_accepts_and_rejects():
    img = constant_image((10, 20, 30))
    reg = camera_integrate(img, constant_map(0.7))
    assert not camera_integrate(img, constant_map(None)).any()          # an empty cell never colours
    assert not camera_integrate(img, constant_map(0.5)).any()           # a surface 20 cm nearer hides the whole band
    # zmin + tolerance splits the band: voxels behind it (camera z, the plane is fronto-parallel) are hidden
    z0 = 0.7 - TRUNC
    part = camera_integrate(img, constant_map(z0))
    vz = voxel_z()
    thr = np.float64(np.float32(np.float32(z0) + np.float32(1.0 * TRUNC)))
    assert np.all(part[(reg != 0) & (vz < thr - 1e-6)] == reg[(reg != 0) & (vz < thr - 1e-6)])
    assert not part[vz > thr + 1e-6].any()
    assert 0 < (part != 0).sum() < (reg != 0).sum()
    # an occluder over part of the image: only the voxels seen through those cells lose their colour
    cmap = constant_map(0.7)
    cmap[10:20, 20:40] = f32_bits(0.3)
    occ = camera_integrate(img, cmap)
    lost = (reg != 0) & (occ == 0)
    assert lost.sum() > 100 and np.array_equal(occ[occ != 0], reg[occ != 0])
    vc = np.stack(np.meshgrid(np.arange(DIMS[2]), np.arange(DIMS[1]), np.arange(DIMS[0]), indexing="ij")[::-1], -1).reshape(-1, 3) * np.array(VS)
    vc = vc + VOL2CAM[1]
    u, v = K[0] * vc[:, 0] / vc[:, 2] + K[2], K[1] * vc[:, 1] / vc[:, 2] + K[3]
    inside = (u >= 20 + 1e-3) & (u < 40 - 1e-3) & (v >= 10 + 1e-3) & (v < 20 - 1e-3)
    outside = (u < 20 - 1e-3) | (u >= 40 + 1e-3) | (v < 10 - 1e-3) | (v >= 20 + 1e-3)
    assert lost[inside & (reg != 0)].all() and not lost[outside].any()


def test_colour_pixel_comes_from_the_colour_camera():
    """a camera shifted by 4 cm along x: every sample is the colour image's pixel at the voxel's colour projection"""
    cam = cco.Camera(COLS, ROWS, K, (np.eye(3, dtype=np.float32), np.array([-0.04, 0.0, 0.0], np.float32)))
    img = np.zeros((ROWS, COLS, 4), np.uint8)
    img[..., 0] = np.arange(COLS)[None, :]                              # B = column, G = row
    img[..., 1] = np.arange(ROWS)[:, None]
    cmap = constant_map(0.7, cam)
    out = camera_integrate(img, cmap, cam)
    got = out[out != 0]
    assert len(got) > 500
    idx = np.flatnonzero(out)
    z, rem = np.divmod(idx, DIMS[0] * DIMS[1])
    y, x = np.divmod(rem, DIMS[0])
    vc = np.stack([x, y, z], -1) * np.array(VS) + VOL2CAM[1]
    uc = K[0] * (vc[:, 0] - 0.04) / vc[:, 2] + K[2]
    vv = K[1] * vc[:, 1] / vc[:, 2] + K[3]
    col, row = (got >> 16) & 0xFF, (got >> 8) & 0xFF                   # the voxel word is R, G, B: B = column, G = row
    assert np.all(np.abs(col - uc) < 1.001) and np.all(np.abs(row - vv) < 1.001)
    ok = np.abs(uc - np.round(uc)) > 1e-3
    assert np.array_equal(col[ok], np.floor(uc[ok]).astype(np.uint32))


# ------------------------------------------------------------------------------------------------------------------------- snapshots
def _snapshot_camera(lib, capi, data):
    cam, present = capi.ColorCamera(), C.c_int(-1)
    buf = np.frombuffer(data, np.uint8)
    st = lib.df_kinfu_snapshot_color_camera(buf.ctypes.data, len(data), C.byref(cam), C.byref(present))
    return st, present.value, bytes(cam)


def test_snapshot_version_3_checks(lib):
    from dynamicfusion_b200 import capi
    from dynamicfusion_b200.kinfu import COLOR
    p1, p2 = sm.small_params(capi, lib, 0), sm.small_params(capi, lib, COLOR)
    dims = tuple(p2.volume_dims)
    length, cls, payload, rgba = sm.color_sections(dims)
    v2 = sm.v1_body(capi, lib, p2) + length + cls + payload + rgba
    cam = sm.camera_bytes(capi)
    v3 = v2 + cam
    snap = sm.header(v3, version=3) + v3
    st, out = sm.read_params(lib, capi, snap)
    assert st == 0 and bytes(out) == bytes(p2)
    assert _snapshot_camera(lib, capi, snap) == (0, 1, cam)
    assert _snapshot_camera(lib, capi, sm.header(v2, version=2) + v2) == (0, 0, bytes(72))   # version 2: no camera
    v1 = sm.v1_body(capi, lib, p1)
    assert _snapshot_camera(lib, capi, sm.header(v1) + v1) == (0, 0, bytes(72))

    def rejected(b, version=3):
        data = sm.header(b, version=version) + b
        return sm.read_params(lib, capi, data)[0] != 0 and _snapshot_camera(lib, capi, data)[0] != 0
    assert rejected(v3, version=2)                                      # the record is not a version-2 section
    assert rejected(v2, version=3)                                      # version 3 without its record
    assert rejected(v3[:-1]) and rejected(v3 + b"\0")                   # a record of the wrong length
    assert rejected(sm.v1_body(capi, lib, p1) + cam)                    # a colourless snapshot has no version 3
    assert rejected(v3, version=4)
    for bad in (sm.camera_bytes(capi, K_=(0.0, 1081.0, 959.5, 539.5)), sm.camera_bytes(capi, cols=0), sm.camera_bytes(capi, t=(float("nan"), 0, 0))):
        assert rejected(v2 + bad)                                       # the record obeys df_color_map_dims' rule
    corrupt = bytearray(snap); corrupt[-3] ^= 1                         # the checksum covers the record
    assert sm.read_params(lib, capi, bytes(corrupt))[0] != 0
    out_cam, present = capi.ColorCamera(), C.c_int()
    assert lib.df_kinfu_snapshot_color_camera(np.frombuffer(snap, np.uint8).ctypes.data, len(snap), None, C.byref(present)) == 0 and present.value == 1
    assert lib.df_kinfu_snapshot_color_camera(np.frombuffer(snap, np.uint8).ctypes.data, len(snap), C.byref(out_cam), None) != 0


def test_python_binding_reads_the_camera(lib):
    from dynamicfusion_b200 import capi
    from dynamicfusion_b200.kinfu import COLOR, KinFu
    p2 = sm.small_params(capi, lib, COLOR)
    length, cls, payload, rgba = sm.color_sections(tuple(p2.volume_dims))
    v2 = sm.v1_body(capi, lib, p2) + length + cls + payload + rgba
    v3 = v2 + sm.camera_bytes(capi)
    cam = KinFu.snapshot_color_camera(sm.header(v3, version=3) + v3)
    assert (cam.cols, cam.rows, cam.intr.fx, cam.depth_to_color.t[0]) == (1920, 1080, 1081.0, np.float32(0.052))
    assert KinFu.snapshot_color_camera(sm.header(v2, version=2) + v2) is None
    assert struct.unpack_from("<I", sm.header(v3, version=3), 8)[0] == 3


# ------------------------------------------------------------------------------------------------------------------------- synth
def test_synth_depth_camera_as_colour_camera_is_bit_identical():
    from dynamicfusion_b200 import synth
    for t in (0, 4, 9):
        d0, c0 = synth.umbrella_rgbd(t)
        d1, c1 = synth.umbrella_rgbd(t, color_camera=(synth.DEFAULT_K, 640, 480, IDENTITY))
        assert np.array_equal(d0, d1) and np.array_equal(c0, c1)


def test_synth_colour_camera_sees_from_its_own_centre():
    from dynamicfusion_b200 import synth
    Kc = (1081.37, 1081.37, 959.5, 539.5)
    d2c = (np.eye(3), np.array([-0.052, 0.0, 0.0]))                      # the colour camera 52 mm to the depth camera's +x
    d0, _ = synth.umbrella_rgbd(2)
    d1, c1 = synth.umbrella_rgbd(2, color_camera=(Kc, 1920, 1080, d2c))
    assert np.array_equal(d0, d1) and c1.shape == (1080, 1920, 4) and np.all(c1[..., 3] == 255)
    # the small sphere's constant colour appears where a ray from the colour centre meets it: project its centre
    R, t = synth.camera_drift(2)
    centre_cam = R.T @ (np.array([0.27, -0.17, 1.02]) - t)              # world -> depth camera
    pc = centre_cam + d2c[1]
    u, v = Kc[0] * pc[0] / pc[2] + Kc[2], Kc[1] * pc[1] / pc[2] + Kc[3]
    assert tuple(c1[int(v), int(u), 2::-1]) == synth.SPHERE_RGB
    # against a colour camera at the depth camera's centre the sphere moves by the parallax of 52 mm at its depth, to smaller u
    _, c2 = synth.umbrella_rgbd(2, color_camera=(Kc, 1920, 1080, IDENTITY))

    def sphere_u(img):
        return np.flatnonzero(np.all(img[..., 2::-1] == synth.SPHERE_RGB, -1).any(0)).mean()
    shift = Kc[0] * 0.052 / centre_cam[2]
    assert abs(sphere_u(c2) - sphere_u(c1) - shift) < 0.1 * shift
