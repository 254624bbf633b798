"""Lens distortion on the GPU: df_undistort and the three _lens colour-camera kernels equal tests/lens_oracle.c bit for bit; a NULL or zero
lens is today's entries bit for bit; the frame loop with a zero lens is the loop without one, with a depth lens it is one launch more and
can be rebuilt from the public entries; a lensed sequence tracks and colours as well as a pinhole one, and measurably worse without its
lens; version-4 snapshots resume and reject; the C++ mirror exports what Python does."""
import ctypes as C
import functools
import os
import struct
import subprocess
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import color_camera_oracle as cco  # noqa: E402
import lens_oracle as lo  # noqa: E402
from dynamicfusion_b200 import build, capi, kinfu as kf, synth  # noqa: E402
import gpu_util as gu  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]
I3 = np.eye(3, dtype=np.float32)
KV2_LENS = (0.09, -0.27, 0.0, 0.0, 0.09)                                # Kinect-v2-like barrel lens
STRONG_LENS = (0.6, -0.1, 0.012, -0.009, 0.02, 0.2, -0.05, 0.01)        # rational model with tangential terms
COLOR_LENS = (0.9, 0.25, 0.0, 0.0, 0.05)                                # a strong pincushion colour lens
K_WIDE = (460.0, 460.0, 320.0, 240.0)                                   # 640 x 480 with a Kinect-v2-class field of view
KV2_CAM = ((1081.37, 1081.37, 959.5, 539.5), 1920, 1080, (I3, np.array([-0.052, 0.0, 0.0], np.float32)))


def _lens(coeffs, K, cols, rows):
    return capi.make_lens(coeffs, None, K, cols, rows)


def _corner_shift(coeffs, K, cols, rows):
    """pixels the lens moves the image corners by"""
    x = np.array([-K[2], cols - 1 - K[2]]) / K[0]
    y = np.array([-K[3], rows - 1 - K[3]]) / K[1]
    xd, yd = synth.distort(x, y, coeffs)
    return float(np.min(np.hypot((xd - x) * K[0], (yd - y) * K[1])))


# ---------------------------------------------------------------------------------------------------------------- df_undistort
@pytest.mark.parametrize("name,K,cols,rows,coeffs,pad", [
    ("zero", synth.DEFAULT_K, 640, 480, (0.0,) * 5, 0),
    ("kinect_v2", K_WIDE, 640, 480, KV2_LENS, 0),
    ("strong", K_WIDE, 640, 480, STRONG_LENS, 3),
    ("ragged_203x151", (151.0, 149.0, 101.3, 74.8), 203, 151, STRONG_LENS, 5)])
def test_undistort_equals_the_oracle(name, K, cols, rows, coeffs, pad):
    lib = capi.load()
    rng = np.random.default_rng(3)
    lens = _lens(coeffs, K, cols, rows)
    if name == "kinect_v2":
        assert _corner_shift(coeffs, K, cols, rows) >= 5
    if name == "strong":
        assert _corner_shift(coeffs, K, cols, rows) >= 20
    for with_bgra in (False, True):
        depth = synth.sphere_wall_depth(cols, rows, K, seed=1)
        bgra = rng.integers(0, 256, (rows, cols, 4), np.uint8)
        d_dev, d_pitch, d_host = gu.padded(depth, pad, 7)
        b_dev, b_pitch, b_host = gu.padded(bgra, pad, 9)
        out = torch.full((rows, cols + pad + 1), 0x1234, dtype=torch.int16, device="cuda")
        bout = torch.full((rows, cols + pad + 2, 4), 77, dtype=torch.uint8, device="cuda")
        capi.check(lib.df_undistort(d_dev.data_ptr(), d_pitch, out.data_ptr(), (cols + pad + 1) * 2, b_dev.data_ptr() if with_bgra else None,
                                    b_pitch, bout.data_ptr() if with_bgra else None, (cols + pad + 2) * 4, cols, rows, capi.make_intr(*K), lens,
                                    gu.stream()))
        g = gu.host(out, np.uint16, (rows, cols + pad + 1))
        gb = bout.cpu().numpy()
        want, want_b = lo.undistort(d_host, K, lens, b_host if with_bgra else None)
        assert np.array_equal(g[:, :cols], want), (name, with_bgra)
        assert np.all(g[:, cols:] == 0x1234)                            # nothing past the row
        if with_bgra:
            assert np.array_equal(gb[:, :cols], want_b) and np.all(gb[:, cols:] == 77)
        else:
            assert np.all(gb == 77)
        if name == "zero":
            assert np.array_equal(g[:, :cols], depth) and (not with_bgra or np.array_equal(gb[:, :cols], bgra))
        else:
            assert (want != d_host).mean() > 0.05


def test_undistort_refusals_write_nothing():
    lib = capi.load()
    K, cols, rows = synth.DEFAULT_K, 64, 48
    depth = gu.dev(np.full((rows, cols), 1000, np.uint16))
    bgra = gu.dev(np.full((rows, cols, 4), 5, np.uint8))
    out = torch.full((rows, cols), 3, dtype=torch.int16, device="cuda")
    bout = torch.full((rows, cols, 4), 3, dtype=torch.uint8, device="cuda")
    good = _lens(KV2_LENS, K, cols, rows)
    intr = capi.make_intr(*K)

    def call(lens=good, dpitch=cols * 2, opitch=cols * 2, src=depth, dst=out, b=bgra, bo=bout, bpitch=cols * 4):
        return lib.df_undistort(src.data_ptr(), dpitch, dst.data_ptr(), opitch, None if b is None else b.data_ptr(), bpitch,
                                None if bo is None else bo.data_ptr(), cols * 4, cols, rows, intr, lens, gu.stream())
    assert call(lens=capi.make_lens((-0.5, 0, 0, 0, 0), 1.0)) != 0      # a folding lens
    assert call(lens=capi.make_lens(KV2_LENS, 0.0)) != 0                 # r2_max not > 0
    assert call(dpitch=cols * 2 - 2) != 0 and call(opitch=cols * 2 + 1) != 0 and call(bpitch=cols * 4 + 2) != 0
    assert call(dst=depth) != 0                                          # in place
    assert call(bo=None) != 0                                            # bgra without its output
    assert call(bo=bgra) != 0                                            # colour in place
    torch.cuda.synchronize()
    assert (out == 3).all() and (bout == 3).all() and (gu.host(depth, np.uint16, (rows, cols)) == 1000).all()
    assert call() == 0


# ------------------------------------------------------------------------------------------------- the three colour-camera kernels
BIG = ((1081.37, 1081.37, 959.5, 539.5), 1920, 1080)
SMALL = ((285.171, 285.171, 159.5, 119.5), 320, 240)
D2C = (np.array([[0.99966, 0.0, 0.02618], [0.0, 1.0, 0.0], [-0.02618, 0.0, 0.99966]], np.float32), np.array([-0.05, 0.004, 0.002], np.float32))


@pytest.mark.parametrize("name,cols,rows,camera,coeffs,pad,cpad", [
    ("big_own_lens", 640, 480, BIG, COLOR_LENS, 0, 0),
    ("small_kinect_v2", 640, 480, SMALL, KV2_LENS, 0, 4),
    ("small_strong", 640, 480, SMALL, STRONG_LENS, 2, 0),
    ("small_zero", 640, 480, SMALL, (0.0,) * 8, 0, 0),
    ("ragged_203x151", 203, 151, ((120.0, 131.0, 104.5, 47.0), 211, 97), STRONG_LENS, 5, 3)])
def test_colour_kernels_equal_the_oracle(name, cols, rows, camera, coeffs, pad, cpad):
    lib = capi.load()
    rng = np.random.default_rng(11)
    K = synth.scaled_K(cols, rows) if cols != 640 else synth.DEFAULT_K
    cam = cco.Camera(camera[1], camera[2], camera[0], D2C)
    cs = capi.make_color_camera(cam.K, cam.cols, cam.rows, cam.d2c)
    lens = _lens(coeffs, cam.K, cam.cols, cam.rows)
    dims, size = (64, 64, 64), 3.0
    nvox = int(np.prod(dims))
    vs = tuple(size / d for d in dims)
    trunc = max(0.04, 2.1 * max(vs))
    intr = capi.make_intr(*K)
    vol2cam = (I3, np.array([-size / 2, -size / 2, 0.5], np.float32))
    tsdf = torch.zeros(nvox, dtype=torch.int32, device="cuda")
    V = capi.make_volume(tsdf.data_ptr(), dims, vs, trunc, 64)
    act = torch.zeros(lib.df_volume_activity_bytes(V), dtype=torch.uint8, device="cuda")
    mc, mr, _ = cco.map_dims(K, cam)
    g_lens, g_null, g_base = (torch.zeros(nvox, dtype=torch.int32, device="cuda") for _ in range(3))
    o_lens = np.zeros(nvox, np.uint32)
    for t in range(3):
        depth = synth.sphere_wall_depth(cols, rows, K, seed=t)
        d_dev, d_pitch, d_host = gu.padded(depth, pad, 7)
        dists = torch.zeros((rows, cols + pad), dtype=torch.int16, device="cuda")
        capi.check(lib.df_compute_dists(d_dev.data_ptr(), d_pitch, cols, rows, intr, dists.data_ptr(), (cols + pad) * 2, gu.stream()))
        capi.check(lib.df_integrate_tracked(V, dists.data_ptr(), (cols + pad) * 2, cols, rows, capi.make_aff(*vol2cam), intr, None,
                                            act.data_ptr(), None, gu.stream()))
        maps = {}
        for key, lp in (("lens", C.byref(lens)), ("null", None), ("base", "base")):
            m = torch.full((mr, mc + cpad), 0x5a5a5a5a, dtype=torch.int32, device="cuda")
            if lp == "base":
                capi.check(lib.df_color_depth_map(d_dev.data_ptr(), d_pitch, cols, rows, intr, cs, m.data_ptr(), (mc + cpad) * 4, gu.stream()))
            else:
                capi.check(lib.df_color_depth_map_lens(d_dev.data_ptr(), d_pitch, cols, rows, intr, cs, lp, m.data_ptr(), (mc + cpad) * 4,
                                                       gu.stream()))
            maps[key] = m
        gmap = gu.host(maps["lens"], np.uint32, (mr, mc + cpad))
        assert np.all(gmap[:, mc:] == 0x5a5a5a5a)
        omap = lo.depth_map(d_host, K, cam, lens)
        assert np.array_equal(gmap[:, :mc], omap), (name, t)
        assert np.array_equal(gu.host(maps["null"], np.uint32, (mr, mc + cpad)), gu.host(maps["base"], np.uint32, (mr, mc + cpad)))
        if name.endswith("zero"):
            assert np.array_equal(gmap, gu.host(maps["base"], np.uint32, (mr, mc + cpad)))
        img = rng.integers(0, 256, (cam.rows, cam.cols, 4), np.uint8)
        i_dev, i_pitch, i_host = gu.padded(img, cpad, 99)
        capi.check(lib.df_integrate_color_camera_lens(V, g_lens.data_ptr(), dists.data_ptr(), (cols + pad) * 2, cols, rows, capi.make_aff(*vol2cam),
                                                      intr, cs, C.byref(lens), i_dev.data_ptr(), i_pitch, maps["lens"].data_ptr(), (mc + cpad) * 4,
                                                      act.data_ptr(), gu.stream()))
        capi.check(lib.df_integrate_color_camera_lens(V, g_null.data_ptr(), dists.data_ptr(), (cols + pad) * 2, cols, rows, capi.make_aff(*vol2cam),
                                                      intr, cs, None, i_dev.data_ptr(), i_pitch, maps["base"].data_ptr(), (mc + cpad) * 4,
                                                      act.data_ptr(), gu.stream()))
        capi.check(lib.df_integrate_color_camera(V, g_base.data_ptr(), dists.data_ptr(), (cols + pad) * 2, cols, rows, capi.make_aff(*vol2cam),
                                                 intr, cs, i_dev.data_ptr(), i_pitch, maps["base"].data_ptr(), (mc + cpad) * 4, act.data_ptr(),
                                                 gu.stream()))
        assert np.array_equal(g_null.cpu().numpy(), g_base.cpu().numpy()), (name, t)   # a NULL lens is the entry without _lens
        dists_host = dists.cpu().numpy().view(np.uint16)[:, :cols]
        lo.integrate_color_camera(o_lens, dims, vs, trunc, 64, dists_host, vol2cam, K, cam, lens, i_host, omap, act.cpu().numpy())
        assert np.array_equal(g_lens.cpu().numpy().view(np.uint32), o_lens), (name, t)
        # frame intensity, level 0, from the frame's vertex map
        pts = torch.zeros((rows, cols, 4), dtype=torch.float32, device="cuda")
        nrm = torch.zeros_like(pts)
        capi.check(lib.df_points_normals(intr, d_dev.data_ptr(), d_pitch, cols, rows, pts.data_ptr(), cols * 16, nrm.data_ptr(), cols * 16,
                                         gu.stream()))
        outs = {}
        for key, lp in (("lens", C.byref(lens)), ("null", None)):
            o = torch.full((rows, cols), 7.0, dtype=torch.float32, device="cuda")
            arr = lambda v, t_: (t_ * 1)(v)  # noqa: E731
            capi.check(lib.df_frame_intensity_lens(i_dev.data_ptr(), i_pitch, C.byref(cs), lp, intr, pts.data_ptr(), cols * 16,
                                                   maps[key if key == "lens" else "base"].data_ptr(), (mc + cpad) * 4, trunc, 1, arr(cols, C.c_int),
                                                   arr(rows, C.c_int), arr(o.data_ptr(), C.c_void_p), arr(cols * 4, C.c_size_t), gu.stream()))
            outs[key] = o.cpu().numpy()
        base = torch.full((rows, cols), 7.0, dtype=torch.float32, device="cuda")
        capi.check(lib.df_frame_intensity(i_dev.data_ptr(), i_pitch, C.byref(cs), intr, pts.data_ptr(), cols * 16, maps["base"].data_ptr(),
                                          (mc + cpad) * 4, trunc, 1, (C.c_int * 1)(cols), (C.c_int * 1)(rows), (C.c_void_p * 1)(base.data_ptr()),
                                          (C.c_size_t * 1)(cols * 4), gu.stream()))
        want = lo.frame_intensity(i_host, K, cam, lens, omap, trunc, pts.cpu().numpy())
        assert gu.same_bits(outs["lens"], want), (name, t)                 # the device's NaN has other payload bits than C's
        assert np.array_equal(outs["null"].view(np.uint32), base.cpu().numpy().view(np.uint32))
        assert (~np.isnan(want)).mean() > 0.05
    w = g_lens.cpu().numpy().view(np.uint32) >> 24
    assert w.max() >= 1 and (w > 0).sum() > 100
    if name.endswith("zero"):
        assert np.array_equal(g_lens.cpu().numpy(), g_null.cpu().numpy())
    else:
        assert not np.array_equal(g_lens.cpu().numpy(), g_null.cpu().numpy())


def test_colour_kernels_refuse_an_invalid_lens():
    lib = capi.load()
    K, cols, rows = synth.DEFAULT_K, 64, 48
    cam = cco.Camera(*SMALL[1:], SMALL[0], D2C)
    cs = capi.make_color_camera(cam.K, cam.cols, cam.rows, cam.d2c)
    mc, mr, _ = cco.map_dims(K, cam)
    intr = capi.make_intr(*K)
    depth = gu.dev(np.full((rows, cols), 1000, np.uint16))
    m = torch.full((mr, mc), 5, dtype=torch.int32, device="cuda")
    dims = (32, 32, 32)
    colours = torch.full((32 ** 3,), 9, dtype=torch.int32, device="cuda")
    V = capi.make_volume(colours.data_ptr(), dims, (3.0 / 32,) * 3, 0.2, 64)
    dists = gu.dev(np.full((rows, cols), 0x3c00, np.uint16))               # fp16 1.0 everywhere
    img = gu.dev(np.full((cam.rows, cam.cols, 4), 200, np.uint8))
    pts = gu.dev(np.tile(np.array([0.0, 0.0, 1.0, 1.0], np.float32), (rows, cols, 1)))
    inten = torch.full((rows, cols), 7.0, dtype=torch.float32, device="cuda")
    vol2cam = capi.make_aff(I3, np.array([-1.5, -1.5, 0.5], np.float32))
    for bad in (capi.make_lens((-0.5, 0, 0, 0, 0), 1.0), capi.make_lens((0,) * 5, 0.0), capi.make_lens((float("nan"), 0, 0, 0, 0), 1.0)):
        assert lib.df_color_depth_map_lens(depth.data_ptr(), cols * 2, cols, rows, intr, cs, C.byref(bad), m.data_ptr(), mc * 4, gu.stream()) != 0
        assert lib.df_integrate_color_camera_lens(V, colours.data_ptr(), dists.data_ptr(), cols * 2, cols, rows, vol2cam, intr, cs, C.byref(bad),
                                                  img.data_ptr(), cam.cols * 4, m.data_ptr(), mc * 4, None, gu.stream()) != 0
        assert lib.df_frame_intensity_lens(img.data_ptr(), cam.cols * 4, C.byref(cs), C.byref(bad), intr, pts.data_ptr(), cols * 16, m.data_ptr(),
                                           mc * 4, 0.2, 1, (C.c_int * 1)(cols), (C.c_int * 1)(rows), (C.c_void_p * 1)(inten.data_ptr()),
                                           (C.c_size_t * 1)(cols * 4), gu.stream()) != 0
    torch.cuda.synchronize()
    assert (m == 5).all() and (colours == 9).all() and (inten == 7.0).all()


# ----------------------------------------------------------------------------------------------------------------------- the frame loop
@functools.lru_cache(maxsize=None)
def _lensed(t, camera=False):
    return synth.umbrella_rgbd(t, lens=KV2_LENS, color_camera=KV2_CAM + (COLOR_LENS,) if camera else None)


@pytest.mark.parametrize("flags,camera", [(0, False), (kf.COLOR, True)], ids=["default", "color_camera"])
def test_zero_lens_is_no_lens(flags, camera):
    objs = [kf.KinFu(gu.kinfu_params(128, flags, max_nodes=1024, cloud_capacity=1_000_000)) for _ in range(2)]
    zero = (0.0,) * 8
    if camera:
        objs[0].set_color_camera(*KV2_CAM)
        objs[1].set_color_camera(*KV2_CAM, lens=capi.make_lens(zero, 0.7))
    objs[1].set_depth_lens(capi.make_lens(zero, 0.5))
    assert objs[1].depth_lens is not None
    for t in range(6):
        depth, bgra = synth.umbrella_rgbd(t, color_camera=KV2_CAM if camera else None)
        for k in objs:
            k(depth, bgra) if flags & kf.COLOR else k(depth)
        assert gu.state(objs[0]) == gu.state(objs[1]) and objs[0].info() == objs[1].info()
        if camera:
            assert np.array_equal(objs[0].buffer("color_volume"), objs[1].buffer("color_volume"))
    assert objs[0].snapshot() == objs[1].snapshot()                     # a zero lens writes no version-4 section
    for k in objs:
        k.close()


def _undistort_on_device(k, depth, bgra):
    """the frame as the object with a depth lens sees it, from df_undistort: device (depth, bgra or None)"""
    p = k.params
    d, out = gu.dev(depth), torch.zeros((p.rows, p.cols), dtype=torch.int16, device="cuda")
    b = bout = None
    if bgra is not None and bgra.shape[:2] == depth.shape:
        b, bout = gu.dev(bgra), torch.zeros((p.rows, p.cols, 4), dtype=torch.uint8, device="cuda")
    capi.check(k.lib.df_undistort(d.data_ptr(), p.cols * 2, out.data_ptr(), p.cols * 2, None if b is None else b.data_ptr(), p.cols * 4,
                                  None if bout is None else bout.data_ptr(), p.cols * 4, p.cols, p.rows, p.intr, k.depth_lens, gu.stream()))
    torch.cuda.synchronize()
    return out, (bout if bout is not None else (None if bgra is None else gu.dev(bgra)))


@pytest.mark.parametrize("overlap", ["1", "0"])
@pytest.mark.parametrize("camera", [False, True], ids=["registered", "color_camera"])
def test_loop_rebuilt_from_the_public_entries(monkeypatch, overlap, camera):
    """an object with a depth lens fed raw frames equals one without, fed df_undistort's output of the same frames"""
    monkeypatch.setenv("DF_KINFU_OVERLAP_EXTRACT", overlap)
    lensed, plain = (kf.KinFu(gu.kinfu_params(128, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000)) for _ in range(2))
    lensed.set_depth_lens(KV2_LENS)
    if camera:
        for k in (lensed, plain):
            k.set_color_camera(*KV2_CAM, lens=COLOR_LENS)
    for t in range(6):
        depth, bgra = _lensed(t, camera)
        lensed(gu.dev(depth), gu.dev(bgra))                              # device frames: the caller's buffers are never written
        d, b = _undistort_on_device(lensed, depth, bgra)
        plain(d, b)
        assert gu.state(lensed) == gu.state(plain)
        assert lensed.info()["launches"] == plain.info()["launches"] + 1
        assert np.array_equal(lensed.buffer("color_volume"), plain.buffer("color_volume"))
        assert np.array_equal(lensed.buffer("cloud_colors"), plain.buffer("cloud_colors"))
    assert (lensed.buffer("color_volume") >> 24).max() == 6
    lensed.reset()                                                       # a reset keeps the lens
    depth, bgra = _lensed(0, camera)
    lensed(depth, bgra)
    assert lensed.info()["launches"] > 0 and lensed.depth_lens is not None
    lensed.close(); plain.close()


def test_caller_frames_are_not_written():
    k = kf.KinFu(gu.kinfu_params(128, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000))
    k.set_depth_lens(KV2_LENS)
    depth, bgra = _lensed(0)
    d, b = gu.dev(depth), gu.dev(bgra)
    k(d, b)
    torch.cuda.synchronize()
    assert np.array_equal(gu.host(d, np.uint16, depth.shape), depth) and np.array_equal(b.cpu().numpy(), bgra)
    k.close()


def test_setters_follow_the_colour_camera_rules():
    k = kf.KinFu(gu.kinfu_params(128, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000))
    with pytest.raises(RuntimeError):
        k.set_depth_lens(capi.make_lens((-0.5, 0, 0, 0, 0), 1.0))      # invalid: nothing changes
    assert k.depth_lens is None
    with pytest.raises(RuntimeError):
        capi.check(k.lib.df_kinfu_set_color_lens(k.h, C.byref(capi.make_lens(KV2_LENS, 1.0))))   # no colour camera
    k.set_color_camera(*KV2_CAM, lens=COLOR_LENS)
    with pytest.raises(RuntimeError):
        k.set_color_camera(*KV2_CAM, lens=(-0.5, 0, 0, 0, 0, 0, 0, 0))  # a lens that folds inside the image: the camera stays as it was
    assert k.color_lens is not None
    depth, bgra = _lensed(0, True)
    k(depth, bgra)
    before = k.state_digest()
    for call in (lambda: k.set_depth_lens(KV2_LENS), lambda: k.set_depth_lens(None),
                 lambda: capi.check(k.lib.df_kinfu_set_color_lens(k.h, None))):
        with pytest.raises(RuntimeError):
            call()                                                       # the sequence is running
    assert k.state_digest() == before
    k.reset()
    k.set_depth_lens(None)
    k.set_color_camera(*KV2_CAM[:3], KV2_CAM[3])                         # a new camera drops the colour lens
    assert k.color_lens is None
    plain = kf.KinFu(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=1_000_000))
    plain.set_depth_lens(KV2_LENS)                                       # a depth lens on any object
    plain(_lensed(0)[0])
    assert plain.info()["frame_counter"] == 1
    k.close(); plain.close()


@pytest.mark.parametrize("lens_first", [True, False], ids=["lens_then_camera", "camera_then_lens"])
def test_registered_images_after_a_camera_is_removed(lens_first):
    """the registered image's buffer follows the camera: a depth lens set before or after a colour camera, then the camera removed, undistorts
    registered images as an object that never had a camera does"""
    k, ref = (kf.KinFu(gu.kinfu_params(128, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000)) for _ in range(2))
    ref.set_depth_lens(KV2_LENS)
    if lens_first:
        k.set_depth_lens(KV2_LENS)
    k.set_color_camera(*KV2_CAM, lens=COLOR_LENS)
    if not lens_first:
        k.set_depth_lens(KV2_LENS)
    with pytest.raises(ValueError):
        k.set_color_camera(None, lens=COLOR_LENS)                          # a colour lens without a colour camera
    assert k.color_camera is not None and k.color_lens is not None
    k.set_color_camera(None)
    for t in range(4):
        depth, bgra = _lensed(t)
        k(depth, bgra)
        ref(depth, bgra)
        assert gu.state(k) == gu.state(ref) and k.info()["launches"] == ref.info()["launches"]
        assert np.array_equal(k.buffer("color_volume"), ref.buffer("color_volume"))
    k.close(); ref.close()


@pytest.mark.parametrize("flags", [kf.LIVE_MODEL, kf.COLOR | kf.COLOR_TRACKING, kf.USE_DEPTH, kf.EXTEND_FIELD, kf.F2_SOLVE,
                                   kf.WARPED_INTEGRATE],
                         ids=["live_model", "color_tracking", "use_depth", "extend_field", "f2_solve", "warped_integrate"])
def test_flags_run_with_a_depth_lens(flags):
    k = kf.KinFu(gu.kinfu_params(128, flags, max_nodes=1024, cloud_capacity=1_000_000))
    k.set_depth_lens(KV2_LENS)
    for t in range(5):
        depth, bgra = _lensed(t)
        k(depth, bgra) if flags & kf.COLOR else k(depth)
        assert k.info()["icp_ok"] == 1
    assert k.info()["frame_counter"] == 5 and k.info()["resets"] == 0
    k.close()


# --------------------------------------------------------------------------------------------------------------------------- fidelity
def _pose_errors(k, n):
    """per frame: (translation error in mm, rotation error in degrees) of the tracked pose against the synthetic camera"""
    out = []
    for t in range(n):
        R, tr = k.getCameraPose(t)
        Rt, tt = synth.camera_drift(t)
        dR = R.astype(np.float64) @ Rt.T
        ang = np.degrees(np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1)))
        out.append((1000 * np.linalg.norm(tr - tt), ang))
    return np.array(out)


def _vertex_errors(k, K, t):
    """mm between the loop's level-0 vertex map of the last frame (the previous frame's map after it) and the true scene points on the
    same pixels' rays (noise-free pinhole rendering), at valid pixels away from depth edges: (median, 95th percentile)"""
    rows, cols = 480, 640
    truth = synth.umbrella_depth(t, cols, rows, K, noise_mm=0, dropout=0, shape_t=0).astype(np.float64) / 1000
    p = np.pad(truth, 1, mode="edge")
    win = np.stack([p[i:i + rows, j:j + cols] for i in range(3) for j in range(3)])
    keep = (truth > 0) & (win.max(0) - win.min(0) <= 0.01)
    xl, yl = synth._rays(cols, rows, K)
    want = np.stack([xl * truth, yl * truth, truth], -1)
    got = k.buffer("prev_points")[..., :3].astype(np.float64)
    ok = keep & np.isfinite(got).all(-1)
    err = 1000 * np.linalg.norm(got[ok] - want[ok], axis=-1)
    return float(np.median(err)), float(np.percentile(err, 95)), float(ok.mean())


def test_tracking_fidelity_rigid_c2_256():
    n = 20
    runs, frame0 = {}, {}
    for name, lens_frames, lens_set in (("pinhole", None, False), ("lens", KV2_LENS, True), ("lens_ignored", KV2_LENS, False)):
        k = kf.KinFu(gu.kinfu_params(256, kf.RIGID_ONLY, max_nodes=1024, cloud_capacity=2_000_000, size=3.0, K=K_WIDE))
        if lens_set:
            k.set_depth_lens(KV2_LENS)
        for t in range(n):
            k(synth.umbrella_depth(t, K=K_WIDE, shape_t=0, lens=lens_frames))
            if t == 0:
                frame0[name] = _vertex_errors(k, K_WIDE, 0)
        assert k.info()["frame_counter"] == n and k.info()["resets"] == 0, name
        runs[name] = _pose_errors(k, n)
        k.close()
    lines = [f"{name}: max translation error {e[:, 0].max():.3f} mm, mean over frames 2.. {e[2:, 0].mean():.3f} mm, max rotation error "
             f"{e[:, 1].max():.4f} deg; frame 0 vertex error median {frame0[name][0]:.2f} mm, p95 {frame0[name][1]:.2f} mm over "
             f"{frame0[name][2]:.3f} of the pixels; per frame mm " + " ".join(f"{v:.2f}" for v in e[:, 0]) + " deg "
             + " ".join(f"{v:.3f}" for v in e[:, 1]) for name, e in runs.items()]
    print("\n".join(lines))
    out = os.environ.get("DF_LENS_FIDELITY_OUT")
    if out:
        Path(out).write_text("\n".join(lines) + "\n")
    # The 3 m volume holds the whole image, corners included, where the lens moves pixels by about 19 px; a volume that holds only the
    # middle of the image cannot tell a loop that applies the lens from one that ignores it.  Bars, set from the first run of this
    # configuration (NVIDIA H100 80GB HBM3, 700 W):
    # - the lensed run, undistorted, tracks within TRACK_BAR_MM / TRACK_BAR_DEG of the pinhole run's error at every frame (measured: at most
    #   0.26 mm and 0.04 degrees more);
    # - the same frames taken as pinhole frames track worse: max rotation error 0.647 degrees against 0.297 (pinhole 0.362), mean
    #   translation error over frames 2..19 1.38 mm against 1.05 (pinhole 1.05); bars IGNORED_WORSE_DEG / IGNORED_WORSE_MM;
    # - the frame's own geometry: the 95th percentile of the level-0 vertex map's distance to the true scene points, measured 1.02 mm
    #   pinhole, 1.09 mm through the lens undistorted, 2.47 mm with the lens ignored; bars VERTEX_BAR_MM / IGNORED_VERTEX_MM.
    dt = runs["lens"] - runs["pinhole"]
    assert (dt[:, 0] <= TRACK_BAR_MM).all() and (dt[:, 1] <= TRACK_BAR_DEG).all(), dt
    assert runs["lens_ignored"][:, 1].max() >= runs["lens"][:, 1].max() + IGNORED_WORSE_DEG, runs
    assert runs["lens_ignored"][2:, 0].mean() >= runs["lens"][2:, 0].mean() + IGNORED_WORSE_MM, runs
    assert frame0["lens"][1] <= frame0["pinhole"][1] + VERTEX_BAR_MM, frame0
    assert frame0["lens_ignored"][1] >= frame0["lens"][1] + IGNORED_VERTEX_MM, frame0


TRACK_BAR_MM, TRACK_BAR_DEG = 0.5, 0.1
IGNORED_WORSE_DEG, IGNORED_WORSE_MM = 0.2, 0.15
VERTEX_BAR_MM, IGNORED_VERTEX_MM = 0.2, 1.0


def _texture_stats(k):
    verts, _, _ = k.mesh()
    rgba = k.mesh_colors()
    r2 = verts[:, 0] ** 2 + verts[:, 1] ** 2
    cap = (r2 < 0.25 ** 2) & (np.abs(verts[:, 2] - (0.9 + 0.6 * r2)) < 0.05)
    coloured = rgba[:, 3] == 255
    err = np.abs(rgba[cap & coloured][:, :3].astype(int) - synth.umbrella_texture(verts[cap & coloured]).astype(int))
    return int(cap.sum()), float(coloured[cap].mean()), float(np.median(err)), float(np.percentile(err, 90))


def test_texture_fidelity_through_a_lensed_colour_camera():
    stats = {}
    frames = [synth.umbrella_rgbd(t, color_camera=KV2_CAM + (COLOR_LENS,)) for t in range(20)]
    for name, lens in (("lens", COLOR_LENS), ("lens_ignored", None)):
        k = kf.KinFu(gu.kinfu_params(256, kf.COLOR, max_nodes=1024, cloud_capacity=2_000_000))
        k.set_color_camera(*KV2_CAM, lens=lens)
        for f in frames:
            k(*f)
        stats[name] = _texture_stats(k)
        k.close()
    line = "; ".join(f"{n}: cap vertices {s[0]} coloured {s[1]:.4f} median {s[2]:.1f} p90 {s[3]:.1f}" for n, s in stats.items())
    print(line)
    out = os.environ.get("DF_LENS_TEXTURE_OUT")
    if out:
        Path(out).write_text(line + "\n")
    # test_color_camera_gpu.py's pinhole camera on the same scene measured median 13 and 90th percentile 52 (all cap vertices coloured);
    # the lensed camera keeps those within TEXTURE_MARGIN levels.  Set from the first run (NVIDIA H100 80GB HBM3, 700 W): through the lens
    # 13 and 52, 99.98 % coloured; the same images taken as pinhole images 15 and 58
    n, frac, med, p90 = stats["lens"]
    assert n > 5000 and frac > 0.9 and med <= 13 + TEXTURE_MARGIN[0] and p90 <= 52 + TEXTURE_MARGIN[1], stats
    _, frac, med, p90 = stats["lens_ignored"]
    assert med > 13 + TEXTURE_MARGIN[0] or p90 > 52 + TEXTURE_MARGIN[1], stats


TEXTURE_MARGIN = (1, 3)                                                 # median, 90th percentile


# -------------------------------------------------------------------------------------------------------------------------- snapshots
def test_version_4_resumes_and_rejects(tmp_path, capfd):
    frames = [_lensed(t, True) for t in range(7)]

    def make(depth_lens=KV2_LENS, color_lens=COLOR_LENS):
        k = kf.KinFu(gu.kinfu_params(64, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000))
        k.set_color_camera(*KV2_CAM, lens=color_lens)
        if depth_lens is not None:
            k.set_depth_lens(depth_lens)
        return k
    ref = make()
    want, snap = [], None
    for i, f in enumerate(frames):
        ref(*f)
        want.append((ref.state_digest(), ref.buffer("color_volume").tobytes(), ref.buffer("cloud_colors").tobytes()))
        if i == 3:
            snap = ref.snapshot()
    assert struct.unpack_from("<I", snap, 8)[0] == 4
    d, c = kf.KinFu.snapshot_lenses(snap)
    assert bytes(d) == bytes(ref.depth_lens) and bytes(c) == bytes(ref.color_lens)
    ref.close()
    d0, c0 = frames[0]
    for obj in (make(depth_lens=None), make(depth_lens=(0.08, -0.27, 0.0, 0.0, 0.09)), make(color_lens=None)):
        obj(d0, c0)
        before = (obj.state_digest(), obj.buffer("color_volume").tobytes())
        with pytest.raises(RuntimeError):
            obj.restore(snap)
        assert (obj.state_digest(), obj.buffer("color_volume").tobytes()) == before
        obj.close()
    assert "lenses differ" in capfd.readouterr().err
    path = tmp_path / "v4.dfsnap"
    path.write_bytes(snap)
    k = kf.KinFu.from_snapshot(path)
    assert k.depth_lens is not None and k.color_lens is not None and k.color_camera is not None
    assert (k.state_digest(), k.buffer("color_volume").tobytes(), k.buffer("cloud_colors").tobytes()) == want[3]
    for i in range(4, 7):
        k(*frames[i])
        assert (k.state_digest(), k.buffer("color_volume").tobytes(), k.buffer("cloud_colors").tobytes()) == want[i]
    assert k.snapshot()[8:12] == struct.pack("<I", 4)
    k.close()


# ---------------------------------------------------------------------------------------------------------------------------- hosts
def test_cpp_mirror_exports_the_same_colours(tmp_path):
    exe = build.build_cpp_program(ROOT / "tests" / "cpp" / "lens_export.cpp", ROOT / "tests" / "cpp" / "_build" / "lens_export")
    frames = [_lensed(t, True) for t in range(5)]
    np.stack([d for d, _ in frames]).tofile(tmp_path / "depth.u16")
    np.stack([c for _, c in frames]).tofile(tmp_path / "bgra.u8")
    K, cols, rows, (R, t) = KV2_CAM
    coeffs = [list(L) + [0.0] * (8 - len(L)) for L in (KV2_LENS, COLOR_LENS)]
    nums = [repr(float(np.float32(x))) for x in list(K) + list(np.asarray(R).reshape(9)) + list(t) + coeffs[0] + coeffs[1]]
    r = subprocess.run([str(exe), str(tmp_path / "depth.u16"), str(tmp_path / "bgra.u8"), str(len(frames)), str(cols), str(rows), *nums,
                        str(tmp_path / "cpp.ply"), str(tmp_path / "cpp.bgra")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    p = kf.KinFuParams.default_params_dynamicfusion()
    p.flags = kf.COLOR
    k = kf.KinFu(p)
    k.set_depth_lens(KV2_LENS)
    k.set_color_camera(*KV2_CAM, lens=COLOR_LENS)
    for depth, bgra in frames:
        k(depth, bgra)
    k.save_mesh(tmp_path / "py.ply", live=True, colors=True)
    img = k.render_image(live=True, flag=4)
    k.close()
    assert (tmp_path / "cpp.ply").read_bytes() == (tmp_path / "py.ply").read_bytes()
    assert (tmp_path / "cpp.bgra").read_bytes() == img.tobytes()
