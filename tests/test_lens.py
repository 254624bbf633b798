"""CPU checks of lens distortion (df_lens): the oracle's distortion against a float64 statement of the OpenCV model, df_lens_check's rules,
df_undistort's rule (tests/lens_oracle.c) as the identity for the zero lens and as the inverse of synth's lens rendering on the C2 scene,
synth's lens inversion, and the version-4 snapshot checks of df_kinfu_snapshot_params / df_kinfu_snapshot_lenses (host code)."""
import ctypes as C

import numpy as np
import pytest

import color_camera_oracle as cco
import lens_oracle as lo
import snapshot_model as sm
from snapshot_model import lib  # noqa: F401  (a fixture)

KV2_LENS = (0.09, -0.27, 0.0, 0.0, 0.09)                     # Kinect-v2-like barrel lens (k1, k2, p1, p2, k3)
STRONG_LENS = (0.6, -0.1, 0.012, -0.009, 0.02, 0.2, -0.05, 0.01)   # eight-coefficient rational model with tangential terms
KV2_DEPTH = ((365.0, 365.0, 256.0, 212.0), 512, 424)          # a Kinect-v2-class depth camera: K, cols, rows


def _np_distort(x, y, c):
    """the OpenCV model in float64"""
    k1, k2, p1, p2, k3, k4, k5, k6 = list(c) + [0.0] * (8 - len(c))
    r2 = x * x + y * y
    radial = (1 + k1 * r2 + k2 * r2 ** 2 + k3 * r2 ** 3) / (1 + k4 * r2 + k5 * r2 ** 2 + k6 * r2 ** 3)
    return x * radial + 2 * p1 * x * y + p2 * (r2 + 2 * x * x), y * radial + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y


@pytest.mark.parametrize("coeffs", [KV2_LENS, STRONG_LENS])
def test_oracle_distortion_is_the_opencv_model(coeffs):
    rng = np.random.default_rng(5)
    r2_max = 1.2
    r = np.sqrt(rng.uniform(0, r2_max, 4000)) * 0.999
    a = rng.uniform(0, 2 * np.pi, r.size)
    x, y = (r * np.cos(a)).astype(np.float32), (r * np.sin(a)).astype(np.float32)
    c8 = np.array(list(coeffs) + [0.0] * (8 - len(coeffs)), np.float32)
    xd, yd, ok = lo.distort(x, y, list(c8) + [r2_max])
    assert ok.all()
    ex, ey = _np_distort(x.astype(np.float64), y.astype(np.float64), c8.astype(np.float64))
    # a few dozen float roundings of values of order 1
    assert np.abs(xd - ex).max() < 2e-6 and np.abs(yd - ey).max() < 2e-6
    # outside the calibrated radius, and NaN, are invalid
    _, _, ok = lo.distort(np.array([1.2, np.nan], np.float32), np.array([0.2, 0.0], np.float32), list(c8) + [r2_max])
    assert not ok.any()


def test_lens_check_rules(lib):
    from dynamicfusion_b200 import capi
    ok = lambda coeffs, r2: lib.df_lens_check(capi.make_lens(coeffs, r2)) == 0   # noqa: E731
    assert ok(KV2_LENS, 1.0) and ok(STRONG_LENS, 1.5) and ok((0,) * 5, 0.3) and ok((0,) * 8, 1e6)
    assert not ok((-0.5, 0, 0, 0, 0), 1.0)                          # r (1 - r^2 / 2) folds back at r^2 = 2/3
    assert ok((-0.5, 0, 0, 0, 0), 0.6)                              # and is monotonic below
    assert not ok((0, 0, 0, 0, 0, -1.0, 0, 0), 2.0)                 # 1 - r^2 vanishes at r^2 = 1
    assert not ok((0, 0, 0, 0, 0, -1.0, 0, 0), 1.0)                 # at the end of the range too
    assert ok((0, 0, 0, 0, 0, -1.0, 0, 0), 0.9)
    for bad in (float("nan"), float("inf")):
        assert not ok((bad, 0, 0, 0, 0), 1.0) and not ok((0, 0, 0, 0, 0, 0, 0, bad), 1.0) and not ok((0,) * 5, bad)
    assert not ok((0,) * 5, 0.0) and not ok((0,) * 5, -1.0) and not ok(KV2_LENS, 0.0)
    with pytest.raises(ValueError):
        capi.make_lens((0.1, 0.2, 0.3), 1.0)                        # 5 or 8 coefficients
    with pytest.raises(ValueError):
        capi.make_lens(KV2_LENS)                                    # a default r2_max needs the camera
    K, cols, rows = KV2_DEPTH
    want = 1.21 * max(((u - K[2]) / K[0]) ** 2 + ((v - K[3]) / K[1]) ** 2 for u in (0, cols) for v in (0, rows))
    assert capi.make_lens(KV2_LENS, None, K, cols, rows).r2_max == np.float32(want) == np.float32(capi.default_r2_max(K, cols, rows))


@pytest.mark.parametrize("r2_max", [1e-3, 1.0, 1e6])
def test_zero_lens_is_the_identity(r2_max):
    rng = np.random.default_rng(1)
    for (K, cols, rows) in (KV2_DEPTH, ((570.342, 570.342, 320.0, 240.0), 640, 480), ((151.0, 149.0, 101.3, 74.8), 203, 151)):
        depth = rng.integers(0, 65536, (rows, cols + 3), np.uint16)[:, :cols]
        bgra = rng.integers(0, 256, (rows, cols + 5, 4), np.uint8)[:, :cols]
        out, bout = lo.undistort(depth, K, (0,) * 8 + (r2_max,), bgra)
        assert np.array_equal(out, depth) and np.array_equal(bout, bgra)


@pytest.mark.parametrize("coeffs", [KV2_LENS, STRONG_LENS])
def test_synth_lens_round_trip(coeffs):
    from dynamicfusion_b200 import synth
    K, cols, rows = KV2_DEPTH
    u, v = np.meshgrid(np.arange(cols, dtype=np.float64), np.arange(rows, dtype=np.float64))
    x, y = synth.undistort((u - K[2]) / K[0], (v - K[3]) / K[1], coeffs)
    xd, yd = synth.distort(x, y, coeffs)
    assert np.abs(xd * K[0] + K[2] - u).max() < 1e-9 and np.abs(yd * K[1] + K[3] - v).max() < 1e-9
    assert np.hypot(xd - x, yd - y).max() * K[0] > 5                # the lens does move pixels
    with pytest.raises(AssertionError):
        synth.undistort(np.array([0.3]), np.array([0.2]), coeffs, max_iter=1)


def test_synth_without_a_lens_is_unchanged():
    from dynamicfusion_b200 import synth
    assert np.array_equal(synth.umbrella_depth(2), synth.umbrella_depth(2, lens=None))
    d, c = synth.umbrella_rgbd(1, lens=None)
    assert np.array_equal(d, synth.umbrella_rgbd(1)[0]) and np.array_equal(c, synth.umbrella_rgbd(1)[1])
    # the lens changes the recorded frame, and a registered colour image shares it
    dl, cl = synth.umbrella_rgbd(1, lens=KV2_LENS)
    assert np.array_equal(dl, synth.umbrella_depth(1, lens=KV2_LENS)) and (dl != d).mean() > 0.1 and (cl != c).any()


def _depth_edges(d):
    """pixels whose 3 x 3 neighbourhood spans more than 10 mm (or touches an invalid pixel)"""
    p = np.pad(d.astype(np.int64), 1, mode="edge")
    rows, cols = d.shape
    win = np.stack([p[i:i + rows, j:j + cols] for i in range(3) for j in range(3)])
    return (win.max(0) - win.min(0) > 10) | (win.min(0) == 0)


def test_undistorted_c2_frame_matches_the_pinhole_truth():
    from dynamicfusion_b200 import capi, synth
    K, cols, rows = KV2_DEPTH
    lens = capi.make_lens(KV2_LENS, None, K, cols, rows)
    for t in (0, 7):
        truth = synth.umbrella_depth(t, cols, rows, K, noise_mm=0, dropout=0)
        raw = synth.umbrella_depth(t, cols, rows, K, noise_mm=0, dropout=0, lens=KV2_LENS)
        ud, _ = lo.undistort(raw, K, lens)
        keep = (truth > 0) & ~_depth_edges(truth)
        border = np.zeros_like(keep)
        border[:40], border[-40:], border[:, :40], border[:, -40:] = True, True, True, True
        good = np.abs(ud.astype(int) - truth.astype(int)) <= 2
        raw_good = np.abs(raw.astype(int) - truth.astype(int)) <= 2
        print(f"t={t}: undistorted {good[keep].mean():.4f} within 2 mm; the raw frame {raw_good[keep].mean():.4f}, at the border "
              f"{raw_good[keep & border].mean():.4f}")
        assert good[keep].mean() >= 0.99 and good[keep & border].mean() >= 0.99
        assert raw_good[keep & border].mean() < 0.9                  # the negative control: the raw frame taken as a pinhole frame fails


# --------------------------------------------------------------------------------------------------------------------------- snapshots
def _lens_section(capi, depth=None, color=None):
    out = b""
    for L in (depth, color):
        out += bytes([L is not None]) + (bytes(L) if L is not None else bytes(36))
    return out


def _snapshot_lenses(lib, capi, data):
    d, c, dp, cp = capi.Lens(), capi.Lens(), C.c_int(-1), C.c_int(-1)
    buf = np.frombuffer(data, np.uint8)
    st = lib.df_kinfu_snapshot_lenses(buf.ctypes.data, len(data), C.byref(d), C.byref(dp), C.byref(c), C.byref(cp))
    return st, dp.value, bytes(d), cp.value, bytes(c)


def test_snapshot_version_4_checks(lib):
    from dynamicfusion_b200 import capi
    from dynamicfusion_b200.kinfu import COLOR, KinFu
    assert C.sizeof(capi.Lens) == 36
    p1, p2 = sm.small_params(capi, lib, 0), sm.small_params(capi, lib, COLOR)
    dims = tuple(p2.volume_dims)
    v1 = sm.v1_body(capi, lib, p1)
    length, cls, payload, rgba = sm.color_sections(dims)
    v2 = sm.v1_body(capi, lib, p2) + length + cls + payload + rgba
    cam = sm.camera_bytes(capi)
    dl, cl = capi.make_lens(KV2_LENS, 1.0), capi.make_lens(STRONG_LENS, 1.5)

    def accepted(body, version=4):
        data = sm.header(body, version=version) + body
        return _call_params(lib, capi, data) == 0 and _snapshot_lenses(lib, capi, data)[0] == 0
    for body, want in ((v1 + _lens_section(capi, dl), (1, bytes(dl), 0, bytes(36))),
                       (v2 + _lens_section(capi, dl), (1, bytes(dl), 0, bytes(36))),
                       (v2 + cam + _lens_section(capi, dl, cl), (1, bytes(dl), 1, bytes(cl))),
                       (v2 + cam + _lens_section(capi, None, cl), (0, bytes(36), 1, bytes(cl)))):
        data = sm.header(body, version=4) + body
        assert accepted(body) and _snapshot_lenses(lib, capi, data)[1:] == want
        d, c = KinFu.snapshot_lenses(data)
        assert (d is not None, c is not None) == (bool(want[0]), bool(want[2]))
    # without a version-4 section there are no lenses
    assert _snapshot_lenses(lib, capi, sm.header(v1) + v1) == (0, 0, bytes(36), 0, bytes(36))
    assert _snapshot_lenses(lib, capi, sm.header(v2 + cam, version=3) + v2 + cam)[1::2] == (0, 0)
    # refusals
    assert not accepted(v1 + _lens_section(capi))                   # version 4 without a lens
    assert not accepted(v1 + _lens_section(capi, dl), version=1)    # the section is not part of version 1
    assert not accepted(v1 + _lens_section(capi, dl)[:-1]) and not accepted(v1 + _lens_section(capi, dl) + b"\0")
    assert not accepted(v1 + _lens_section(capi, None, cl))         # a colour lens without a camera
    assert not accepted(v2 + _lens_section(capi, None, cl))
    assert not accepted(v1 + _lens_section(capi, capi.make_lens((-0.5, 0, 0, 0, 0), 1.0)))     # a folding lens
    assert not accepted(v1 + _lens_section(capi, capi.make_lens((0,) * 5, 1.0)))              # the zero lens is no lens
    bad = bytearray(v1 + _lens_section(capi, dl)); bad[len(v1)] = 2
    assert not accepted(bytes(bad))                                 # a presence byte of 0 or 1
    bad = bytearray(v1 + _lens_section(capi, dl)); bad[-1] = 1
    assert not accepted(bytes(bad))                                 # an absent record is zero
    good = v1 + _lens_section(capi, dl)
    corrupt = bytearray(sm.header(good, version=4) + good); corrupt[-40] ^= 1
    assert _call_params(lib, capi, bytes(corrupt)) != 0              # the checksum covers the section
    assert lib.df_kinfu_snapshot_lenses(np.frombuffer(good, np.uint8).ctypes.data, len(good), None, None, None, None) != 0


def _call_params(lib, capi, data):
    out = capi.KinfuParams()
    buf = np.frombuffer(data, np.uint8)
    return lib.df_kinfu_snapshot_params(buf.ctypes.data, len(data), C.byref(out))


def test_oracle_without_a_lens_is_the_colour_camera_oracle():
    """lens_oracle.c's colour rules with a NULL or zero lens are color_camera_oracle.c's"""
    from dynamicfusion_b200 import synth
    K = synth.DEFAULT_K
    cam = cco.Camera(320, 240, (285.171, 285.171, 159.5, 119.5), (np.eye(3, dtype=np.float32), np.array([-0.05, 0.0, 0.0], np.float32)))
    depth = synth.umbrella_depth(0)
    want = cco.depth_map(depth, K, cam)
    assert np.array_equal(lo.depth_map(depth, K, cam, None), want)
    assert np.array_equal(lo.depth_map(depth, K, cam, (0,) * 8 + (0.5,)), want)
    assert not np.array_equal(lo.depth_map(depth, K, cam, STRONG_LENS + (1.5,)), want)
