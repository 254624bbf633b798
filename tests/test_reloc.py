"""The relocaliser's rules on the CPU (DF_KINFU_RELOCALISE, include/dfusion.h): the library's fern table equals the oracle's, the oracle's
codes, lookup, harvest and gate on hand-made inputs, and the library's gate decision at its thresholds.  No GPU needed."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

import reloc_oracle as ro
from dynamicfusion_b200 import capi

ROOT = Path(__file__).resolve().parents[1]
F = capi.RELOC_FERNS


def _lib():
    from dynamicfusion_b200 import build
    build.build()
    return capi.load()


def test_constants_match_the_header():
    text = (ROOT / "include" / "dfusion.h").read_text()
    defs = dict(re.findall(r"^#define\s+DF_(RELOC_[A-Z_]+|KINFU_RELOCALISE)\s+(\S+)", text, flags=re.M))
    for name in ("FERNS", "CANDIDATES", "KEYFRAMES", "NEAR_MM", "FAR_MM", "HARVEST_FERNS", "MIN_VALID", "GATE_WS_BYTES"):
        assert int(defs["RELOC_" + name]) == getattr(capi, "RELOC_" + name), name
    assert int(defs["RELOC_SEED"].rstrip("ul"), 16) == capi.RELOC_SEED
    assert float(defs["RELOC_MIN_INLIER_FRAC"].rstrip("f")) == capi.RELOC_MIN_INLIER_FRAC
    assert float(defs["RELOC_MAX_RMS"].rstrip("f")) == capi.RELOC_MAX_RMS
    from dynamicfusion_b200 import kinfu
    assert int(defs["KINFU_RELOCALISE"]) == kinfu.RELOCALISE == 2048
    assert C.sizeof(capi.RelocGate) == 72


@pytest.mark.parametrize("seed", [capi.RELOC_SEED, 12345])
@pytest.mark.parametrize("size", [(160, 120), (203, 151)])
def test_fern_table_equals_the_oracle(seed, size):
    cols, rows = size
    got = np.empty(F * 12, np.int32)
    assert _lib().df_reloc_fern_table(seed, cols, rows, F, got.ctypes.data) == 0
    want = ro.fern_table(seed, cols, rows)
    assert np.array_equal(got.reshape(F, 4, 3), want)
    assert want[..., 0].min() >= 0 and want[..., 0].max() < cols and want[..., 1].max() < rows
    assert want[..., 2].min() >= capi.RELOC_NEAR_MM and want[..., 2].max() < capi.RELOC_FAR_MM
    assert len(np.unique(want[..., 2])) > 1000                        # the thresholds spread over the range
    assert _lib().df_reloc_fern_table(seed, 0, rows, F, got.ctypes.data) != 0


def test_codes_on_hand_made_images():
    depth = np.zeros((4, 8), np.uint16)
    depth[0, 1], depth[0, 2], depth[0, 3] = 1000, 999, 0
    # fern 0: (1, 0) at 1000 -> d == theta gives 0; (2, 0) at 1000 -> 999 < 1000 gives 1; (3, 0) invalid gives 0; (2, 0) at 2000 gives 1
    table = np.array([[[1, 0, 1000], [2, 0, 1000], [3, 0, 5000], [2, 0, 2000]],
                      [[3, 0, 400], [3, 0, 2999], [1, 0, 1001], [7, 3, 500]]], np.int32)
    codes = ro.encode(depth, table)
    assert codes.tolist() == [0b1010, 0b0100]


def test_dissimilarity_and_topk_ties():
    cap = 8
    db = np.zeros((cap, F), np.uint8)
    code = np.zeros(F, np.uint8)
    db[0, :10] = 1          # 10
    db[1, :3] = 2           # 3
    db[2, :10] = 3          # 10
    db[3, :3] = 1           # 3
    db[4, :1] = 1           # 1
    idx, dis, add, n = ro.match(db, 5, code, False, capacity=cap)
    assert idx.tolist() == [4, 1, 3] and dis.tolist() == [1, 3, 3] and not add and n == 5
    idx, dis, _, _ = ro.match(db, 2, code, False, capacity=cap)
    assert idx.tolist() == [1, 0, -1] and dis.tolist() == [3, 10, F + 1]
    idx, dis, _, _ = ro.match(db, 0, code, False, capacity=cap)
    assert idx.tolist() == [-1, -1, -1]


def test_harvest_at_the_threshold_and_at_capacity():
    h = capi.RELOC_HARVEST_FERNS
    cap = 4
    db = np.zeros((cap, F), np.uint8)
    code = np.zeros(F, np.uint8)
    assert ro.match(db, 0, code, True, capacity=cap)[2:] == (True, 1)          # an empty database always takes the frame
    near = code.copy(); near[:h] = 5                                             # exactly at the bar: not novel
    assert ro.match(db, 1, near, True, capacity=cap)[2:] == (False, 1)
    far = code.copy(); far[:h + 1] = 5                                           # one fern more: novel
    assert ro.match(db, 1, far, True, capacity=cap)[2:] == (True, 2)
    assert np.array_equal(db[1], far)
    assert ro.match(db, 2, far, False, capacity=cap)[2:] == (False, 2)          # a lookup never appends
    other = code.copy(); other[100:100 + h + 1] = 9
    assert ro.match(db, cap, other, True, capacity=cap)[2:] == (False, cap)     # full: no growth, nothing evicted


def _plane(z, cols=100, rows=80, K=(100.0, 100.0, 50.0, 40.0)):
    fx, fy, cx, cy = K
    y, x = np.mgrid[0:rows, 0:cols].astype(np.float32) + np.float32(0.25)   # each point projects a quarter pixel inside its pixel
    v = np.stack([(x - cx) / fx * z, (y - cy) / fy * z, np.full_like(x, z), np.zeros_like(x)], -1).astype(np.float32)
    n = np.zeros_like(v)
    n[..., 2] = -1.0
    return v, n, K


def test_gate_on_hand_made_maps():
    v, n, K = _plane(1.0)
    ident = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float32)
    n_valid, n_in, amb, s = ro.gate(v, n, v, n, K, ident, 0.1, np.float32(30 * 0.017453293))
    assert (n_valid, n_in, amb, s) == (8000, 8000, 0, 0.0)
    v2 = v.copy(); v2[:20, :, 0] = np.nan                                # invalid current pixels do not count
    shift = ident.copy(); shift[11] = 0.02                               # 2 cm along z: every residual is 2 cm
    n_valid, n_in, amb, s = ro.gate(v2, n, v, n, K, shift, 0.1, np.float32(30 * 0.017453293))
    assert n_valid == 6000 and n_in == 6000 and abs(s - 6000 * 0.02 ** 2) < 1e-6
    far = ident.copy(); far[11] = 0.2                                    # 20 cm: beyond the distance test
    assert ro.gate(v2, n, v, n, K, far, 0.1, np.float32(30 * 0.017453293))[1] == 0


@pytest.mark.parametrize("case,want", [
    ((1, 10000, 10000, 0.0), True),
    ((0, 10000, 10000, 0.0), False),                                             # ICP failed
    ((1, capi.RELOC_MIN_VALID - 1, capi.RELOC_MIN_VALID - 1, 0.0), False),        # too little depth
    ((1, 10000, 1000, 0.0), True),                                               # exactly the inlier share
    ((1, 10000, 999, 0.0), False),
    ((1, 10000, 10000, 10000 * 0.0299 ** 2), True),                               # just inside the RMS bar
    ((1, 10000, 10000, 10000 * 0.0301 ** 2), False),
])
def test_gate_decision_library_equals_oracle(case, want):
    g = capi.RelocGate()
    g.ok, g.n_valid, g.n_in, g.sum_sq = case
    assert bool(_lib().df_reloc_gate_accepts(C.byref(g))) == want
    assert ro.accepts(*case) == want


# ---------------------------------------------------------------------------------------------- version-5 snapshots (host-side checks)
import struct  # noqa: E402

import snapshot_model as sm  # noqa: E402
from snapshot_model import lib  # noqa: E402,F401  (the module's fixture)

RELOC_HEAD = struct.Struct("<IB3xqqQii")         # base version, lost, lost frames, relocalisations, fern seed, keyframe count, ferns


def _reloc_section(count, base=1, lost=1, seed=capi.RELOC_SEED, ferns=F, length=None):
    rng = np.random.default_rng(count)
    body = RELOC_HEAD.pack(base, lost, 3, 1, seed, count, ferns)
    body += rng.integers(0, 16, count * F, np.uint8).tobytes() + rng.random(count * 12, np.float32).tobytes()
    return body + struct.pack("<Q", len(body) + 8 if length is None else length)


def _v5(lib, flags=2048, version=5, **kw):
    p = sm.small_params(capi, lib, flags)
    body = sm.v1_body(capi, lib, p) + _reloc_section(**kw)
    return sm.header(body, version=version) + body


def test_version5_snapshot_header_length_and_flag_checks(lib):
    st, p = sm.read_params(lib, capi, _v5(lib, count=4))
    assert st == 0 and p.flags == 2048
    assert sm.read_params(lib, capi, _v5(lib, count=0))[0] == 0
    assert sm.read_params(lib, capi, _v5(lib, count=capi.RELOC_KEYFRAMES))[0] == 0
    good = _v5(lib, count=4)
    bad = {
        "truncated": sm.reseal(good[:-1]),
        "section cut short": sm.reseal(good[:-9] + good[-8:]),
        "flag without the section": (lambda b: sm.header(b) + b)(sm.v1_body(capi, lib, sm.small_params(capi, lib, 2048))),
        "section without the flag": _v5(lib, flags=0, count=4),
        "more keyframes than the database": _v5(lib, count=capi.RELOC_KEYFRAMES + 1),
        "another seed": _v5(lib, count=4, seed=capi.RELOC_SEED + 1),
        "another fern count": _v5(lib, count=4, ferns=F - 4),
        "base version 0": _v5(lib, count=4, base=0),
        "base version 5": _v5(lib, count=4, base=5),
        "lost byte 2": _v5(lib, count=4, lost=2),
        "length field too long": _v5(lib, count=4, length=len(_reloc_section(4)) + 1),
        "length field too short": _v5(lib, count=4, length=8),
    }
    for name, data in bad.items():
        assert sm.read_params(lib, capi, sm.reseal(data) if name != "truncated" else data)[0] != 0, name
    v1 = sm.v1_body(capi, lib, sm.small_params(capi, lib, 0))
    assert sm.read_params(lib, capi, sm.header(v1, version=6) + v1)[0] != 0
