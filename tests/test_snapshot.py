"""CPU checks of the snapshot format: df_kinfu_snapshot_params is host code, so headers built here from the format's description must be
accepted or rejected exactly as dfusion.h says, without a GPU.  The C++ program that saves and resumes through the mirror must build."""
import ctypes as C
import struct
from pathlib import Path

import numpy as np

import snapshot_model as sm
from snapshot_model import lib  # noqa: F401  (a fixture)

ROOT = Path(__file__).resolve().parents[1]


def _snapshot(capi, lib, p, n_poses=2, M=3, cloud=5, payload_words=7):
    """a well-formed snapshot of made-up state (no GPU involved)"""
    dims = tuple(p.volume_dims)
    vol = capi.make_volume(None, dims, (1.0, 1.0, 1.0), 0.1, 64)
    activity = lib.df_volume_activity_bytes(vol)
    assert lib.df_volume_brick_count(vol) == sm.brick_count(dims) == 4 * 3 * 3
    pyr = sum((p.cols >> l) * (p.rows >> l) * 32 for l in range(2))
    rng = np.random.default_rng(3)
    body = bytes(p) + bytes(capi.F2Params()) + sm.COUNTERS.pack(4, 1, 1, M, cloud, n_poses, 0, 4 * payload_words)
    body += rng.random(n_poses * 12, np.float32).tobytes() + rng.random(M * 12, np.float32).tobytes()
    body += bytes(activity) + rng.random(pyr // 4, np.float32).tobytes() + rng.random(cloud * 8, np.float32).tobytes()
    body += bytes(sm.brick_count(dims)) + rng.integers(0, 2 ** 32, payload_words, np.uint32).tobytes()
    return sm.header(body) + body


def test_valid_snapshot_returns_its_params(lib):
    from dynamicfusion_b200 import capi
    p = sm.small_params(capi, lib, 0)
    snap = _snapshot(capi, lib, p)
    st, out = sm.read_params(lib, capi, snap)
    assert st == 0 and bytes(out) == bytes(p)
    from dynamicfusion_b200.kinfu import KinFu
    assert bytes(KinFu.snapshot_params(snap)) == bytes(p)


def test_malformed_snapshots_are_rejected(lib):
    from dynamicfusion_b200 import capi
    p = sm.small_params(capi, lib, 0)
    snap = _snapshot(capi, lib, p)
    body = snap[sm.HEADER:]
    bad = {
        "empty": b"",
        "shorter than the header": snap[:20],
        "truncated": snap[:-1],
        "padded": snap + b"\0",
        "truncated, header patched": sm.header(body[:-4]) + body[:-4],
        "wrong magic": sm.header(body, magic=b"DFUSNAQ\0") + body,
        "wrong version": sm.header(body, version=2) + body,
        "bad checksum": snap[:-1] + bytes([snap[-1] ^ 1]),
        "checksum field": sm.header(body, check=sm.checksum(body) ^ 1) + body,
    }
    # counters that do not match the section lengths, checksum patched so that only the layout check can catch them
    off = sm.counters_offset(C.sizeof(capi.KinfuParams)) - sm.HEADER
    for name, fields in {"one pose too many": (4, 1, 1, 3, 5, 3, 0, 28), "no pose": (4, 1, 1, 3, 5, 0, 0, 28),
                         "negative node count": (4, 1, 1, -1, 5, 2, 0, 28), "payload not whole words": (4, 1, 1, 3, 5, 2, 0, 27),
                         "cloud over capacity": (4, 1, 1, 3, 1001, 2, 0, 28)}.items():
        b2 = body[:off] + sm.COUNTERS.pack(*fields) + body[off + sm.COUNTERS.size:]
        bad[name] = sm.header(b2) + b2
    for name, data in bad.items():
        st, _ = sm.read_params(lib, capi, data)
        assert st != 0, name


def test_checksum_model_matches_the_library(lib):
    """a snapshot sealed with the numpy checksum is accepted; every single-bit flip of its body is caught"""
    from dynamicfusion_b200 import capi
    p = sm.small_params(capi, lib, 0)
    snap = bytearray(_snapshot(capi, lib, p))
    rng = np.random.default_rng(0)
    for pos in rng.integers(sm.HEADER, len(snap), 16):
        flipped = bytearray(snap)
        flipped[pos] ^= 1 << int(rng.integers(0, 8))
        assert sm.read_params(lib, capi, bytes(flipped))[0] != 0
    assert struct.unpack_from("<Q", snap, 24)[0] == sm.checksum(bytes(snap[sm.HEADER:]))


def test_snapshot_cpp_program_compiles_and_links():
    from dynamicfusion_b200 import build
    exe = build.build_cpp_program(ROOT / "tests" / "cpp" / "snapshot_resume.cpp", ROOT / "tests" / "cpp" / "_build" / "snapshot_resume")
    assert exe.exists()
