"""numpy model of the snapshot format (include/dfusion.h, "Snapshots"): the checksum, the three-class brick packing of a volume, and the
byte offsets of a snapshot's sections -- written from the format's description, so the tests pin it independently of the C++ code.  Also
the byte strings of made-up snapshots the host-side checks feed to the library, and the `lib` fixture those checks call it through."""
import ctypes as C
import struct

import numpy as np
import pytest

from scenes import word

MAGIC = b"DFUSNAP\0"
VERSION = 1
HEADER = 32
F2_BYTES = 48
COUNTERS = struct.Struct("<6iqQ")          # frame_counter, resets, last_ok, M, cloud_count, n_poses, solve_overflows, payload_bytes
BRICK = 8
GOLDEN = 0x9E3779B97F4A7C15


def checksum(body: bytes) -> int:
    n = len(body)
    w = np.frombuffer(body + b"\0" * (-n % 8), "<u8")
    with np.errstate(over="ignore"):
        z = w ^ (np.arange(len(w), dtype=np.uint64) * np.uint64(GOLDEN))
        z = z + np.uint64(GOLDEN)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
        return (int(z.sum(dtype=np.uint64)) + n) % (1 << 64)


def header(body: bytes, magic=MAGIC, version=VERSION, total=None, check=None) -> bytes:
    total = HEADER + len(body) if total is None else total
    check = checksum(body) if check is None else check
    return magic + struct.pack("<IIQQ", version, HEADER, total, check)


def reseal(snap: bytes) -> bytes:
    """the same snapshot with its checksum recomputed (for tests that must get past the checksum)"""
    return header(snap[HEADER:]) + snap[HEADER:]


def counters_offset(params_bytes: int) -> int:
    return HEADER + params_bytes + F2_BYTES


def counters(snap: bytes, params_bytes: int):
    return COUNTERS.unpack_from(snap, counters_offset(params_bytes))


def brick_count(dims) -> int:
    return int(np.prod([(d + BRICK - 1) // BRICK for d in dims]))


def pack(vol: np.ndarray, dims):
    """(class bytes, payload u32 words) of a volume of dims (x, y, z): brick order z, y, x; 0 empty, 1 uniform (one word), 2 mixed (512
    words in (z, y, x) order, slots outside the volume 0)"""
    Dx, Dy, Dz = dims
    nbx, nby, nbz = [(d + BRICK - 1) // BRICK for d in dims]
    pad = np.zeros((nbz * BRICK, nby * BRICK, nbx * BRICK), np.uint32)
    inside = np.zeros(pad.shape, bool)
    pad[:Dz, :Dy, :Dx] = vol.reshape(Dz, Dy, Dx)
    inside[:Dz, :Dy, :Dx] = True

    def bricks(a):
        return a.reshape(nbz, BRICK, nby, BRICK, nbx, BRICK).transpose(0, 2, 4, 1, 3, 5).reshape(-1, BRICK ** 3)
    b, m = bricks(pad), bricks(inside)
    first = b[:, 0]
    same = np.all((b == first[:, None]) | ~m, axis=1)
    cls = np.where(same, np.where(first != 0, 1, 0), 2).astype(np.uint8)
    parts = [b[i] if c == 2 else first[i:i + 1] for i, c in enumerate(cls) if c]
    payload = np.concatenate(parts) if parts else np.zeros(0, np.uint32)
    return cls, payload



# ------------------------------------------------------------------------------------------------------- made-up snapshots (host code only)
@pytest.fixture(scope="module")
def lib():
    from dynamicfusion_b200 import build, capi
    build.build()
    return capi.load()


def small_params(capi, lib, flags):
    """the library's default parameters for a 64 x 48 frame and a 32 x 24 x 20 volume, with `flags`"""
    p = capi.KinfuParams()
    lib.df_kinfu_default_params(C.byref(p), 0)
    p.cols, p.rows = 64, 48
    for i in range(3):
        p.volume_dims[i] = (32, 24, 20)[i]
    p.icp_iter_num[:] = [3, 2, 0, 0]
    p.cloud_capacity = 1000
    p.flags = flags
    return p


def v1_body(capi, lib, p, cloud=5):
    """the body of a version-1 snapshot of made-up state for the parameters p"""
    dims = tuple(p.volume_dims)
    vol = capi.make_volume(None, dims, (1.0, 1.0, 1.0), 0.1, 64)
    pyr = sum((p.cols >> l) * (p.rows >> l) * 32 for l in range(2))
    rng = np.random.default_rng(3)
    body = bytes(p) + bytes(capi.F2Params()) + COUNTERS.pack(4, 1, 1, 3, cloud, 2, 0, 4 * 7)
    body += rng.random(2 * 12, np.float32).tobytes() + rng.random(3 * 12, np.float32).tobytes()
    body += bytes(lib.df_volume_activity_bytes(vol)) + rng.random(pyr // 4, np.float32).tobytes() + rng.random(cloud * 8, np.float32).tobytes()
    body += bytes(brick_count(dims)) + rng.integers(0, 2 ** 32, 7, np.uint32).tobytes()
    return body


def color_sections(dims, cloud=5):
    """version 2's trailing sections for a colour volume with one uniform and one mixed brick"""
    vol = np.zeros(dims[::-1], np.uint32)
    vol[0:8, 0:8, 0:8] = word(1, 2, 3, 4)
    vol[8:16, 8:12, 0:5] = word(9, 9, 9, 1)
    cls, payload = pack(vol.reshape(-1), dims)
    assert sorted(np.unique(cls)) == [0, 1, 2] and len(payload) == 1 + 512
    return struct.pack("<Q", 4 * len(payload)), cls.tobytes(), payload.tobytes(), np.arange(cloud, dtype=np.uint32).tobytes()


def camera_bytes(capi, K_=(1081.0, 1081.0, 959.5, 539.5), cols=1920, rows=1080, t=(0.052, 0.0, 0.0)):
    """version 3's colour-camera record"""
    cam = capi.make_color_camera(K_, cols, rows, ((1, 0, 0, 0, 1, 0, 0, 0, 1), t))
    assert C.sizeof(cam) == 72
    return bytes(cam)


def read_params(lib, capi, data: bytes):
    """(status, parameters) of df_kinfu_snapshot_params on data"""
    out = capi.KinfuParams()
    buf = np.frombuffer(data, np.uint8) if data else np.zeros(1, np.uint8)
    return lib.df_kinfu_snapshot_params(buf.ctypes.data, len(data), C.byref(out)), out
