"""Snapshots on the GPU: brick packing of volumes against the numpy model of the format, exact resume of the frame loop in every
configuration, rejection of damaged or mismatched snapshots without touching the target, determinism, and the C++ mirror."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import snapshot_model as sm  # noqa: E402
from dynamicfusion_b200 import capi, kinfu as kf, synth  # noqa: E402
import gpu_util as gu  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]
PARAMS_BYTES = C.sizeof(capi.KinfuParams)


# ---------------------------------------------------------------------------------------------------------------------------------
# df_volume_pack_* / df_volume_unpack
def _vol(t, dims):
    return capi.make_volume(t.data_ptr(), dims, (1.0, 1.0, 1.0), 0.1, 64)


def _gpu_pack(lib, vol_np, dims):
    v = torch.from_numpy(vol_np.view(np.int32)).cuda()
    V = _vol(v, dims)
    nb = lib.df_volume_brick_count(V)
    ws = torch.zeros(lib.df_volume_pack_workspace_bytes(V), dtype=torch.uint8, device="cuda")
    cls = torch.full((nb,), 77, dtype=torch.uint8, device="cuda")
    nbytes = torch.zeros(1, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    capi.check(lib.df_volume_pack_count(V, ws.data_ptr(), cls.data_ptr(), nbytes.data_ptr(), s))
    n = int(nbytes.item())
    guard = 64
    pay = torch.full((n // 4 + guard,), -1, dtype=torch.int32, device="cuda")
    capi.check(lib.df_volume_pack_emit(V, ws.data_ptr(), cls.data_ptr(), pay.data_ptr(), n, s))
    out = pay.cpu().numpy().view(np.uint32)
    assert np.all(out[n // 4:] == 0xFFFFFFFF)                         # nothing past `capacity`
    if n >= 8:                                                        # a short capacity cuts the payload, never writes beyond it
        short = torch.full((n // 4,), -1, dtype=torch.int32, device="cuda")
        capi.check(lib.df_volume_pack_emit(V, ws.data_ptr(), cls.data_ptr(), short.data_ptr(), n - 8, s))
        sh = short.cpu().numpy().view(np.uint32)
        assert np.array_equal(sh[:-2], out[:n // 4 - 2]) and np.all(sh[-2:] == 0xFFFFFFFF)
    return cls.cpu().numpy(), out[:n // 4].copy()


def _gpu_unpack(lib, cls, payload, dims, fill):
    t = torch.from_numpy(fill.view(np.int32).copy()).cuda()
    V = _vol(t, dims)
    ws = torch.zeros(lib.df_volume_pack_workspace_bytes(V), dtype=torch.uint8, device="cuda")
    c = torch.from_numpy(cls.copy()).cuda()
    p = torch.from_numpy(np.concatenate([payload, np.zeros(1, np.uint32)]).view(np.int32)).cuda()
    status = torch.full((1,), -5, dtype=torch.int32, device="cuda")
    capi.check(lib.df_volume_unpack(V, c.data_ptr(), p.data_ptr(), payload.nbytes, ws.data_ptr(), status.data_ptr(),
                                    torch.cuda.current_stream().cuda_stream))
    return int(status.item()), t.cpu().numpy().view(np.uint32)


def _volumes():
    rng = np.random.default_rng(11)
    k = kf.KinFu(gu.kinfu_params(64, 0, max_nodes=512, cloud_capacity=400000))
    for t in range(4):
        k(synth.umbrella_depth(t))
    scene = k.buffer("volume").copy()
    k.close()
    dims = (96, 60, 44)
    ragged = np.zeros(dims[::-1], np.uint32)
    ragged[:20] = 0x00013C00                                          # free space: F = 1, W = 1
    ragged[30:, 50:, :] = 0x00023C00                                  # a uniform region that ends in the ragged bricks
    ragged[25, 10:30, 40:70] = rng.integers(1, 2 ** 32, (20, 30), np.uint32)
    ragged[43, 59, 95] = 7                                            # the last voxel: one mixed edge brick
    return {"umbrella_64": (scene, (64, 64, 64)), "ragged_96x60x44": (ragged.reshape(-1), dims),
            "zero": (np.zeros(64 ** 3, np.uint32), (64, 64, 64)), "same_word": (np.full(64 ** 3, 0x00053C00, np.uint32), (64, 64, 64)),
            "random": (rng.integers(0, 2 ** 32, 32 * 40 * 24, np.uint32), (32, 40, 24))}


def test_pack_unpack_round_trip_bit_for_bit():
    lib = capi.load()
    rng = np.random.default_rng(5)
    for name, (vol, dims) in _volumes().items():
        cls, payload = _gpu_pack(lib, vol, dims)
        mcls, mpay = sm.pack(vol, dims)
        assert np.array_equal(cls, mcls) and np.array_equal(payload, mpay), name
        counts = np.bincount(cls, minlength=3)
        assert payload.size == counts[1] + 512 * counts[2], name
        if name == "zero":
            assert counts[0] == cls.size and payload.size == 0
        if name == "same_word":
            assert counts[1] == cls.size
        if name == "random":
            assert counts[2] == cls.size
        if name.startswith("umbrella"):                               # free space of a real scan carries varying weights: no uniform bricks
            assert counts[0] > 0 and counts[2] > 0
        if name.startswith("ragged"):
            assert counts[2] > 0 and counts[1] > 0 and counts[0] > 0
        for fill in (np.zeros_like(vol), rng.integers(0, 2 ** 32, vol.size, np.uint32)):
            st, out = _gpu_unpack(lib, cls, payload, dims, fill)
            assert st == 0 and np.array_equal(out, vol), name
        # rejected inputs leave the volume untouched
        garbage = rng.integers(0, 2 ** 32, vol.size, np.uint32)
        bad = cls.copy(); bad[-1] = 3
        st, out = _gpu_unpack(lib, bad, payload, dims, garbage)
        assert st == 1 and np.array_equal(out, garbage), name
        st, out = _gpu_unpack(lib, cls, np.concatenate([payload, np.zeros(1, np.uint32)]), dims, garbage)
        assert st == 2 and np.array_equal(out, garbage), name
        if payload.size:
            st, out = _gpu_unpack(lib, cls, payload[:-1], dims, garbage)
            assert st == 2 and np.array_equal(out, garbage), name


# ---------------------------------------------------------------------------------------------------------------------------------
# exact resume of the frame loop
FRAMES = [synth.umbrella_depth(t) for t in range(8)]


def _state(k):
    R, t = k.getCameraPose()
    return {"digest": k.state_digest(), "pose": np.concatenate([R.reshape(9), t]).view(np.uint32), "nodes": k.buffer("nodes").view(np.uint32).copy(),
            "prev_points": k.buffer("prev_points").view(np.uint32).copy(), "prev_normals": k.buffer("prev_normals").view(np.uint32).copy(),
            "volume": k.buffer("volume").copy(), "info": {x: y for x, y in k.info().items() if x not in ("launches", "lm_iters", "pcg_iters")}}


def _same(a, b):
    for key in a:
        if isinstance(a[key], np.ndarray):
            assert np.array_equal(a[key], b[key]), key
        else:
            assert a[key] == b[key], key


def _straight(flags):
    k = kf.KinFu(gu.kinfu_params(64, flags, max_nodes=512, cloud_capacity=400000))
    states = []
    for d in FRAMES:
        k(d)
        states.append(_state(k))
    k.close()
    return states


@pytest.mark.parametrize("flags", [0, kf.RIGID_ONLY, kf.WARPED_INTEGRATE, kf.EXTEND_FIELD, kf.USE_DEPTH])
def test_resume_equals_the_uninterrupted_run(flags, tmp_path):
    straight = _straight(flags)
    assert straight[-1]["info"]["resets"] == 0
    for k_stop in (0, 3):
        a = kf.KinFu(gu.kinfu_params(64, flags, max_nodes=512, cloud_capacity=400000))
        for d in FRAMES[:k_stop + 1]:
            a(d)
        path = tmp_path / f"s{k_stop}.dfsnap"
        n = a.save(path)
        assert n == path.stat().st_size
        a.close()
        b = kf.KinFu.from_snapshot(path)
        loaded, want = _state(b), dict(straight[k_stop])
        if flags & kf.USE_DEPTH:                                      # that loop keeps the previous frame as depth: its points are scratch
            del loaded["prev_points"], want["prev_points"]
        _same(loaded, want)
        assert b.snapshot() == path.read_bytes()                     # the save of a resumed object is the snapshot it came from
        for t in range(k_stop + 1, 8):
            assert b(FRAMES[t])
            _same(_state(b), straight[t])
        b.close()


def test_f2_solve_restores_exactly_and_keeps_tracking(tmp_path):
    flags = kf.F2_SOLVE
    a = kf.KinFu(gu.kinfu_params(64, flags, max_nodes=512, cloud_capacity=400000))
    poses = []
    for d in FRAMES:
        a(d)
        poses.append(np.concatenate([x.reshape(-1) for x in a.getCameraPose()]))
    a.close()
    a = kf.KinFu(gu.kinfu_params(64, flags, max_nodes=512, cloud_capacity=400000))
    for d in FRAMES[:4]:
        a(d)
    snap = a.snapshot()
    b = kf.KinFu(gu.kinfu_params(64, flags, max_nodes=512, cloud_capacity=400000))
    b.restore(snap)
    assert b.snapshot() == snap
    _same(_state(b), _state(a))
    a.close()
    for t in range(4, 8):
        assert b(FRAMES[t])
        assert np.allclose(np.concatenate([x.reshape(-1) for x in b.getCameraPose()]), poses[t], atol=1e-3)
    assert b.info()["resets"] == 0


def test_snapshot_after_a_tracking_loss_resumes_into_a_first_frame(tmp_path):
    a = kf.KinFu(gu.kinfu_params(64, 0, max_nodes=512, cloud_capacity=400000))
    for d in FRAMES[:3]:
        a(d)
    assert a(np.zeros((480, 640), np.uint16)) is False                 # ICP degenerate -> reset
    assert a.info()["frame_counter"] == 0 and a.info()["resets"] == 1
    snap = a.snapshot()
    b = kf.KinFu(gu.kinfu_params(64, 0, max_nodes=512, cloud_capacity=400000))
    b.restore(snap)
    assert (a(FRAMES[3]), b(FRAMES[3])) == (False, False)              # both take the first-frame path
    _same(_state(b), _state(a))
    for t in (4, 5):
        assert a(FRAMES[t]) and b(FRAMES[t])
        _same(_state(b), _state(a))


def test_loading_over_another_sequence_equals_loading_into_a_fresh_object():
    a = kf.KinFu(gu.kinfu_params(64, 0, max_nodes=512, cloud_capacity=400000))
    for d in FRAMES[:4]:
        a(d)
    snap = a.snapshot()
    used = kf.KinFu(gu.kinfu_params(64, 0, max_nodes=512, cloud_capacity=400000))
    for t in range(5):
        used(synth.umbrella_depth(t, seed=7))
    fresh = kf.KinFu(gu.kinfu_params(64, 0, max_nodes=512, cloud_capacity=400000))
    used.restore(snap)
    fresh.restore(snap)
    assert used.snapshot() == fresh.snapshot() == snap
    for t in range(4, 8):
        assert used(FRAMES[t]) and fresh(FRAMES[t])
        _same(_state(used), _state(fresh))


def test_snapshot_resumes_on_another_device():
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    straight = _straight(0)
    a = kf.KinFu(gu.kinfu_params(64, 0, max_nodes=512, cloud_capacity=400000))
    for d in FRAMES[:4]:
        a(d)
    snap = a.snapshot()
    a.close()
    with torch.cuda.device(1):
        b = kf.KinFu(gu.kinfu_params(64, 0, max_nodes=512, cloud_capacity=400000))
        b.restore(snap)
        for t in range(4, 8):
            assert b(FRAMES[t])
            _same(_state(b), straight[t])
        b.close()


def test_rejected_snapshots_leave_the_object_untouched():
    a = kf.KinFu(gu.kinfu_params(64, 0, max_nodes=512, cloud_capacity=400000))
    for d in FRAMES[:3]:
        a(d)
    snap = a.snapshot()
    target = kf.KinFu(gu.kinfu_params(64, 0, max_nodes=512, cloud_capacity=400000))
    for d in FRAMES[:2]:
        target(d)
    before, before_snap = target.state_digest(), target.snapshot()
    pb = sm.counters(snap, PARAMS_BYTES)[7]
    classes_at = len(snap) - pb - sm.brick_count((64, 64, 64))
    three = bytearray(snap); three[classes_at + 10] = 3
    flipped = bytearray(snap); flipped[-5] ^= 0x10
    bad = {"truncated": snap[:-1], "flipped payload byte": bytes(flipped), "class byte 3": sm.reseal(bytes(three))}
    other = kf.KinFu(gu.kinfu_params(96, 0, max_nodes=512, cloud_capacity=400000))
    for d in FRAMES[:2]:
        other(d)
    other_snap = other.snapshot()
    for name, data in bad.items():
        with pytest.raises(RuntimeError):
            target.restore(data)
        assert target.state_digest() == before, name
    with pytest.raises(RuntimeError):
        target.restore(other_snap)                                     # params mismatch (other dims)
    with pytest.raises(RuntimeError):
        other.restore(snap)
    assert target.state_digest() == before and target.snapshot() == before_snap
    # the target still runs on, as if nothing had happened
    assert target(FRAMES[2])
    target.restore(snap)
    assert target.snapshot() == snap


def test_two_saves_of_the_same_state_are_identical():
    a = kf.KinFu(gu.kinfu_params(64, 0, max_nodes=512, cloud_capacity=400000))
    for d in FRAMES[:5]:
        a(d)
    s1 = a.snapshot()
    s2 = a.snapshot()
    assert s1 == s2
    assert bytes(kf.KinFu.snapshot_params(s1)) == bytes(a.params)


def test_cpp_mirror_save_and_load_resume_bit_for_bit(tmp_path):
    from dynamicfusion_b200 import build
    exe = build.build_cpp_program(ROOT / "tests" / "cpp" / "snapshot_resume.cpp", ROOT / "tests" / "cpp" / "_build" / "snapshot_resume")
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "all checks passed" in r.stdout
