"""The relocaliser on the GPU (DF_KINFU_RELOCALISE): df_fern_encode and df_fern_match equal tests/reloc_oracle.c bit for bit,
df_icp_inliers stays inside the oracle's bracket, a run that never loses tracking is the run without the flag bit for bit (plus three
launches a frame), blank frames leave the state alone, a lost camera comes back from a keyframe and not from an unrelated view, and reset
and create do what the header says."""
import ctypes as C
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("orc")]

import reloc_oracle as ro  # noqa: E402
import gpu_util as gu  # noqa: E402
from dynamicfusion_b200 import capi, kinfu as kf, synth  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]
F, K_CAND = capi.RELOC_FERNS, capi.RELOC_CANDIDATES


def _params(flags, dim=128):
    return gu.kinfu_params(dim, flags, max_nodes=1024, cloud_capacity=1_000_000)


def _level2(k):
    return k.buffer("curr_depth", 2)


# ------------------------------------------------------------------------------------------------------------ kernels against the oracle
def _gpu_encode(depth, table, extra_bytes):
    rows, cols = depth.shape
    d, pitch, _ = gu.padded(depth, extra_bytes // 2, 7)
    t = gu.dev(np.ascontiguousarray(table, np.int32))
    out = torch.zeros(len(table), dtype=torch.uint8, device="cuda")
    capi.check(capi.load().df_fern_encode(d.data_ptr(), pitch, cols, rows, t.data_ptr(), len(table), out.data_ptr(), gu.stream()))
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("scene", ["C1", "C2", "ragged"])
@pytest.mark.parametrize("extra", [0, 2, 512])
def test_fern_codes_equal_the_oracle(scene, extra):
    if scene == "ragged":
        rng = np.random.default_rng(3)
        depth = rng.integers(0, 3200, (151, 203)).astype(np.uint16)
        depth[rng.random(depth.shape) < 0.1] = 0
    else:
        k = kf.KinFu(_params(kf.RELOCALISE | kf.RIGID_ONLY))
        k(synth.sphere_wall_depth() if scene == "C1" else synth.umbrella_depth(3))
        depth = np.ascontiguousarray(_level2(k))
    rows, cols = depth.shape
    table = ro.fern_table(capi.RELOC_SEED, cols, rows).reshape(F, 12)
    lib_table = np.empty(F * 12, np.int32)
    capi.check(capi.load().df_reloc_fern_table(capi.RELOC_SEED, cols, rows, F, lib_table.ctypes.data))
    assert np.array_equal(lib_table.reshape(F, 12), table)
    want = ro.encode(depth, table)
    assert np.array_equal(_gpu_encode(depth, table, extra), want)
    if scene != "ragged":                                              # the loop codes its own level-2 image with this table: keyframe 0
        assert np.array_equal(k.keyframes()[1][0], want)
    assert 0 < np.count_nonzero(want) < F                              # the codes say something about the image


@pytest.mark.parametrize("count", [0, 1, 511, 512])
@pytest.mark.parametrize("append", [0, 1])
def test_match_topk_and_append_equal_the_oracle(count, append):
    rng = np.random.default_rng(count + 17 * append)
    cap = capi.RELOC_KEYFRAMES
    db = rng.integers(0, 16, (cap, F)).astype(np.uint8)
    code = rng.integers(0, 16, F).astype(np.uint8)
    if count > 4 and not append:                                       # ties: three entries at the same distance, one near duplicate
        for i in (5, 9, 300):
            db[i] = code
            db[i, :45] ^= 1
        db[200] = code
        db[200, :3] ^= 1
    poses = rng.standard_normal((cap, 12)).astype(np.float32)
    pose = capi.make_aff(np.eye(3) * 0.5, (1.0, 2.0, 3.0))
    d_db, d_poses = gu.dev(db), gu.dev(poses)
    d_count = gu.dev(np.array([count], np.int32))
    d_code = gu.dev(code)
    out = torch.zeros(C.sizeof(capi.RelocMatch), dtype=torch.uint8, device="cuda")
    capi.check(capi.load().df_fern_match(d_db.data_ptr(), d_poses.data_ptr(), d_count.data_ptr(), cap, d_code.data_ptr(), F, append, pose,
                                         out.data_ptr(), gu.stream()))
    torch.cuda.synchronize()
    m = capi.RelocMatch.from_buffer_copy(out.cpu().numpy().tobytes())
    want_db = db.copy()
    idx, dis, add, n = ro.match(want_db, count, code, bool(append))
    assert list(m.index) == idx.tolist() and list(m.dissimilarity) == dis.tolist()
    assert bool(m.appended) == add and m.count == n and int(d_count.cpu().numpy()[0]) == n
    for r in range(K_CAND):
        assert np.array_equal(np.array(m.pose[r]), poses[idx[r]] if idx[r] >= 0 else np.zeros(12, np.float32))
    assert np.array_equal(gu.host(d_db, np.uint8, db.shape), want_db)
    got_poses = d_poses.cpu().numpy()
    if add:
        assert np.array_equal(got_poses[count], np.array(list(pose.R) + list(pose.t), np.float32))
    assert np.array_equal(got_poses[:count], poses[:count])
    assert add == (append == 1 and count < cap)                        # random codes are novel: the append fills the database at 511


def _rot(deg, axis):
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    i, j = [(1, 2), (0, 2), (0, 1)][axis]
    R = np.eye(3)
    R[i, i], R[i, j], R[j, i], R[j, j] = c, -s, s, c
    return R


@pytest.mark.parametrize("which", ["identity", "near", "far"])
def test_gate_counts_within_the_oracle_bracket(which):
    k = kf.KinFu(_params(kf.RELOCALISE | kf.RIGID_ONLY))
    for t in range(3):
        k(synth.umbrella_depth(t))
    vc, nc = k.buffer("curr_points"), k.buffer("curr_normals")
    vp, np_ = k.buffer("prev_points"), k.buffer("prev_normals")
    R, t = {"identity": (np.eye(3), (0, 0, 0)), "near": (_rot(1.0, 1), (0.004, -0.002, 0.003)), "far": (_rot(8.0, 0), (0.06, 0.0, 0.0))}[which]
    T12 = np.concatenate([np.asarray(R, np.float32).reshape(9), np.asarray(t, np.float32)])
    p = k.params
    Kp = (p.intr.fx, p.intr.fy, p.intr.cx, p.intr.cy)
    n_valid, n_in, amb, s = ro.gate(vc, nc, vp, np_, Kp, T12, p.icp_dist_thres, p.icp_angle_thres)
    keep, maps = [], []                                                 # the device copies live until the calls are done
    for a in (vc, nc, vp, np_):
        d, pitch, _ = gu.padded(np.ascontiguousarray(a, np.float32), 4, np.nan)
        keep.append(d)
        maps += [d.data_ptr(), pitch]
    d_T = gu.dev(T12)
    ws = torch.zeros(capi.RELOC_GATE_WS_BYTES, dtype=torch.uint8, device="cuda")
    out = torch.zeros(C.sizeof(capi.RelocGate), dtype=torch.uint8, device="cuda")
    results = []
    for _ in range(2):                                                 # the workspace is left zeroed: the second call equals the first
        capi.check(capi.load().df_icp_inliers(*maps, p.cols, p.rows, capi.make_intr(*Kp), d_T.data_ptr(), None, p.icp_dist_thres,
                                              p.icp_angle_thres, out.data_ptr(), ws.data_ptr(), gu.stream()))
        torch.cuda.synchronize()
        results.append(capi.RelocGate.from_buffer_copy(out.cpu().numpy().tobytes()))
    g = results[0]
    assert bytes(results[1]) == bytes(g)
    assert g.ok == 1 and np.array_equal(np.array(g.T, np.float32), T12)
    assert g.n_valid == n_valid and n_valid > 100_000
    assert abs(g.n_in - n_in) <= amb
    # float residuals: each r^2 to a relative 1e-5 (a few float ulps of r), plus the bracket's pixels at most dist_thres^2 each
    assert abs(g.sum_sq - s) <= 1e-5 * s + amb * p.icp_dist_thres ** 2
    if which == "identity":                                            # every point projects onto a pixel centre: all on a boundary
        assert n_in > 0.5 * n_valid
    else:
        assert amb <= n_in // 10


# ------------------------------------------------------------------------------------------------------------ the frame loop
SEQUENCES = {
    "default": (0, "C2"),
    "warped": (kf.WARPED_INTEGRATE | kf.EXTEND_FIELD, "C2"),
    "color": (kf.COLOR | kf.COLOR_TRACKING, "C2rgbd"),
    "rigid": (kf.RIGID_ONLY, "C1"),
}


def _frame(kind, t):
    if kind == "C1":
        return synth.sphere_wall_depth(seed=t), None
    if kind == "C2rgbd":
        return synth.umbrella_rgbd(t)
    return synth.umbrella_depth(t), None


@pytest.mark.parametrize("name", list(SEQUENCES))
def test_no_loss_means_no_change(name):
    flags, kind = SEQUENCES[name]
    off, on = kf.KinFu(_params(flags)), kf.KinFu(_params(flags | kf.RELOCALISE))
    for t in range(60):
        d, c = _frame(kind, t)
        assert off(d, c) == on(d, c)
        assert gu.state(off) == gu.state(on), f"frame {t}"
        a, b = off.info(), on.info()
        if t > 0:
            assert b["launches"] - a["launches"] == 3, f"frame {t}"
    info = on.info()
    assert info["lost_frames"] == 0 and info["lost"] == 0 and info["resets"] == 0 and info["keyframes"] >= 2
    poses, codes = on.keyframes()
    assert poses.shape == (info["keyframes"], 12) and codes.shape == (info["keyframes"], F)
    assert np.array_equal(poses[0], np.concatenate([np.eye(3, dtype=np.float32).reshape(9), np.zeros(3, np.float32)]))


BLANK = np.zeros((480, 640), np.uint16)


def test_blank_frames_are_lost_and_leave_the_state_alone():
    frames = [synth.umbrella_depth(t) for t in range(30)]
    off = kf.KinFu(_params(0))
    for d in frames[:20] + [BLANK] * 3 + frames[20:]:
        off(d)
    # without the flag the first blank frame resets the object, the second becomes a new first frame, and the third fails its ICP against
    # that empty model and resets again
    assert off.info()["resets"] == 2
    ref = kf.KinFu(_params(kf.RELOCALISE))
    on = kf.KinFu(_params(kf.RELOCALISE))
    for t in range(20):
        ref(frames[t]), on(frames[t])
    before = gu.state(on)
    for _ in range(3):
        assert on(BLANK) is False
        assert gu.state(on) == before and on.info()["lost"] == 1
    assert on.info()["lost_frames"] == 3
    for t in range(20, 30):
        assert on(frames[t]) == ref(frames[t])
        assert gu.state(on) == gu.state(ref), f"frame {t}"
    info = on.info()
    assert info["lost"] == 0 and info["relocalisations"] == 1 and info["resets"] == 0


def _angle_deg(Ra, Rb):
    c = (np.trace(np.asarray(Ra, np.float64).T @ np.asarray(Rb, np.float64)) - 1) / 2
    return np.degrees(np.arccos(np.clip(c, -1, 1)))


def _pose_error(k, t):
    """(cm, degrees) between the object's latest pose and the synthetic camera at frame t, both relative to frame 0's camera"""
    R, tr = k.getCameraPose()
    Rg, tg = synth.camera_drift(t)
    R0, t0 = synth.camera_drift(0)
    Rrel, trel = R0.T @ Rg, R0.T @ (tg - t0)
    return 100 * np.linalg.norm(tr - trel), _angle_deg(R, Rrel)


DRIFT, EARLY = 150, 6


def _static(t, **kw):
    return synth.umbrella_depth(t, shape_t=0, **kw)


@pytest.mark.parametrize("flags", [kf.RIGID_ONLY, 0], ids=["rigid", "default"])
def test_relocalise_from_a_keyframe(flags):
    k = kf.KinFu(_params(flags | kf.RELOCALISE))
    for t in range(DRIFT):
        k(_static(t))
    assert k.info()["lost_frames"] == 0
    tracked_launches = k.info()["launches"]
    assert k(BLANK) is False
    R_last, _ = k.getCameraPose()
    Rg, tg = synth.camera_drift(EARLY)
    assert np.linalg.norm(tg - synth.camera_drift(DRIFT - 1)[1]) >= 0.1 and _angle_deg(R_last, Rg) >= 10
    assert k(_static(EARLY, seed=5)) is True
    info = k.info()
    assert info["relocalisations"] == 1 and info["lost"] == 0
    cm, deg = _pose_error(k, EARLY)
    assert cm < 1.0 and deg < 1.0, (cm, deg)
    # candidate 0 (the ordinary ICP from the last good pose) was rejected: the frame went on to ray-cast and track a keyframe
    assert info["launches"] > tracked_launches + 2 * sum(k.params.icp_iter_num)
    for t in range(EARLY + 1, EARLY + 11):
        assert k(_static(t)) is True
    assert k.info()["lost_frames"] == 1


def test_no_false_relocalisation():
    k = kf.KinFu(_params(kf.RELOCALISE | kf.RIGID_ONLY))
    for t in range(40):
        k(_static(t))
    assert k(BLANK) is False
    before = gu.state(k)
    for s in range(5):
        assert k(synth.sphere_wall_depth(seed=s, centre=(0.0, 0.0, 2.0), wall_z=2.6)) is False
        assert gu.state(k) == before
    assert k.info()["relocalisations"] == 0 and k.info()["lost_frames"] == 6
    assert k(_static(40)) is True
    assert k.info()["relocalisations"] == 1


def test_reset_empties_the_database():
    k = kf.KinFu(_params(kf.RELOCALISE | kf.RIGID_ONLY))
    for t in range(20):
        k(_static(t))
    k(BLANK)
    assert k.info()["lost"] == 1 and k.info()["keyframes"] >= 2
    k.reset()
    info = k.info()
    assert info["lost"] == 0 and info["keyframes"] == 0
    k(_static(0))
    assert k.info()["keyframes"] == 1


@pytest.mark.parametrize("other", [kf.USE_DEPTH, kf.LIVE_MODEL])
def test_create_refuses(other):
    with pytest.raises(RuntimeError):
        kf.KinFu(_params(kf.RELOCALISE | other))
    p = _params(kf.RELOCALISE)
    p.icp_iter_num[2] = 0
    with pytest.raises(RuntimeError):
        kf.KinFu(p)


def test_environment_enables_it():
    code = ("import sys; sys.path.insert(0, %r); from dynamicfusion_b200 import kinfu as kf; sys.path.insert(0, %r); import gpu_util as gu; "
            "k = kf.KinFu(gu.kinfu_params(64, 1, max_nodes=64, cloud_capacity=100000)); "
            "from dynamicfusion_b200 import synth; k(synth.umbrella_depth(0)); print(k.info()['keyframes'])") % (str(ROOT), str(ROOT / "tests"))
    env = dict(os.environ, DF_KINFU_RELOCALISE="1")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, check=True)
    assert out.stdout.strip().splitlines()[-1] == "1"


def _resume_state(k):
    info = k.info()
    return gu.state(k), {key: info[key] for key in ("frame_counter", "poses", "resets", "lost", "lost_frames", "relocalisations", "keyframes")}, \
        [a.tobytes() for a in k.keyframes()]


@pytest.mark.parametrize("flags", [kf.RIGID_ONLY, 0], ids=["rigid", "default"])
def test_snapshots_while_lost_and_after_relocalising_resume_exactly(flags):
    frames = [_static(t) for t in range(30)] + [BLANK, _static(EARLY, seed=5)] + [_static(t) for t in range(EARLY + 1, EARLY + 4)]
    ref = kf.KinFu(_params(flags | kf.RELOCALISE))
    states, snaps = [], {}
    for i, d in enumerate(frames):
        ref(d)
        states.append(_resume_state(ref))
        if i in (30, 31):                                              # taken while lost, and right after relocalising
            snaps[i] = ref.snapshot()
    assert states[30][1]["lost"] == 1 and states[31][1]["relocalisations"] == 1
    for i, data in snaps.items():
        assert kf.KinFu.snapshot_params(data).flags & kf.RELOCALISE
        k = kf.KinFu(_params(flags | kf.RELOCALISE))
        k.restore(data)
        assert _resume_state(k) == states[i]
        for j in range(i + 1, len(frames)):
            k(frames[j])
            assert _resume_state(k) == states[j], f"snapshot {i}, frame {j}"


def test_version5_rejections_leave_the_state_unchanged():
    k = kf.KinFu(_params(kf.RELOCALISE | kf.RIGID_ONLY))
    for t in range(12):
        k(_static(t))
    k(BLANK)
    good = k.snapshot()
    for t in range(12, 15):
        k(_static(t))
    before = _resume_state(k)
    import snapshot_model as sm
    cut = sm.reseal(good[:-9] + good[-8:])                             # one keyframe pose byte short
    count_off = len(good) - 8 - int(np.frombuffer(good[-8:], "<u8")[0]) + 32
    over = bytearray(good)
    over[count_off:count_off + 4] = np.int32(capi.RELOC_KEYFRAMES + 1).tobytes()
    plain = kf.KinFu(_params(kf.RIGID_ONLY))
    plain(_static(0))
    for data in (cut, sm.reseal(bytes(over)), plain.snapshot()):
        with pytest.raises(RuntimeError):
            k.restore(data)
        assert _resume_state(k) == before
    with pytest.raises(RuntimeError):                                  # and the other way round: a version-5 snapshot into a plain object
        plain.restore(good)


def test_cpp_mirror_equals_python_on_blank_frames(tmp_path):
    from dynamicfusion_b200 import build
    exe = build.build_cpp_program(ROOT / "tests" / "cpp" / "reloc_export.cpp", ROOT / "tests" / "cpp" / "_build" / "reloc_export")
    frames = [synth.umbrella_depth(t) for t in range(20)] + [BLANK] * 3 + [synth.umbrella_depth(t) for t in range(20, 25)]
    np.stack(frames).tofile(tmp_path / "depth.u16")
    r = subprocess.run([str(exe), str(tmp_path / "depth.u16"), str(len(frames)), str(tmp_path / "frames.bin"), str(tmp_path / "cpp.ply")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    rec = np.fromfile(tmp_path / "frames.bin", np.uint8).reshape(len(frames), 50)
    p = kf.KinFuParams.default_params_dynamicfusion()
    p.flags = kf.RELOCALISE
    k = kf.KinFu(p)
    for t, d in enumerate(frames):
        fused = k(d)
        R, tr = k.getCameraPose()
        assert rec[t, 0] == fused and rec[t, 1] == k.info()["lost"], f"frame {t}"
        assert rec[t, 2:].tobytes() == np.concatenate([R.reshape(9), tr]).astype(np.float32).tobytes(), f"frame {t}"
    assert rec[20:23, 0].tolist() == [0, 0, 0] and rec[20:23, 1].tolist() == [1, 1, 1] and rec[23, :2].tolist() == [1, 0]
    k.save_mesh(tmp_path / "py.ply", live=True)
    assert (tmp_path / "cpp.ply").read_bytes() == (tmp_path / "py.ply").read_bytes()
