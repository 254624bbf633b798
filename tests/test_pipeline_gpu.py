"""GPU parity of the whole per-frame loop (df_kinfu_* through the C ABI) vs the oracle's restated loop on the same
seeded sequence.  The two sides are NOT bit-identical end to end: the bilateral filter uses expf (CUDA's and glibc's differ
by <= 2 ulp, +-1 LSB on a handful of depth pixels) and the ICP sums are reduced in a different order, so the comparison
is statistical on the volume and tolerance-based on poses / nodes; every individual stage is compared bit-exactly in
test_tsdf_gpu.py / test_stages_gpu.py."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from dynamicfusion_b200 import kinfu as kf, synth  # noqa: E402
import gpu_util as gu  # noqa: E402


@pytest.mark.parametrize("flags", [0, kf.RIGID_ONLY])
def test_sequence_matches_oracle(orc, flags):
    from oracle import orc_pipe
    p = gu.kinfu_params(64, flags, max_nodes=512, cloud_capacity=400000)
    gpu = kf.KinFu(p)
    cpu = orc_pipe.KinFu(orc_pipe.params_from(p))
    frames = [synth.umbrella_depth(t) for t in range(4)]
    for t, d in enumerate(frames):
        # alternate the two entry points: host buffer (upload inside) and device-resident input
        r_gpu = gpu(d) if t % 2 == 0 else gpu(torch.from_numpy(d.view(np.int16).copy()).cuda())
        r_cpu = cpu(d)
        assert r_gpu == r_cpu == (t > 0)
    gi, ci = gpu.info(), cpu.info()
    assert gi["poses"] == ci["poses"] == 4 and gi["resets"] == ci["resets"] == 0
    for t in range(4):
        Rg, tg = gpu.getCameraPose(t)
        Rc, tc = cpu.getCameraPose(t)
        assert np.abs(Rg - Rc).max() < 2e-4 and np.abs(tg - tc).max() < 2e-4, t
    vg, vc = gpu.buffer("volume"), cpu.buffer("volume")
    fg, wg = gu.tsdf(vg)
    fc, wc = gu.tsdf(vc)
    tol = 2e-3 if flags else 2e-2      # non-rigid: +-1 LSB bilateral differences move a few removed pixels (whole rays of voxels)
    assert np.mean(wg != wc) < tol
    same = wg == wc
    assert np.mean(np.abs(fg[same] - fc[same]) > 2e-3) < tol
    # any-bit differences of the packed voxels: half-precision LSB flips that follow the ~6e-6 pose difference between the device ICP
    # (float partial sums per thread) and the oracle's (double running sum); measured 5.3e-3 rigid with f-mismatch (> 2e-3) at 2e-4
    assert np.mean(vg != vc) < 4 * tol
    if not flags:
        assert gi["nodes"] == ci["nodes"] >= 8
        assert abs(gi["cloud_points"] - ci["cloud_points"]) <= 0.01 * ci["cloud_points"] + 5
        ng, nc = gpu.buffer("nodes")[: gi["nodes"]], cpu.buffer("nodes")
        assert np.array_equal(ng[:, :7], nc[:, :7])                      # same vertices, identity rotations
        tg, tc = 2 * ng[:, 8:11], 2 * nc[:, 8:11]
        scale = max(np.abs(tc).max(), 1e-6)
        # PCG stops on the reference's q-tolerance (1e-4): weakly constrained nodes keep a few % of slack, the bulk agrees tightly
        assert np.abs(tg - tc).max() <= 1.5e-1 * scale + 2e-5
        assert np.median(np.abs(tg - tc)) <= 5e-3 * scale + 2e-6
        sg, sc = gpu.buffer("solve_stats"), cpu.buffer("solve_stats")
        assert abs(sg[3] - sc[3]) <= 0.01 * sc[3]
        assert abs(sg[1] - sc[1]) <= 5e-2 * sc[1]
        cg, cc = gpu.buffer("canonical"), cpu.buffer("canonical")
        both = ~np.isnan(cg[..., 0]) & ~np.isnan(cc[..., 0])
        assert np.mean(np.isnan(cg[..., 0]) != np.isnan(cc[..., 0])) < 5e-3
        assert np.median(np.abs(cg[both][:, :3] - cc[both][:, :3])) < 1e-4
    gpu.close(); cpu.close()


def test_first_frame_bit_exact_when_bilateral_is_bypassed(orc):
    """frame 0 only touches dists -> integrate -> extract: those must be bit-identical to the oracle (no expf involved)"""
    from oracle import orc_pipe
    p = gu.kinfu_params(96, 0, max_nodes=512, cloud_capacity=400000)
    gpu = kf.KinFu(p)
    cpu = orc_pipe.KinFu(orc_pipe.params_from(p))
    d = synth.umbrella_depth(0)
    assert gpu(d) is False and cpu(d) is False
    assert np.array_equal(gpu.buffer("volume"), cpu.buffer("volume"))
    assert np.array_equal(gpu.buffer("cloud").view(np.uint32), cpu.buffer("cloud").view(np.uint32))
    assert np.array_equal(gpu.buffer("cloud_normals").view(np.uint32), cpu.buffer("cloud_normals").view(np.uint32))
    gi = gpu.info()
    assert np.array_equal(gpu.buffer("nodes")[: gi["nodes"]], cpu.buffer("nodes"))
    gpu.close(); cpu.close()


def test_reset_on_tracking_loss_and_recovery():
    p = gu.kinfu_params(32, kf.RIGID_ONLY, max_nodes=512, cloud_capacity=400000)
    k = kf.KinFu(p)
    assert k(synth.sphere_wall_depth(seed=0)) is False
    assert k(synth.sphere_wall_depth(seed=1)) is True
    assert k(np.zeros((480, 640), np.uint16)) is False                   # ICP degenerate -> reset (kinfu.cpp:276-277)
    i = k.info()
    assert i["resets"] == 1 and i["frame_counter"] == 0 and i["poses"] == 1
    assert int(np.abs(k.buffer("volume").astype(np.int64)).sum()) == 0   # volume cleared
    assert k(synth.sphere_wall_depth(seed=2)) is False                   # first frame again
    assert k(synth.sphere_wall_depth(seed=3)) is True
    k.close()


def test_volume_dims_must_be_multiple_of_32():
    p = gu.kinfu_params(40, 0, max_nodes=512, cloud_capacity=400000)
    with pytest.raises(RuntimeError):
        kf.KinFu(p)                                                      # CV_Assert(dims[0] % 32 == 0), kinfu.cpp:97


def test_stage_timing_and_launch_count():
    p = gu.kinfu_params(64, kf.STAGE_TIMING, max_nodes=512, cloud_capacity=400000)
    k = kf.KinFu(p)
    for t in range(3):
        k(synth.umbrella_depth(t))
    ms = k.stage_ms()
    assert set(ms) == set(kf.STAGES) and all(v >= 0 for v in ms.values()) and ms["integrate"] > 0
    assert k.info()["launches"] >= 50
    k.close()


def test_batch_entry_advances_independent_sequences_concurrently():
    """df_kinfu_batch_process_host (SURVEY 8e, config 5): n objects -- one per GPU where there are several, all on this GPU otherwise --
    advanced concurrently by one host thread each must end in exactly the state of the same sequences run one by one"""
    import ctypes as C
    ndev = torch.cuda.device_count()
    n, frames = 3, 4
    seqs = [[synth.umbrella_depth(t, seed=s) for t in range(frames)] for s in range(n)]
    want, want_nodes = [], []
    for s in range(n):
        k = kf.KinFu(gu.kinfu_params(64, 0, max_nodes=512, cloud_capacity=400000))
        for d in seqs[s]:
            k(d)
        want.append(k.state_digest())
        want_nodes.append(k.buffer("nodes")[: k.info()["nodes"]].copy())
        k.close()
    ks = []
    for s in range(n):
        torch.cuda.set_device(s % ndev)
        ks.append(kf.KinFu(gu.kinfu_params(64, 0, max_nodes=512, cloud_capacity=400000)))
    torch.cuda.set_device(0)
    lib = ks[0].lib
    handles = (C.c_void_p * n)(*[k.h for k in ks])
    pitches = (C.c_size_t * n)(*([640 * 2] * n))
    results = (C.c_int * n)()
    for t in range(frames):
        ptrs = (C.c_void_p * n)(*[seqs[s][t].ctypes.data for s in range(n)])
        assert lib.df_kinfu_batch_process_host(handles, ptrs, pitches, n, results) == 0
        assert list(results) == [int(t > 0)] * n
    got = [k.state_digest() for k in ks]
    got_nodes = [k.buffer("nodes")[: k.info()["nodes"]].copy() for k in ks]
    for k in ks:
        k.close()
    # Every sequence must be reproduced -- to rounding, not bit for bit: the order of a node's incidence list comes from an atomic cursor
    # (solve_fill), so under different kernel timing (three host threads feeding one stream here) the double sums of the row assembly
    # are added in a different order, a translation can differ in its last bit, and a last bit can move a warped vertex across a pixel
    # border of project-and-remove (DESIGN 4: known limit of the solve's reproducibility; one object per stream/GPU, run alone, has
    # reproduced its digests exactly in every bench run so far).
    assert len({g[0] for g in got}) == n                             # they really are different sequences
    for g, w in zip(got, want):
        assert abs(g[2] - w[2]) <= 2e-3 * w[2] + 2                    # extracted cloud points
    for a, b in zip(got_nodes, want_nodes):
        assert a.shape == b.shape and np.array_equal(a[:, :7], b[:, :7])
        assert np.median(np.abs(a[:, 7:11] - b[:, 7:11])) <= 1e-4 * max(np.abs(b[:, 7:11]).max(), 1e-6) + 1e-9


def test_use_depth_loop_tracks_like_the_points_loop():
    """DF_KINFU_USE_DEPTH: the reference's compile-time USE_DEPTH frame loop (internal.hpp:6; kinfu.cpp:237-238,271,293-295) -- depth-pyramid
    ICP against a model ray-cast stored as a depth map.  The oracle has no such loop (the reference's default build is the points loop, and
    its USE_DEPTH build hands KinFu::dynamicfusion a vertex map it never fills); every operator of it is compared with the reference's own
    kernels in test_render_gpu.py / test_stages_gpu.py, so the loop is checked by what it must share with the points loop: same first frame
    bit for bit, poses within millimetres, no tracking loss."""
    frames = [synth.umbrella_depth(t) for t in range(5)]
    runs = {}
    for flags in (0, kf.USE_DEPTH):
        k = kf.KinFu(gu.kinfu_params(64, flags, max_nodes=512, cloud_capacity=400000))
        vols = []
        for t, d in enumerate(frames):
            assert k(d) == (t > 0)
            if t == 0:
                vols.append(k.buffer("volume").copy())
        runs[flags] = (vols[0], [k.getCameraPose(t) for t in range(5)], k.info(), k.buffer("volume") >> 16)
        k.close()
    a, b = runs[0], runs[kf.USE_DEPTH]
    assert np.array_equal(a[0], b[0])                                   # frame 0 does not depend on the ICP variant
    assert a[2]["resets"] == b[2]["resets"] == 0 and a[2]["nodes"] == b[2]["nodes"]
    for (Ra, ta), (Rb, tb) in zip(a[1], b[1]):
        # different correspondences (depth-map association vs vertex-map association): measured 7e-3 rad in the weakly constrained
        # in-plane rotation of this rotationally symmetric scene, 1e-3 elsewhere
        assert np.abs(Ra - Rb).max() < 2e-2 and np.abs(ta - tb).max() < 1e-2
    assert np.mean(a[3] != b[3]) < 0.1


def test_f2_solve_in_the_frame_loop():
    """DF_KINFU_F2_SOLVE: the frame's warp solve is df_solve_f2 (robust 6-DoF data term + regulariser, SURVEY 8f(2)); opt-in, parity unpinned --
    checked here only for what must hold: the loop runs, the energy of every frame's solve does not increase, nodes stay finite and the
    rotations move (the translation-only solve leaves them at identity)."""
    import ctypes as C
    k = kf.KinFu(gu.kinfu_params(64, kf.F2_SOLVE, max_nodes=512, cloud_capacity=400000))
    for t in range(4):
        assert k(synth.umbrella_depth(t)) == (t > 0)
        if t:
            ptr, pitch, c_, r_ = C.c_void_p(), C.c_size_t(), C.c_int(), C.c_int()
            from dynamicfusion_b200 import capi
            capi.check(k.lib.df_kinfu_get_buffer(k.h, kf.BUF["f2_stats"], C.byref(ptr), C.byref(pitch), C.byref(c_), C.byref(r_)))
            st = np.empty(16, np.float64)
            capi.check(k.lib.df_kinfu_read_buffer(k.h, kf.BUF["f2_stats"], st.ctypes.data, 128))
            assert np.all(np.isfinite(st)) and st[3] > 10_000 and st[1] <= st[0]
    i = k.info()
    nodes = k.buffer("nodes")[: i["nodes"]]
    assert i["resets"] == 0 and np.all(np.isfinite(nodes))
    assert np.abs(nodes[:, 4:7]).max() > 1e-6                           # rotation increments were applied
    assert np.allclose(np.linalg.norm(nodes[:, 3:7], axis=1), 1.0, atol=1e-5)
    k.close()
