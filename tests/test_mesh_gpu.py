"""The mesh extraction on the GPU (df_mesh_*, df_kinfu_mesh): triangles equal the oracle's element for element on both load paths and
both scan levels, with and without the activity map; the mesh of the frame loop uses the extracted cloud as its vertex buffer, changes no
state, is a consistently wound 2-manifold, warps like the loop warps, refuses a truncated cloud or a short buffer without writing, survives
a snapshot, and is exported identically by the C++ mirror."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from dynamicfusion_b200 import capi, host, kinfu as kf, synth  # noqa: E402
import gpu_util as gu  # noqa: E402
import mesh_oracle  # noqa: E402
from oracle import orc  # noqa: E402
from scenes import pack, sphere_volume  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]
IDENT = (np.eye(3, dtype=np.float32), np.zeros(3, np.float32))


def _activity(lib, vol_np, V):
    """the per-stretch bytes of an activity map, from the voxels themselves (non-zero iff the stretch holds an active voxel)"""
    w, f = vol_np >> 16, vol_np & 0xFFFF
    act = (w != 0) & (f != 0x3C00)
    n = -(-act.size // 1024)
    stretch = np.zeros(n * 1024, bool)
    stretch[:act.size] = act
    out = np.zeros(lib.df_volume_activity_bytes(V), np.uint8)
    out[:n] = stretch.reshape(n, 1024).any(1)
    return torch.from_numpy(out).cuda()


def _gpu_mesh(vol_np, dims, vs, trunc, use_activity):
    lib = capi.load()
    s = torch.cuda.current_stream().cuda_stream
    t = torch.from_numpy(vol_np.view(np.int32)).cuda()
    V = capi.make_volume(t.data_ptr(), dims, (vs,) * 3, trunc, 64)
    act = _activity(lib, vol_np, V) if use_activity else None
    ap = act.data_ptr() if act is not None else None
    cap = 3 * int(np.prod(dims))
    cloud = torch.empty((cap, 4), dtype=torch.float32, device="cuda")
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    ews = torch.empty(lib.df_extract_workspace_bytes(V), dtype=torch.uint8, device="cuda")
    capi.check(lib.df_extract_cloud_tracked(V, capi.make_aff(*IDENT), cloud.data_ptr(), cap, count.data_ptr(), ews.data_ptr(), ap, s))
    mws = torch.empty(lib.df_mesh_workspace_bytes(V), dtype=torch.uint8, device="cuda")
    dev = torch.full((2,), -9, dtype=torch.int32, device="cuda")
    capi.check(lib.df_mesh_count(V, ap, count.data_ptr(), mws.data_ptr(), dev.data_ptr(), dev[1:].data_ptr(), s))
    T, status = [int(x) for x in dev.cpu()]
    assert status == 0
    tris = torch.full((T + 32, 3), -7, dtype=torch.int32, device="cuda")
    capi.check(lib.df_mesh_emit(V, ap, mws.data_ptr(), tris.data_ptr(), T, s))
    out = tris.cpu().numpy()
    assert np.all(out[T:] == -7)                                          # nothing at or past the capacity
    if T > 4:                                                              # a short capacity cuts the list, never writes beyond it
        short = torch.full((T, 3), -7, dtype=torch.int32, device="cuda")
        capi.check(lib.df_mesh_emit(V, ap, mws.data_ptr(), short.data_ptr(), T - 3, s))
        sh = short.cpu().numpy()
        assert np.array_equal(sh[:T - 3], out[:T - 3]) and np.all(sh[T - 3:] == -7)
    n = int(count.item())
    # a stale count is refused
    bad = torch.tensor([n + 1], dtype=torch.int32, device="cuda")
    capi.check(lib.df_mesh_count(V, ap, bad.data_ptr(), mws.data_ptr(), dev.data_ptr(), dev[1:].data_ptr(), s))
    assert int(dev[1].item()) == 1                                        # DF_MESH_CLOUD_MISMATCH
    return cloud[:n].cpu().numpy(), out[:T]


def _cases():
    sph = sphere_volume()
    yield "sphere", sph[0], sph[1], sph[2][0], sph[3]
    yield ("c1_256",) + gu.c1_volume()
    odd = sphere_volume(dims=(99, 70, 45), radius_vox=17.2, centre_vox=(50.3, 33.1, 22.6))
    yield "odd_99x70x45", odd[0], odd[1], odd[2][0], odd[3]
    big = sphere_volume(dims=(256, 256, 80), radius_vox=30.4, centre_vox=(120.2, 131.7, 40.3))
    yield "blocks_256x256x80", big[0], big[1], big[2][0], big[3]


def test_triangles_equal_the_oracle():
    lib = capi.load()
    for name, vol, dims, vs, trunc in _cases():
        if name == "blocks_256x256x80":
            assert -(-int(np.prod(dims)) // 4096) > 1024                   # both levels of the block scan
        ref_cloud = orc.extract_cloud(vol, dims, (vs,) * 3, trunc, 64, IDENT, 3 * int(np.prod(dims)))
        ref = mesh_oracle.mesh(vol, dims, len(ref_cloud))
        assert ref is not None and len(ref) > 1000, name
        for use_activity in (False, True):
            cloud, tris = _gpu_mesh(vol, dims, vs, trunc, use_activity)
            assert len(cloud) == len(ref_cloud), name
            assert np.array_equal(cloud.view(np.uint32), ref_cloud.view(np.uint32)), (name, use_activity)   # point for point, in order
            assert np.array_equal(tris, ref), (name, use_activity)
            assert tris.min() >= 0 and tris.max() < len(cloud)
        if name.startswith("odd"):
            t = torch.from_numpy(vol.view(np.int32)).cuda()
            assert dims[0] % 4 != 0                                        # the 1-voxel path
            V = capi.make_volume(t.data_ptr(), dims, (vs,) * 3, trunc, 64)
            assert lib.df_mesh_workspace_bytes(V) >= 4 * int(np.prod(dims))


def test_plane_mesh_on_the_gpu():
    dims, vs = (64, 48, 40), 0.02
    z = np.arange(dims[2])[:, None, None] * np.ones((1, dims[1], dims[0]))
    vol = pack(np.clip(((z + 0.5) * vs - 17.3 * vs) / (3 * vs), -1.0, 1.0))
    _, tris = _gpu_mesh(vol, dims, vs, 3 * vs, True)
    assert len(tris) == 2 * (dims[0] - 1) * (dims[1] - 1)


# ------------------------------------------------------------------ the frame loop ------------------------------------------------------------
FRAMES = [synth.umbrella_depth(t) for t in range(10)]


def test_vertices_are_the_cloud_and_state_is_unchanged():
    k = gu.run(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=1_000_000), FRAMES[:6])
    before = k.state_digest()
    v, n, f = k.mesh()
    assert k.state_digest() == before
    cloud, cn = k.buffer("cloud"), k.buffer("cloud_normals")
    assert np.array_equal(v.view(np.uint32), cloud[:, :3].view(np.uint32))
    assert np.array_equal(n.view(np.uint32), cn[:, :3].view(np.uint32))
    assert len(f) > 1000 and f.min() >= 0 and f.max() < len(cloud)
    v2, n2, f2 = k.mesh()
    assert np.array_equal(f2, f) and np.array_equal(v2.view(np.uint32), v.view(np.uint32))
    k.close()


@pytest.mark.parametrize("overlap", ["1", "0"])
def test_meshing_every_frame_changes_nothing(monkeypatch, overlap):
    monkeypatch.setenv("DF_KINFU_OVERLAP_EXTRACT", overlap)
    a, b = (kf.KinFu(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=1_000_000)) for _ in range(2))
    for t, d in enumerate(FRAMES[:8]):
        a(d)
        b(d)
        b.mesh()
        if b.info()["nodes"] >= 8:
            b.mesh(live=True)
        assert a.state_digest() == b.state_digest(), t
    a.close()
    b.close()


def test_sequence_mesh_is_a_consistently_wound_manifold():
    k = gu.run(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=1_000_000), FRAMES)
    _, _, f = k.mesh()
    k.close()
    und = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    _, counts = np.unique(und, axis=0, return_counts=True)
    assert counts.max() <= 2
    directed = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    uniq, dcount = np.unique(directed, axis=0, return_counts=True)
    assert dcount.max() == 1                                               # an edge of two faces is traversed once in each direction


def test_live_mesh_is_the_loops_warp_of_the_cloud():
    k = gu.run(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=1_000_000), FRAMES[:6])
    assert k.info()["nodes"] >= 8
    vc, nc, fc = k.mesh()
    vl, nl, fl = k.mesh(live=True)
    assert np.array_equal(fl, fc)
    cloud, cn, nodes = k.buffer("cloud"), k.buffer("cloud_normals"), k.buffer("nodes")
    lib = capi.load()
    pts = torch.from_numpy(cloud.copy()).cuda()
    nrm = torch.from_numpy(cn.copy()).cuda()
    nd = torch.from_numpy(np.ascontiguousarray(nodes)).cuda()
    capi.check(lib.df_warp(nd.data_ptr(), len(nodes), None, pts.data_ptr(), nrm.data_ptr(), len(cloud), 4, capi.make_aff(*IDENT), 0, None,
                           None, torch.cuda.current_stream().cuda_stream))
    pw, nw = pts.cpu().numpy(), nrm.cpu().numpy()
    assert np.array_equal(vl.view(np.uint32), pw[:, :3].view(np.uint32))
    assert np.array_equal(nl.view(np.uint32), nw[:, :3].view(np.uint32))
    rp, rn = cloud.copy(), cn.copy()
    orc.warp(np.ascontiguousarray(nodes), rp, rn)
    assert np.allclose(vl, rp[:, :3], rtol=0, atol=1e-4)
    ok = ~np.isnan(rn[:, 0])
    assert np.array_equal(np.isnan(nl[:, 0]), ~ok) and np.allclose(nl[ok], rn[ok, :3], rtol=0, atol=1e-4)
    k.close()


def test_live_mesh_needs_a_warp_field():
    k = gu.run(gu.kinfu_params(128, kf.RIGID_ONLY, max_nodes=1024, cloud_capacity=1_000_000), FRAMES[:3])
    assert k.info()["nodes"] < 8
    with pytest.raises(RuntimeError):
        k.mesh(live=True)
    k.close()


def test_failures_write_nothing():
    lib = capi.load()
    k = gu.run(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=2000), FRAMES[:4])  # the cloud is cut at 2000 points
    assert k.info()["cloud_points"] == 2000
    before = k.state_digest()
    with pytest.raises(RuntimeError):
        k.mesh()
    assert k.state_digest() == before
    k.close()
    k = gu.run(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=1_000_000), FRAMES[:4])
    nv, nt = C.c_int(), C.c_int()
    capi.check(lib.df_kinfu_mesh(k.h, 0, None, None, None, 0, 0, C.byref(nv), C.byref(nt)))
    v = np.full((nv.value, 3), 7.0, np.float32)
    nrm = np.full((nv.value, 3), 7.0, np.float32)
    f = np.full((nt.value, 3), 7, np.int32)
    st = lib.df_kinfu_mesh(k.h, 0, v.ctypes.data, nrm.ctypes.data, f.ctypes.data, nv.value, nt.value - 1, C.byref(nv), C.byref(nt))
    assert st != 0
    assert np.all(v == 7.0) and np.all(nrm == 7.0) and np.all(f == 7)
    k.close()


def test_restored_object_gives_the_same_mesh(tmp_path):
    k = gu.run(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=1_000_000), FRAMES[:6])
    want = [k.mesh(), k.mesh(live=True)]
    k.save(tmp_path / "s.dfsnap")
    k.close()
    r = kf.KinFu.from_snapshot(tmp_path / "s.dfsnap")
    got = [r.mesh(), r.mesh(live=True)]
    r.close()
    for w, g in zip(want, got):
        for a, b in zip(w, g):
            assert a.tobytes() == b.tobytes()


def _read_ply(path):
    data = Path(path).read_bytes()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode().splitlines()
    nv = int(next(h for h in head if h.startswith("element vertex")).split()[-1])
    nf = int(next(h for h in head if h.startswith("element face")).split()[-1])
    ncol = sum(1 for h in head if h.startswith("property float"))
    v = np.frombuffer(data[end:end + nv * ncol * 4], "<f4").reshape(nv, ncol)
    rec = np.frombuffer(data[end + nv * ncol * 4:], np.dtype([("n", "u1"), ("v", "<i4", (3,))]))
    assert len(rec) == nf and np.all(rec["n"] == 3)
    return v, rec["v"]


def test_cpp_mirror_writes_the_same_mesh(tmp_path):
    from dynamicfusion_b200 import build
    exe = build.build_cpp_program(ROOT / "tests" / "cpp" / "mesh_export.cpp", ROOT / "tests" / "cpp" / "_build" / "mesh_export")
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "all checks passed" in r.stdout
    k = kf.KinFu.from_snapshot(tmp_path / "mesh_export.dfsnap")
    for live, name in ((False, "canonical.ply"), (True, "live.ply")):
        k.save_mesh(tmp_path / ("py_" + name), live=live)
        cv, cf = _read_ply(tmp_path / name)
        pv, pf = _read_ply(tmp_path / ("py_" + name))
        assert len(cf) > 1000
        assert cv.tobytes() == pv.tobytes() and np.array_equal(cf, pf)
        assert (tmp_path / name).read_bytes() == (tmp_path / ("py_" + name)).read_bytes()
    k.close()
