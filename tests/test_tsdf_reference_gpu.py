"""The rigid TSDF stage on the GPU against the C oracle (bit for bit) and the float64 reference (tsdf_reference.py), on non-cubic volumes
with anisotropic voxels on both sides of every integrate dispatch, and on ragged frames at dense and padded pitches.  Every entry is
called through capi with explicit pitches.  Per case the largest |GPU - f64| / bar and the ambiguous fractions are printed."""
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("orc")]

import gpu_util as gu  # noqa: E402
import tsdf_cases as tc  # noqa: E402
import tsdf_reference as tr  # noqa: E402
from dynamicfusion_b200 import capi  # noqa: E402

AMB_MAX = 1e-3
CAPACITY = 1 << 20


def _lib():
    return capi.load()


class Vol:
    """a device volume of tsdf_cases' shape `name`, with its activity map when tracked"""

    def __init__(self, name, tracked):
        self.name = name
        self.dims, _ = tc.VOLUMES[name]
        self.vs, self.trunc = tc.voxel_size(name), tc.trunc_dist(name)
        self.data = torch.zeros(int(np.prod(self.dims)), dtype=torch.int32, device="cuda")
        self.act = None
        if tracked:
            self.act = torch.zeros(int(_lib().df_volume_activity_bytes(self.v())), dtype=torch.uint8, device="cuda")

    def v(self):
        return capi.make_volume(self.data.data_ptr(), self.dims, self.vs, self.trunc, tc.MAX_W)

    def words(self):
        torch.cuda.synchronize()
        return self.data.cpu().numpy().view(np.uint32).copy()


def _dists(depth, K, pad):
    """df_compute_dists on a depth image and into a distance image, both with `pad` bytes past each row: (device image, pitch, host)"""
    rows, cols = depth.shape
    d_dev, pitch, _ = gu.padded(depth, pad // 2, 7)
    out, opitch, _ = gu.padded(np.zeros_like(depth), pad // 2, 0)
    capi.check(_lib().df_compute_dists(d_dev.data_ptr(), pitch, cols, rows, capi.make_intr(*K), out.data_ptr(), opitch, gu.stream()))
    host = gu.host(out, np.uint16, (rows, cols + pad // 2))
    assert np.all(host[:, cols:] == 0)                                  # nothing written past the row
    return out, opitch, np.ascontiguousarray(host[:, :cols])


def _integrate(vol, dists, pitch, cols, rows, v2c, K):
    n = torch.zeros(1, dtype=torch.int64, device="cuda")
    capi.check(_lib().df_integrate_tracked(vol.v(), dists.data_ptr(), pitch, cols, rows, capi.make_aff(*v2c), capi.make_intr(*K), n.data_ptr(),
                                           vol.act.data_ptr() if vol.act is not None else None, None, gu.stream()))
    torch.cuda.synchronize()
    return int(n.item()), int(_lib().df_integrate_last_kernel())


def _run(name, pose_kind, K, cols, rows, pad=0, tracked=False):
    """three frames into a fresh volume: (volume, [(prev words, words, host dists, vol2cam, n_updated, kernel, pitch, depth)])"""
    vol = Vol(name, tracked)
    frames = []
    prev = vol.words()
    for f in range(3):
        depth = tc.scene_depth(name, pose_kind, cols, rows, K, f)
        d, pitch, dh = _dists(depth, K, pad)
        v2c = tc.vol2cam(name, pose_kind, f)
        n, kern = _integrate(vol, d, pitch, cols, rows, v2c, K)
        now = vol.words()
        frames.append((prev, now, dh, v2c, n, kern, pitch, depth))
        prev = now
    return vol, frames


def _raycast(vol, c2v, K, cols, rows, dense, pad_px=32):
    """points and normals (rows, cols, 4) from maps whose rows are pad_px float4 longer than the image"""
    Rinv = np.linalg.inv(c2v[0].astype(np.float64)).astype(np.float32)
    pc = cols + pad_px
    P = torch.full((rows, pc, 4), 7.0, dtype=torch.float32, device="cuda")
    N = torch.full((rows, pc, 4), 7.0, dtype=torch.float32, device="cuda")
    args = (vol.v(), capi.make_aff(*c2v), capi.f9(Rinv), capi.make_intr(*K), cols, rows, tc.STEP_FACTOR, tc.DELTA_FACTOR,
            P.data_ptr(), pc * 16, N.data_ptr(), pc * 16)
    if dense:
        capi.check(_lib().df_raycast_points(*args, gu.stream()))
    else:
        capi.check(_lib().df_raycast_points_tracked(*args, vol.act.data_ptr(), gu.stream()))
    P, N = P.cpu().numpy(), N.cpu().numpy()
    assert np.all(P[:, cols:] == 7.0) and np.all(N[:, cols:] == 7.0)
    return np.ascontiguousarray(P[:, :cols]), np.ascontiguousarray(N[:, :cols]), Rinv


def _extract(vol, pose, tracked):
    ws = torch.empty(int(_lib().df_extract_workspace_bytes(vol.v())), dtype=torch.uint8, device="cuda")
    out = torch.full((CAPACITY, 4), 7.0, dtype=torch.float32, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    capi.check(_lib().df_extract_cloud_tracked(vol.v(), capi.make_aff(*pose), out.data_ptr(), CAPACITY, cnt.data_ptr(), ws.data_ptr(),
                                               vol.act.data_ptr() if tracked else None, gu.stream()))
    n = int(cnt.item())
    assert n < CAPACITY
    return out[:n].cpu().numpy()


def _normals(vol, cloud, pose):
    Rinv = np.linalg.inv(pose[0].astype(np.float64)).astype(np.float32)
    pts = torch.from_numpy(np.ascontiguousarray(cloud)).cuda()
    out = torch.empty((max(len(cloud), 1), 4), dtype=torch.float32, device="cuda")
    capi.check(_lib().df_extract_normals(vol.v(), pts.data_ptr(), len(cloud), None, capi.make_aff(*pose), capi.f9(Rinv), tc.DELTA_FACTOR,
                                         out.data_ptr(), gu.stream()))
    return out[:len(cloud)].cpu().numpy(), Rinv


def _check_frames(orc, name, K, cols, rows, frames, report):
    """every frame: the kernel that ran, the oracle bit for bit, the float64 bars and n_updated's bracket"""
    dims = tc.VOLUMES[name][0]
    vs, trunc = tc.voxel_size(name), tc.trunc_dist(name)
    nvox = int(np.prod(dims))
    for f, (prev, now, dh, v2c, n, kern, pitch, depth) in enumerate(frames):
        want = tr.integrate_kernel_for(dims, 5, K, v2c, vs, trunc, cols, rows, pitch)[0]
        assert kern == want, (f, kern, want)
        assert np.array_equal(dh, orc.compute_dists(depth, K))
        _, h64, damb = tr.dists64(depth, K)
        assert np.array_equal(dh[~damb], h64[~damb])
        ref = prev.copy()
        n_orc = orc.integrate(ref, dims, vs, trunc, tc.MAX_W, dh, v2c, K)
        assert n == n_orc and np.array_equal(now, ref), f"frame {f}: {np.count_nonzero(now != ref)} voxels differ from the oracle"
        r = tr.integrate64(prev, dims, vs, trunc, tc.MAX_W, dh, v2c, K)
        bad, ratio, nupd, namb = tr.integrate_check(prev, now, r)
        assert bad == 0, f"frame {f}: {bad} voxels outside the float64 bars"
        assert nupd <= n <= nupd + namb
        # a voxel is ambiguous near a pixel edge: their density, and with it the ambiguous fraction, grows with the focal length in pixels
        assert namb / nvox < AMB_MAX * max(1.0, cols / 640), namb / nvox
        report["int_ratio"] = max(report.get("int_ratio", 0.0), ratio)
        report["int_amb"] = max(report.get("int_amb", 0.0), namb / nvox)
        report["kernel"] = kern


def _print(case, report):
    print("\n[tsdf-f64] " + case + " " + json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in report.items()}), flush=True)


@pytest.mark.parametrize("case", tc.VOLUME_CASES, ids=lambda c: f"{c[0]}-{c[1]}")
def test_volume_matches_oracle_and_float64(orc, case):
    name, pose_kind, K, view = case
    dims = tc.VOLUMES[name][0]
    vs, trunc = tc.voxel_size(name), tc.trunc_dist(name)
    vol, frames = _run(name, pose_kind, K, 640, 480, tracked=True)
    plain, pframes = _run(name, pose_kind, K, 640, 480, tracked=False)
    assert np.array_equal(vol.words(), plain.words())                   # the activity marks change nothing in the volume
    report = {}
    _check_frames(orc, name, K, 640, 480, frames, report)
    words = frames[-1][1]

    # ray-cast: brick-skipping march == dense march == oracle, both against the float64 reference
    c2v = tc.cam2vol(name, pose_kind, view)
    pt, nt, Rinv = _raycast(vol, c2v, K, 640, 480, dense=False)
    pd, nd, _ = _raycast(vol, c2v, K, 640, 480, dense=True)
    assert np.array_equal(pt.view(np.uint32), pd.view(np.uint32)) and np.array_equal(nt.view(np.uint32), nd.view(np.uint32))
    rp, rn, _ = orc.raycast_points(words, dims, vs, trunc, tc.MAX_W, c2v, Rinv, K, 640, 480, tc.STEP_FACTOR, tc.DELTA_FACTOR)
    assert gu.same_bits(pd, rp) and gu.same_bits(nd, rn)
    ref = tr.raycast64(words, dims, vs, trunc, c2v, Rinv, K, 640, 480, tc.STEP_FACTOR, tc.DELTA_FACTOR)
    bad, rv, rnv, nhit, namb = tr.raycast_check(pd, nd, ref)
    assert bad == 0, f"{bad} rays outside the float64 bars"
    assert namb / ref["pix"].size < AMB_MAX, namb / ref["pix"].size
    report.update(rc_hits=nhit, rc_vertex=rv, rc_normal=rnv, rc_amb=namb / ref["pix"].size)

    # extraction: tracked == full scan == oracle; the point set and order exact against the float64 crossing rule, coordinates in bars
    pose = tc.f32(tc.volume_pose(name, pose_kind))
    full, trk = _extract(vol, pose, False), _extract(vol, pose, True)
    assert np.array_equal(full.view(np.uint32), trk.view(np.uint32))
    assert np.array_equal(full.view(np.uint32), orc.extract_cloud(words, dims, vs, trunc, tc.MAX_W, pose, CAPACITY).view(np.uint32))
    P, B, _, _ = tr.extract64(words, dims, vs, pose)
    assert len(full) == len(P) > 500
    ratio = np.abs(full[:, :3] - P) / B
    assert np.all(ratio <= 1.0)
    nrm, Rp = _normals(vol, full, pose)
    assert gu.same_bits(nrm, orc.extract_normals(words, dims, vs, trunc, tc.MAX_W, full, pose, Rp, tc.DELTA_FACTOR))
    N, NB, namb_n = tr.normals64(words, dims, vs, full, pose, Rp, tc.DELTA_FACTOR)
    assert np.array_equal(np.isnan(nrm[~namb_n, 0]), np.isnan(N[~namb_n, 0]))
    m = ~namb_n & ~np.isnan(N[:, 0])
    nratio = np.abs(nrm[m, :3] - N[m]) / NB[m]
    assert m.sum() > 0.3 * len(full) and np.all(nratio <= 1.0)
    report.update(points=len(full), ex_ratio=float(ratio.max()), nrm_ratio=float(nratio.max()), nrm_amb=float(namb_n.mean()))
    _print(f"{name}-{pose_kind}", report)


def _raycast_rows(rows):
    """the rows the float64 ray-cast checks: all of a small frame, every 4th of a larger one"""
    return np.arange(rows) if rows <= 240 else np.arange(0, rows, 4)


@pytest.mark.parametrize("case", tc.FRAME_CASES, ids=lambda c: f"{c[0]}-{c[1][0]}x{c[1][1]}")
def test_frame_sizes_and_pitches(orc, case):
    name, (cols, rows) = case
    K = tc.frame_K(cols, rows)
    pose_kind = "tilted"
    runs = [_run(name, pose_kind, K, cols, rows, pad=pad) for pad in tc.PITCH_PAD]
    for _, frames in runs[1:]:                                          # padded pitches: the dense result bit for bit
        for (_, a, da, *_), (_, b, db, *_) in zip(runs[0][1], frames):
            assert np.array_equal(da, db) and np.array_equal(a, b)
    report = {}
    _check_frames(orc, name, K, cols, rows, runs[0][1], report)
    vol = runs[0][0]
    words = runs[0][1][-1][1]
    c2v = tc.cam2vol(name, pose_kind, pose_kind)
    dims = tc.VOLUMES[name][0]
    p0, n0, Rinv = _raycast(vol, c2v, K, cols, rows, dense=True, pad_px=0)
    p1, n1, _ = _raycast(vol, c2v, K, cols, rows, dense=True, pad_px=32)
    assert np.array_equal(p0.view(np.uint32), p1.view(np.uint32)) and np.array_equal(n0.view(np.uint32), n1.view(np.uint32))
    pix = (_raycast_rows(rows)[:, None] * cols + np.arange(cols)[None, :]).ravel()
    ref = tr.raycast64(words, dims, tc.voxel_size(name), tc.trunc_dist(name), c2v, Rinv, K, cols, rows, tc.STEP_FACTOR, tc.DELTA_FACTOR, pix)
    bad, rv, rnv, nhit, namb = tr.raycast_check(p0, n0, ref)
    assert bad == 0, f"{bad} rays outside the float64 bars"
    assert cols * rows < 1000 or namb / len(pix) < AMB_MAX
    report.update(rc_hits=nhit, rc_vertex=rv, rc_normal=rnv, rc_amb=namb / len(pix))
    _print(f"{name}-{cols}x{rows}", report)


# ------------------------------------------------------------------ every integrate implementation, and PDL off ---------------------------
def output_digests():
    """sha256 of every case's outputs (volumes after each frame, activity map, both ray-casts, both extractions and the normals) with the
    integrate kernel that ran: what DF_INTEGRATE_IMPL must not change in the volumes, and DF_PDL in anything"""
    out = {}
    for name, pose_kind, K, view in tc.VOLUME_CASES:
        vol, frames = _run(name, pose_kind, K, 640, 480, tracked=True)
        h = hashlib.sha256(b"".join(f[1].tobytes() for f in frames) + vol.act.cpu().numpy().tobytes())
        c2v = tc.cam2vol(name, pose_kind, view)
        pose = tc.f32(tc.volume_pose(name, pose_kind))
        cloud = _extract(vol, pose, True)
        g = hashlib.sha256(b"".join(a.tobytes() for a in _raycast(vol, c2v, K, 640, 480, dense=False)[:2] + _raycast(vol, c2v, K, 640, 480, dense=True)[:2])
                           + cloud.tobytes() + _extract(vol, pose, False).tobytes() + _normals(vol, cloud, pose)[0].tobytes())
        out[f"{name}-{pose_kind}"] = [h.hexdigest(), frames[-1][5], g.hexdigest()]
    for name, (cols, rows) in tc.FRAME_CASES:
        vol, frames = _run(name, "tilted", tc.frame_K(cols, rows), cols, rows, pad=2)
        out[f"{name}-{cols}x{rows}"] = [hashlib.sha256(b"".join(f[1].tobytes() + f[2].tobytes() for f in frames)).hexdigest(), frames[-1][5], ""]
    return out


def _digests_in_subprocess(env):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = "import sys, json; sys.path[:0] = ['tests', '.']; import test_tsdf_reference_gpu as t; print(json.dumps(t.output_digests()))"
    r = subprocess.run([sys.executable, "-c", code], cwd=root, env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.fixture(scope="module")
def digests():
    return output_digests()


@pytest.mark.parametrize("impl", ["1", "3"])
def test_integrate_implementations_agree_in_subprocess(impl, digests):
    """DF_INTEGRATE_IMPL is read once per process: 1 (plain) and 3 (scalar with culling) store the default's volumes and activity maps after
    every frame bit for bit, and launch the kernel the predictor names for them"""
    there = _digests_in_subprocess({"DF_INTEGRATE_IMPL": impl})
    assert {k: v[0] for k, v in there.items()} == {k: v[0] for k, v in digests.items()}
    for k, (_, kern, _) in there.items():
        assert kern == (0 if impl == "1" else (3 if digests[k][1] == 5 else digests[k][1])), (k, kern)


def test_pdl_off_in_subprocess(digests):
    """DF_PDL is read once per process: with it off, every output of every case -- the volumes after each frame, the distance images, the
    activity maps, both ray-casts, both extractions and the normals -- equals bit for bit what the tests above checked against the oracle and
    the float64 reference"""
    assert _digests_in_subprocess({"DF_PDL": "0"}) == digests
