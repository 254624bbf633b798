"""The warp side on the GPU against the float64 reference (warp_reference.py), and warped fusion also against the C oracle, on the shapes of
warp_cases.py, through capi with explicit pitches: df_knn8 on the exhaustive scan (node counts across 1024-node tiles) and the grid walk;
df_warp with a non-identity warp_to_live under every flag; df_integrate_warped on every case, with the switches and pitches that must not
change a bit.  Per case the largest |GPU - f64| / bar, the ambiguous fractions, the search path and the wall time are printed."""
import hashlib
import json
import os
import time

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("orc")]

import gpu_util as gu  # noqa: E402
import warp_cases as wc  # noqa: E402
import warp_reference as wr  # noqa: E402
from dynamicfusion_b200 import capi  # noqa: E402

AMB_MAX = 1e-3
AMB_VOXELS = 1e-2                   # voxels: a 1.2 k-node cluster puts up to 0.7 % of them near a neighbour-set decision
W2L = wc.f32(wc.W2L)
REF_NORMAL_INDEX, ROTATE_ONLY, REUSE_KNN = 1, 2, 4


def _lib():
    return capi.load()


def _print(tag, report):
    print(f"\n[warp-f64] {tag} " + json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in report.items()}), flush=True)


def _grid(nodes_t):
    M = nodes_t.shape[0]
    g = torch.empty(int(_lib().df_node_grid_bytes(M)), dtype=torch.uint8, device="cuda")
    capi.check(_lib().df_build_node_grid(nodes_t.data_ptr(), M, g.data_ptr(), gu.stream()))
    return g


# ------------------------------------------------------------------ k-NN -------------------------------------------------------------------
@pytest.mark.parametrize("M", [5, 8, 1500, 3000])
def test_knn8_scan_and_grid_against_float64(orc, M):
    rng = np.random.default_rng(M + 1)
    nodes = wc.random_nodes(orc, M, M)
    q = wc.queries(rng, 20000)
    nt, qt = torch.from_numpy(nodes).cuda(), torch.from_numpy(q).cuda()
    grid = _grid(nt)
    out = []
    for g in (None, grid.data_ptr()):
        idx = torch.full((len(q), 8), -7, dtype=torch.int32, device="cuda")
        d2 = torch.full((len(q), 8), -7.0, dtype=torch.float32, device="cuda")
        capi.check(_lib().df_knn8(nt.data_ptr(), M, g, qt.data_ptr(), len(q), 4, idx.data_ptr(), d2.data_ptr(), gu.stream()))
        out.append((idx.cpu().numpy(), d2.cpu().numpy()))
    (i0, d0), (i1, d1) = out
    assert np.array_equal(i0, i1) and np.array_equal(d0.view(np.uint32), d1.view(np.uint32))
    ref = wr.knn64(nodes, wr.f64(q)[:, :3])
    assert np.all(wr.knn_admissible(ref, i0.astype(np.int64)))
    ok = i0 >= 0
    V = wr.f64(nodes)[:, :3]
    exact = ((wr.f64(q)[:, None, :3] - V[np.where(ok, i0, 0)]) ** 2).sum(-1)
    ratio = np.abs(d0[ok] - exact[ok]) / np.maximum(wr.KNN_MARGIN * wr.U * exact[ok], 1e-300)
    assert np.all(ratio <= 1.0)
    amb = float(1 - ref["forced"].mean())
    _print(f"knn M={M}", {"d2_ratio": float(ratio.max()), "amb": amb})
    assert amb < AMB_MAX


# ------------------------------------------------------------------ warp -------------------------------------------------------------------
def _warp(nodes_t, grid, pts, nrm, flags, idx=None, w=None, want=False):
    p, n = torch.from_numpy(pts).cuda(), torch.from_numpy(nrm).cuda()
    N = len(pts)
    if want:
        idx = torch.full((N, 8), -7, dtype=torch.int32, device="cuda")
        w = torch.full((N, 8), -7.0, dtype=torch.float32, device="cuda")
    capi.check(_lib().df_warp(nodes_t.data_ptr(), nodes_t.shape[0], grid.data_ptr(), p.data_ptr(), n.data_ptr(), N, 4, capi.make_aff(*W2L), flags,
                              idx.data_ptr() if idx is not None else None, w.data_ptr() if w is not None else None, gu.stream()))
    return p.cpu().numpy(), n.cpu().numpy(), idx, w


def _check_warp(nodes, pts, nrm, gp, gn, gidx, rotate_only, tag):
    """float64 bars on every point; where the exact neighbour set is not forced, the GPU's own set must be admissible and the warp is
    evaluated with it"""
    ref = wr.warp64(nodes, pts, nrm, W2L, rotate_only)
    knn = ref[5]
    gidx = gidx.astype(np.int64)
    assert np.all(wr.knn_admissible(knn, gidx)), tag
    bad, rp, rn, nchk = wr.warp_check(gp, gn, ref)
    loose = np.flatnonzero(~knn["forced"])
    if len(loose):
        alt = wr.warp64(nodes, pts[loose], nrm[loose], W2L, rotate_only, idx=gidx[loose])
        b2, rp2, rn2, _ = wr.warp_check(gp[loose], gn[loose], alt)
        bad, rp, rn = bad + b2, max(rp, rp2), max(rn, rn2)
    assert bad == 0, f"{tag}: {bad} values outside the float64 bars"
    amb = float(ref[4].mean())
    assert amb < AMB_MAX and nchk > 0.99 * len(pts)
    _print(tag, {"point_ratio": rp, "normal_ratio": rn, "knn_amb": float(1 - knn["forced"].mean()), "ill": amb})


def test_warp_flags_against_float64(orc):
    """df_warp with warp_to_live and flags 0, ROTATE_ONLY, REUSE_KNN (neighbours and weights of an earlier pass, rotated nodes),
    DF_WARP_IMAGE_COLS (8 x 4 pixel patches per warp) and REF_NORMAL_INDEX (the reference's normal cursor)"""
    rng = np.random.default_rng(11)
    nodes = wc.random_nodes(orc, 700, 5)
    nt = torch.from_numpy(nodes).cuda()
    grid = _grid(nt)
    cols, rows = 64, 40
    pts = wc.queries(rng, cols * rows)
    nrm = rng.normal(size=(cols * rows, 4)).astype(np.float32)
    nrm[:, :3] /= np.linalg.norm(nrm[:, :3], axis=1, keepdims=True)
    p0, n0, idx, w = _warp(nt, grid, pts, nrm, 0, want=True)
    gidx = idx.cpu().numpy()
    _check_warp(nodes, pts, nrm, p0, n0, gidx, False, "warp flags=0")
    p2, n2, _, _ = _warp(nt, grid, pts, nrm, ROTATE_ONLY)
    assert np.array_equal(p2.view(np.uint32), p0.view(np.uint32))
    _check_warp(nodes, pts, nrm, p2, n2, gidx, True, "warp ROTATE_ONLY")
    p4, n4, _, _ = _warp(nt, grid, pts, nrm, REUSE_KNN, idx=idx, w=w)
    assert np.array_equal(p4.view(np.uint32), p0.view(np.uint32)) and np.array_equal(n4.view(np.uint32), n0.view(np.uint32))
    pc, nc, _, _ = _warp(nt, grid, pts, nrm, (cols & 0xffff) << 8)
    assert np.array_equal(pc.view(np.uint32), p0.view(np.uint32)) and np.array_equal(nc.view(np.uint32), n0.view(np.uint32))
    # the reference's normal cursor: NaN points are skipped, the j-th valid point takes normal j, nothing moves past the first NaN normal
    pr, nr = pts.copy(), nrm.copy()
    pr[::13, 0] = np.nan
    nr[2000, 0] = np.nan
    gp, gn, _, _ = _warp(nt, grid, pr, nr, REF_NORMAL_INDEX)
    valid = np.flatnonzero(~np.isnan(pr[:, 0]))
    rank = np.arange(len(valid))
    moved = valid[rank < 2000]
    untouched = valid[rank >= 2000]
    assert np.array_equal(gp[untouched].view(np.uint32), pr[untouched].view(np.uint32))
    assert gu.same_bits(gn[2000:], nr[2000:])
    _check_warp(nodes, pr[moved], nr[:len(moved)], gp[moved], gn[:len(moved)], gidx[moved], False, "warp REF_NORMAL_INDEX")


# ------------------------------------------------------------------ warped fusion ------------------------------------------------------------
class Run:
    """one case through df_integrate_warped: the volume words and activity map after each pass and the kernel's counters"""

    def __init__(self, c, nodes, pad=0, env=None):
        self.c = c
        dims = c["dims"]
        nvox = int(np.prod(dims))
        nt = torch.from_numpy(nodes).cuda()
        grid = _grid(nt)
        data = torch.zeros(nvox, dtype=torch.int32, device="cuda")
        V = capi.make_volume(data.data_ptr(), dims, c["vs"], c["trunc"], c["maxw"])
        act = torch.zeros(int(_lib().df_volume_activity_bytes(V)), dtype=torch.uint8, device="cuda")
        capi.check(_lib().df_clear_volume(V, gu.stream()))
        self.words, self.counts, self.depths = [self._words(data)], [], []
        saved = {k: os.environ.get(k) for k in (env or {})}
        os.environ.update(env or {})
        try:
            for p in range(c["passes"]):
                depth = wc.case_depth(c, p)
                d_dev, pitch, _ = gu.padded(depth, pad // 2, 7)
                counters = torch.zeros(2, dtype=torch.int64, device="cuda")
                capi.check(_lib().df_integrate_warped(V, d_dev.data_ptr(), pitch, c["cols"], c["rows"], capi.make_aff(*c["pose_v"]),
                                                      capi.make_aff(*wc.case_world2cam(c, p)), capi.make_intr(*c["K"]), nt.data_ptr(), len(nodes),
                                                      grid.data_ptr(), float(c["ws"]), counters.data_ptr(), act.data_ptr(), None, gu.stream()))
                self.words.append(self._words(data))
                self.counts.append([int(v) for v in counters.cpu().numpy()])
                self.depths.append(depth)
        finally:
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        self.act = act.cpu().numpy()

    @staticmethod
    def _words(data):
        torch.cuda.synchronize()
        return data.cpu().numpy().view(np.uint32).copy()

    def digest(self):
        h = hashlib.sha256(b"".join(w.tobytes() for w in self.words) + self.act.tobytes() + json.dumps([c[0] for c in self.counts]).encode())
        return h.hexdigest()


def _reference_voxels(c):
    """the voxels the float64 reference evaluates: all of them, or on the bench's volume every 16th z-slice"""
    if c["vol"] != "bench":
        return None
    Dx, Dy, Dz = c["dims"]
    z = np.arange(5, Dz, 16)
    return (z[:, None] * (Dx * Dy) + np.arange(Dx * Dy)[None, :]).ravel()


def _check_case(orc, c, nodes, run, report):
    dims = c["dims"]
    nvox = int(np.prod(dims))
    lin = _reference_voxels(c)
    t0 = time.time()
    warped = wr.warp_voxels(nodes, dims, c["vs"], c["pose_v"], lin)
    n_eval = len(warped["lin"])
    for p in range(c["passes"]):
        prev, now, depth = run.words[p], run.words[p + 1], run.depths[p]
        w2c = wc.case_world2cam(c, p)
        n = run.counts[p][0]
        # the oracle from the same previous volume: the existing 1e-5 budget
        ref = prev.copy()
        n_orc = orc.integrate_warped(ref, dims, c["vs"], c["trunc"], c["maxw"], depth, c["pose_v"], w2c, c["K"], nodes, c["ws"])
        mism = int(np.count_nonzero(now != ref))
        assert mism <= max(2, int(1e-5 * nvox)) and abs(n - n_orc) <= max(2, int(1e-5 * nvox)), (p, mism, n, n_orc)
        r = wr.integrate_warped64(prev, warped, depth, c["K"], w2c, c["trunc"], c["maxw"], c["ws"])
        bad, ratio, nupd, namb = wr.integrate_warped_check(prev, now, r)
        assert bad == 0, f"pass {p}: {bad} voxels outside the float64 bars"
        if lin is None:
            assert nupd <= n <= nupd + namb, (nupd, n, namb)
        assert namb / n_eval < AMB_VOXELS, namb / n_eval
        if p == 0 and c["id"] in wc.STRADDLE:
            # voxels of the runs straddling the camera plane that the frame updates for certain: the cull must have kept them
            keep = _straddle_voxels(c, warped["lin"])
            report["straddle_updated"] = int(r["upd"][keep].sum())
            assert report["straddle_updated"] >= 8, report["straddle_updated"]
        report["int_ratio"] = max(report.get("int_ratio", 0.0), ratio)
        report["amb"] = max(report.get("amb", 0.0), namb / n_eval)
        report["updated"] = report.get("updated", 0) + n
        report["oracle_differ"] = report.get("oracle_differ", 0) + mism
    report["knn_amb"] = float(1 - warped["forced"].mean())
    report["ref_s"] = round(time.time() - t0, 1)
    assert report["updated"] > 500
    words = run.words[-1]
    active = np.flatnonzero(((words >> 16) != 0) & ((words & 0xffff) != 0x3c00))
    assert np.all(run.act[active // 1024] == 1)
    if c["maxw"] == 8 and c["ws"] >= 400:
        assert ((words >> 16) == 8).sum() > 100                      # the weight clamps were reached


def _straddle_voxels(c, lin):
    """positions in lin of the voxels of the runs warp_reference.straddle_runs finds for pass 0"""
    runs = wr.straddle_runs(c["dims"], c["vs"], wc.case_vol2cam(c, 0), c["K"], c["cols"], c["rows"])
    assert runs, "no run straddles the camera plane with voxels in view"
    Dx, Dy, Dz = c["dims"]
    x, y, z = lin % Dx, (lin // Dx) % Dy, lin // (Dx * Dy)
    keep = np.zeros(len(lin), bool)
    for (x0, y0, z0), _ in runs:
        keep |= (x >= x0) & (x < x0 + 8) & (y >= y0) & (y < y0 + 4) & (z >= z0) & (z < z0 + 8)
    return keep


def _variants(c, nodes, base):
    """the switches and pitches that must not change a bit"""
    want = base.digest()
    for env in ({"DF_FUSION_CULL": "0"}, {"DF_FUSION_LIST": "0"}, {"DF_FUSION_ZCHUNK": "5"}, {"DF_FUSION_ZCHUNK": "12"}, {"DF_FUSION_ZCHUNK": "40"}):
        assert Run(c, nodes, env=env).digest() == want, env
    for pad in wc.PITCH_PAD[1:]:
        assert Run(c, nodes, pad=pad).digest() == want, pad


@pytest.mark.parametrize("cid", list(wc.CASES))
def test_integrate_warped_against_oracle_and_float64(orc, cid):
    t0 = time.time()
    c = wc.case(cid)
    nodes = wc.case_nodes(orc, c)
    sp = wr.search_path(nodes, c["dims"], c["vs"], c["pose_v"])
    assert wr.path_of(sp) == c["path"], (wr.path_of(sp), sp["list"], sp["tree"])
    run = Run(c, nodes)
    bn, rn = np.asarray(sp["block_n"]), np.asarray(sp["run_n"])
    report = {"path": c["path"], "list": round(sp["list"], 3), "block_max": int(bn.max()) if len(bn) else None,
              "run_max": int(rn.max()) if len(rn) else None}
    _check_case(orc, c, nodes, run, report)
    _variants(c, nodes, run)
    report["wall_s"] = round(time.time() - t0, 1)
    _print(cid, report)

