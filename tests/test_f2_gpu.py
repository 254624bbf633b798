"""GPU parity of df_solve_f2 (SURVEY 8f(2): robust data term over 6-DoF node increments + regulariser, csrc/regsolve.cu) against
its oracle restatement (oracle/orc_reg.c).  PARITY UNPINNED by the reference (no reference code evaluates this energy): the oracle is
pinned by tests/test_f2_oracle.py, the CUDA solver is compared with the oracle here.  The oracle solves every Gauss-Newton system
exactly (dense Cholesky); the CUDA solver runs block-Jacobi PCG to 1e-12 of the initial residual, so energies agree to ~1e-6 relative and
node parameters to ~1e-4 of their scale (the rotation Jacobians are kept in float on the device)."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from dynamicfusion_b200 import host  # noqa: E402
from scenes import node_patch, rot_y  # noqa: E402


def _run_both(orc, node_pts, src, dst, weight, **kw):
    ref_nodes = orc.make_nodes(node_pts, weight=weight)
    ost = orc.solve_f2(ref_nodes, src, dst, orc.f2_params(**kw))
    wf = host.WarpField()
    wf.setNodes(torch.from_numpy(orc.make_nodes(node_pts, weight=weight)).cuda())
    gst = wf.optimiseWarpF2(torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda(), **kw).cpu().numpy()
    return ost, gst, ref_nodes, wf.nodes_.cpu().numpy()


@pytest.mark.parametrize("flags,lam", [(0, 0.0), (1, 0.0), (1, 2.0), (1 | 4, 2.0), (1 | 2, 0.0), (7, 5.0)])
def test_f2_matches_oracle(orc, flags, lam):
    rng = np.random.default_rng(17 + flags)
    node_pts, src = node_patch(rng, 6000)
    dst = src.copy()
    dst[:, :3] = (src[:, :3] @ rot_y(3.0).T + np.array([0.008, -0.002, 0.004])).astype(np.float32)
    dst[:, 2] += (0.004 * np.sin(9 * src[:, 1])).astype(np.float32)
    out = rng.choice(len(src), len(src) // 20, replace=False)
    dst[out, :3] += rng.uniform(0.05, 0.2, (len(out), 3)).astype(np.float32)
    src[::97, 0] = np.nan
    dst[::131, 1] = np.nan
    ost, gst, rn, gn = _run_both(orc, node_pts, src, dst, 0.08, reg_lambda=lam, flags=flags, gn_iters=4, tukey_c=0.05, huber_delta=1e-3,
                                 reg_k=4, lin_iters=400)
    assert gst[3] == ost[3] and gst[2] == ost[2] == 4
    assert gst[6] == ost[6] or lam == 0.0
    for i in range(5):
        assert abs(gst[8 + i] - ost[8 + i]) <= 2e-5 * max(ost[8 + i], 1e-12) + 1e-10, (i, gst[8 + i], ost[8 + i])
    assert abs(gst[1] - ost[1]) <= 2e-5 * ost[1] + 1e-10 and gst[1] < gst[0]
    assert abs(gst[4] - ost[4]) <= 2e-5 * ost[1] + 1e-10 and abs(gst[5] - ost[5]) <= 2e-5 * ost[1] + 1e-10
    tg, tr = orc.node_translations(gn)[:, 1:], orc.node_translations(rn)[:, 1:]
    assert np.abs(tg - tr).max() <= 2e-3 * np.abs(tr).max()
    dq = np.minimum(np.abs(gn[:, 3:7] - rn[:, 3:7]).max(), np.abs(gn[:, 3:7] + rn[:, 3:7]).max())
    assert dq <= 2e-4
    if not (flags & 1):
        assert np.array_equal(gn[:, 3:7], orc.make_nodes(node_pts)[:, 3:7])      # translation-only: rotations untouched


def test_f2_full_size_properties():
    """bench-sized problem (2k nodes, 300k vertices): no oracle (dense 12k x 12k), size-independent properties instead -- the energy never
    increases over the Gauss-Newton steps, the PCG converges, twist beats translation-only on a rotating scene"""
    rng = np.random.default_rng(2)
    M, N = 2000, 300_000
    node_pts = np.stack([rng.uniform(-0.4, 0.4, M), rng.uniform(-0.3, 0.3, M), 1.0 + 0.05 * rng.standard_normal(M)], 1).astype(np.float32)
    src = np.zeros((N, 4), np.float32)
    src[:, 0] = rng.uniform(-0.4, 0.4, N); src[:, 1] = rng.uniform(-0.3, 0.3, N); src[:, 2] = 1.0 + 0.03 * np.sin(7 * src[:, 0])
    dst = src.copy()
    dst[:, :3] = (src[:, :3] @ rot_y(2.0).T + np.array([0.004, 0.0, 0.002])).astype(np.float32)
    e = {}
    for flags in (0, 7):
        n = np.zeros((M, 12), np.float32); n[:, :3] = node_pts; n[:, 3] = 1; n[:, 7] = 1; n[:, 11] = 0.05
        wf = host.WarpField()
        wf.setNodes(torch.from_numpy(n).cuda())
        st = wf.optimiseWarpF2(torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda(), reg_lambda=1.0 if flags else 0.0, flags=flags,
                               gn_iters=3, tukey_c=0.05, huber_delta=1e-3, lin_iters=60).cpu().numpy()
        assert st[3] == N and np.all(np.isfinite(st))
        assert st[9] <= st[8] and st[10] <= st[9] * 1.001 and st[1] <= st[10] * 1.001
        assert np.all(np.isfinite(wf.nodes_.cpu().numpy()))
        w, nr = torch.from_numpy(src.copy()).cuda(), torch.zeros((N, 4), device="cuda")
        nr[:, 2] = 1
        wf.warp(w, nr)                                                # the pipeline's own DQB warp applies the solved field
        e[flags] = float((w[:, :3] - torch.from_numpy(dst[:, :3]).cuda()).abs().mean().item())
    assert e[7] < 0.5 * e[0]
