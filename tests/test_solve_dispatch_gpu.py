"""The data-term solve on every LM kernel and assembly path the problem size selects, against the float64 least-squares reference.

solve_data_term_ev picks the LM kernel from the node count M and the cluster size the part runs (solve_cases.lm_path restates the rule);
stats[7] says which one ran.  Each case of solve_cases.py is solved through WarpField.optimiseWarpData, then checked against
tests/solve_reference.py: the neighbours (cKDTree), the assembled normal system read back with df_solve_normal_system, the costs the LM
reports, the distance of the result from the float64 minimum (bars calibrated on the CPU oracle, tests/test_solve_float64.py) and the
parts of the nodes the solve must not touch.  The last test re-runs the file under the switches that select the other kernels."""
import ctypes as C
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import solve_cases as sc  # noqa: E402
from dynamicfusion_b200 import capi, host  # noqa: E402
from solve_reference import Problem, decode_bound, ell_compare, knn8_check, node_translations, rel_gap  # noqa: E402

IMPL = int(os.environ.get("DF_SOLVE_LM_IMPL", "6"))
WANT_CTAS = int(os.environ.get("DF_SOLVE_LM_CTAS", "16"))
FORCE_FALLBACK = int(os.environ.get("DF_SOLVE_V6_FORCE_FALLBACK", "0")) != 0
ROWCAP = 512                                            # ELL slots per row (dfusion.h, df_solve_normal_system)
_RUNS = {}


def _grab(ws, ptr, count, dtype):
    """`count` elements at device pointer `ptr` inside the workspace tensor, copied to the host"""
    off = ptr.value - ws.data_ptr()
    nbytes = count * torch.empty(0, dtype=dtype).element_size()
    assert 0 <= off and off + nbytes <= ws.numel()
    return ws[off:off + nbytes].view(dtype).cpu().numpy()


def _solve(name):
    if name in _RUNS:
        return _RUNS[name]
    case = sc.make_case(name)
    M, N = case["M"], case["N"]
    wf = host.WarpField(use_grid=case["use_grid"])
    wf.setNodes(torch.from_numpy(case["nodes"].copy()).cuda())
    canon, live = torch.from_numpy(case["canon"]).cuda(), torch.from_numpy(case["live"]).cuda()
    stats = wf.optimiseWarpData(canon, live, sc.LM_ITERS, sc.LIN_ITERS, case["flags"]).cpu().numpy()
    out = wf.nodes_.cpu().numpy()
    lib, ws = capi.load(), wf._ws
    p = [C.c_void_p() for _ in range(5)]
    capi.check(lib.df_solve_normal_system(ws.data_ptr(), M, N, *[C.byref(q) for q in p]))
    system = (_grab(ws, p[0], M, torch.int32), _grab(ws, p[1], M * ROWCAP, torch.int32), _grab(ws, p[2], M * ROWCAP, torch.float64),
              _grab(ws, p[3], 3 * M, torch.float64), _grab(ws, p[4], M, torch.float64))
    pi, pw = C.c_void_p(), C.c_void_p()
    capi.check(lib.df_solve_knn_buffers(ws.data_ptr(), M, N, C.byref(pi), C.byref(pw)))
    knn = _grab(ws, pi, N * 8, torch.int32).reshape(N, 8), _grab(ws, pw, N * 8, torch.float32).reshape(N, 8)
    _RUNS[name] = (case, stats, out, system, knn)
    return _RUNS[name]


@pytest.fixture(scope="module")
def cluster():
    """the largest cluster this part runs, inferred from M = 4097: v5 on 16 CTAs where 16-CTA clusters fit, the one-block kernel on 8.
    None where the switches leave no cluster kernel to tell it by (every size then takes the same path whatever the part)."""
    if IMPL < 5 or WANT_CTAS != 16:
        return None
    _, stats, *_ = _solve("m4097-image")
    kernel, _ = sc.kernel_of(stats[7])
    size = 16 if kernel == "v5" else 8
    print(f"\n[solve dispatch] 16-CTA clusters {'available' if size == 16 else 'not available'}: cluster size {size}")
    return size


def test_path_predictor_restates_the_size_bounds():
    """the bounds the predictor is built from: 24 M + 40960 <= 216 KiB (16 CTAs), ceil(M / 8) <= 512 (8 CTAs), v6 up to 4096 nodes"""
    assert sc.lm_path(7509, 16) == ("v5", 16) and sc.lm_path(7510, 16) == ("one-block", 16)
    assert sc.lm_path(4096, 8) == ("v6", 8) and sc.lm_path(4097, 8) == ("one-block", 8)
    assert sc.lm_path(4096, 16) == ("v6", 16) and sc.lm_path(4097, 16) == ("v5", 16)
    assert sc.lm_path(255, 16) == ("v6", 8) and sc.lm_path(256, 16) == ("v6", 16)
    assert sc.lm_path(2000, 16, impl=1)[0] == "one-block" and sc.lm_path(2000, 16, impl=5)[0] == "v5"
    assert sc.lm_path(2000, 16, force_fallback=True)[0] == "v5" and sc.lm_path(300, 16, want_ctas=8) == ("v6", 8)
    # the rows of the large systems stream from L2: ~30 entries per row against these per-lane capacities
    assert sc.lm_entry_cap(4096, "v6", 16) == 8 and sc.lm_entry_cap(4096, "v6", 8) == 7 and sc.lm_entry_cap(7000, "v5", 16) == 10


@pytest.mark.parametrize("name", sc.case_names())
def test_solve_matches_float64_reference(name, cluster):
    """m7000 runs v5 with ent_cap = (216 KiB - 24 * 7000 - 16) / (512 * 10) = 10 entries per lane in shared memory; with
    ceil(7000 / 16) = 438 rows per CTA a row has one lane (tpr = 1) and its ~30 entries, so ~20 of them come from L2 in every mat-vec.
    m4096 runs v6 with cap6 = 8 (16 CTAs, 2 lanes per row) or 7 (8 CTAs, 1 lane per row): the same streamed tail."""
    case, stats, out, (rownnz, col, val, gb, diag), (idx, w) = _solve(name)
    M, nodes_in = case["M"], case["nodes"]
    assert not np.isnan(stats).any() and not np.isnan(out).any(), stats
    assert stats[5] == 0, "no row of these systems exceeds the row capacity"

    # which LM kernel, and which assembly
    kernel, tiles = sc.kernel_of(stats[7])
    want, ncta = sc.lm_path(M, cluster, IMPL, WANT_CTAS, FORCE_FALLBACK)
    if name == "scattered" and want == "v6":
        want = "v5"                                     # its halo / send lists do not fit: v6 hands the solve to v5
    assert kernel == want, (name, stats[7], want, ncta)
    if name == "coherent" and want == "v6":
        assert stats[7] >= 0
    assert tiles == (case["flags"] != 0), (name, stats[7])

    # the neighbours against an independent 8-NN, then the system against the float64 one built from them
    fails, compared = knn8_check(nodes_in, case["canon"], idx, w)
    assert not fails, fails[:10]
    prob = Problem(M, idx, w, case["canon"], case["live"])
    assert stats[3] == prob.nvalid
    assert stats[6] == rownnz.sum()
    if tiles:
        assert stats[6] <= prob.nnz
    else:
        assert stats[6] == prob.nnz
    fails = ell_compare(prob, rownnz, col, val, gb, diag, tiles)
    assert not fails, fails

    # the costs the LM reports are the energy at its start and at the nodes it wrote
    x0, x = node_translations(nodes_in), node_translations(out)
    e0 = prob.energy(x0)
    assert abs(stats[0] - e0) <= 1e-10 * e0 + decode_bound(prob, x0), (stats[0], e0)
    ex = prob.energy(x)
    assert abs(stats[1] - ex) <= 1e-9 * e0 + 2 * decode_bound(prob, x), (stats[1], ex, e0)

    # how close to the float64 minimum, against the calibrated bars
    if prob.supported.any():
        xmin = prob.minimiser(x0)
        gap = rel_gap(prob, x, x0, xmin)
        assert gap <= sc.gap_bar(name, prob, x, x0, xmin), (gap, sc.ORACLE[name])
        if case["t_true"] is not None:
            s, t = prob.supported, case["t_true"]
            terr = float(np.sqrt(((x[s] - t[s]) ** 2).sum(1).mean() / (t[s] ** 2).sum(1).mean()))
            assert terr <= sc.t_bar(name), (terr, sc.ORACLE[name])

    # what the solve must not touch: positions, rotations and radii of every node; all of a node no valid row references.  The kernels write
    # every node back, re-encoding an unreferenced one from its own translation: bit for bit from the canonical encoding of a zero
    # translation (dual +0), to a float32 rounding from a rotated, translated start
    keep = [0, 1, 2, 3, 4, 5, 6, 11]
    assert np.array_equal(out[:, keep].view(np.uint32), nodes_in[:, keep].view(np.uint32))
    free = ~prob.referenced
    if not np.any(x0[free]):
        assert np.array_equal(out[free].view(np.uint32), nodes_in[free].view(np.uint32))
    else:
        assert np.all(np.abs(x[free] - x0[free]) <= 2.0 ** -20 * np.abs(x0[free]).max(1, keepdims=True))


def test_all_invalid_and_stride3_cases_are_what_they_claim():
    case = sc.make_case("all-invalid")
    assert np.isnan(case["canon"][:, 0]).all()
    assert sc.make_case("stride3")["canon"].shape[1] == 3
    w = sc.make_case("warm")["nodes"]
    assert np.abs(node_translations(w)).max() > 0.005 and np.abs(w[:, 4:7]).max() > 0.1


@pytest.mark.parametrize("env", [{"DF_SOLVE_LM_IMPL": "5"}, {"DF_SOLVE_LM_IMPL": "1"}, {"DF_SOLVE_V6_FORCE_FALLBACK": "1"},
                                 {"DF_SOLVE_LM_CTAS": "8"}], ids=["v5", "one-block", "v6-fallback", "ctas8"])
def test_other_lm_kernels_in_subprocess(env):
    """Each switch is read once per process: the whole file again in a fresh interpreter, every kernel held to the same float64 bars."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_solve_dispatch_gpu.py", "-q", "-s", "-m", "gpu", "-k", "not subprocess"],
                       cwd=root, env=dict(os.environ, **env), capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and "failed" not in r.stdout
