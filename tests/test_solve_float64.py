"""CPU: the float64 reference of the data-term solve (tests/solve_reference.py) pinned against the CPU oracle's matrix-free LM / PCG, and the
oracle's distance to the float64 optimum on every case of tests/test_solve_dispatch_gpu.py -- the numbers the GPU bars are set from."""
import numpy as np
import pytest

import solve_cases as sc
from solve_reference import Problem, decode_bound, ell_compare, knn8_check, node_translations, rel_gap


def _oracle_weights(orc, nodes, canon, live):
    """the oracle's neighbours and weights of the solve's rows (orc_solve_big.c: exp in double of the float32 squared distance)"""
    idx, d2 = orc.knn8(nodes, canon)
    r = nodes[np.maximum(idx, 0), 11].astype(np.float32)
    with np.errstate(over="ignore"):                     # empty slots (M < 8) carry a huge distance
        w = np.exp((-d2 / (np.float32(2) * r * r)).astype(np.float64)).astype(np.float32)
    w[idx < 0] = 0
    return idx, w


def oracle_solve(orc, case):
    """-> (Problem, x0, x_oracle, oracle stats) for one case"""
    from oracle import orc_pipe
    nodes = case["nodes"].copy()
    idx, w = _oracle_weights(orc, nodes, case["canon"], case["live"])
    prob = Problem(case["M"], idx, w, case["canon"], case["live"])
    x0 = node_translations(nodes)
    stats = orc_pipe.solve_data_term_big(nodes, case["canon"], case["live"], flags=0, lm_iters=sc.LM_ITERS, lin_iters=sc.LIN_ITERS)
    return prob, x0, node_translations(nodes), stats, nodes


def oracle_errors(prob, x0, x, t_true):
    """(share of the reducible energy left, RMS translation error of the supported nodes relative to RMS |t*| or None)"""
    xmin = prob.minimiser(x0)
    gap = rel_gap(prob, x, x0, xmin) if prob.supported.any() else 0.0
    terr = None
    if t_true is not None and prob.supported.any():
        s = prob.supported
        terr = float(np.sqrt(((x[s] - t_true[s]) ** 2).sum(1).mean() / (t_true[s] ** 2).sum(1).mean()))
    return gap, terr


@pytest.mark.parametrize("name", sc.case_names())
def test_reference_agrees_with_oracle_and_calibrates_the_bars(orc, name):
    case = sc.make_case(name)
    prob, x0, x, stats, _ = oracle_solve(orc, case)
    assert stats[3] == prob.nvalid
    e0 = prob.energy(x0)
    # the oracle's initial cost is the reference's energy at the starting translations
    assert abs(stats[0] - e0) <= 1e-10 * e0 + decode_bound(prob, x0) + 1e-300
    # and its final cost is the reference's energy at the translations it wrote back (float32 nodes)
    ex = prob.energy(x)
    assert abs(stats[1] - ex) <= 1e-9 * e0 + 2 * decode_bound(prob, x) + 1e-300, (stats[1], ex)
    # no solve gets below the float64 minimum
    xmin = prob.minimiser(x0)
    emin = prob.energy(xmin)
    assert ex >= emin - 1e-12 * e0 - decode_bound(prob, x)
    assert np.abs(prob.gradient(xmin)[prob.supported]).max(initial=0) <= 1e-9 * max(np.abs(prob.gb).max(initial=0), 1e-300)
    gap, terr = oracle_errors(prob, x0, x, case["t_true"])
    want_gap, want_t = sc.ORACLE[name]
    floor = sc.gap_floor(prob, x, x0, xmin)
    # the recorded numbers still describe the oracle (its OpenMP sums make the last bits vary from run to run: within 2x + rounding)
    assert gap <= 2 * want_gap + floor, f"oracle gap {gap:.3e}: re-measure ORACLE[{name!r}] in solve_cases.py"
    assert (terr is None) == (want_t is None)
    if terr is not None:
        assert want_t / 2 <= terr <= 2 * want_t, f"oracle translation error {terr:.3e}: re-measure ORACLE[{name!r}]"
    # the oracle meets the bars the kernels are held to
    assert gap <= sc.gap_bar(name, prob, x, x0, xmin)
    assert terr is None or terr <= sc.t_bar(name)


@pytest.mark.parametrize("name", ["bench-flat", "m5-image", "warm"])
def test_knn_check_accepts_the_oracle_neighbours_and_rejects_a_swap(orc, name):
    case = sc.make_case(name)
    idx, w = _oracle_weights(orc, case["nodes"], case["canon"], case["live"])
    fails, compared = knn8_check(case["nodes"], case["canon"], idx, w)
    assert not fails and compared > 0.9 * np.sum(~np.isnan(case["canon"][:, 1]))
    if case["M"] > 8:
        bad = idx.copy()
        v = int(np.flatnonzero(~np.isnan(case["canon"][:, 1]))[3])
        far = int(np.argmax(((case["nodes"][:, :3] - case["canon"][v, :3]) ** 2).sum(1)))
        bad[v, 7] = far
        assert any(f[0] == v for f in knn8_check(case["nodes"], case["canon"], bad, w)[0])
    w2 = w.copy()
    w2[np.flatnonzero(~np.isnan(case["canon"][:, 1]))[5], 0] += 1e-4
    assert knn8_check(case["nodes"], case["canon"], idx, w2)[0]


def test_reference_normal_system_matches_a_dense_restatement():
    """A, gb, diag and the structural pattern on a tiny problem, against dense numpy: a zero weight keeps its pattern entry"""
    M = 4
    idx = np.array([[0, 1, -1, -1, -1, -1, -1, -1], [1, 2, 3, -1, -1, -1, -1, -1], [2, 3, -1, -1, -1, -1, -1, -1]], np.int32)
    w = np.array([[0.5, 0.25, 0, 0, 0, 0, 0, 0], [1.0, 0.0, 0.125, 0, 0, 0, 0, 0], [0.75, 0.5, 0, 0, 0, 0, 0, 0]], np.float32)
    canon = np.zeros((3, 4), np.float32)
    live = np.array([[1, 2, 3, 0], [4, 5, 6, 0], [7, 8, 9, 0]], np.float32)
    live[2, 1] = np.nan                                  # row 2 leaves the solve: columns 2 and 3 keep only row 1's couplings
    p = Problem(M, idx, w, canon, live)
    Wd = np.zeros((2, M)); Wd[0, :2] = [0.5, 0.25]; Wd[1, 1:] = [1.0, 0.0, 0.125]
    b = live[:2, :3].astype(np.float64)
    assert np.array_equal(p.A.toarray(), Wd.T @ Wd) and np.array_equal(p.gb, Wd.T @ b)
    assert p.nnz == 4 + 9 - 1                            # {0,1}^2 and {1,2,3}^2 share (1,1)
    assert p.referenced.tolist() == [True, True, True, True] and p.supported.tolist() == [True, True, False, True] and p.nvalid == 2
    x = np.arange(12, dtype=np.float64).reshape(M, 3) * 0.1
    assert p.energy(x) == pytest.approx(0.5 * ((b - Wd @ x) ** 2).sum(), rel=1e-15)


def _ell_of(prob, cap=16):
    """the reference's own system in the solver's read-back layout"""
    M = prob.M
    A = prob.pattern.copy().astype(np.float64)
    A.data[:] = 0.0
    A = (A + prob.A).tocsr()                             # the full pattern, with its exact zeros
    A.sort_indices()
    rownnz = np.diff(A.indptr).astype(np.int32)
    col = np.zeros(cap * M, np.int32); val = np.zeros(cap * M)
    for i in range(M):
        for e, k in enumerate(range(A.indptr[i], A.indptr[i + 1])):
            col[e * M + i] = A.indices[k]; val[e * M + i] = A.data[k]
    return rownnz, col, val, prob.gb.T.reshape(-1).copy(), prob.diag.copy()


def test_ell_compare_accepts_the_reference_and_rejects_small_faults(orc):
    case = sc.make_case("m255-flat")
    idx, w = _oracle_weights(orc, case["nodes"], case["canon"], case["live"])
    w[3, 2] = 0.0                                        # an underflowed weight: a structural entry whose value may be 0
    prob = Problem(case["M"], idx, w, case["canon"], case["live"])
    rownnz, col, val, gb, diag = _ell_of(prob, cap=int(np.diff(prob.pattern.indptr).max()) + 2)
    assert ell_compare(prob, rownnz, col, val, gb, diag, tiles=False) == []
    M = prob.M
    v2 = val.copy(); v2[M + 7] *= 1 + 1e-9               # one entry off in its 9th digit
    assert ell_compare(prob, rownnz, col, v2, gb, diag, tiles=False)
    g2 = gb.copy(); g2[2 * M + 9] += 1e-9 * prob.gb_scale[9, 2] + 1e-300
    assert ell_compare(prob, rownnz, col, val, g2, diag, tiles=False)
    r2 = rownnz.copy(); r2[11] -= 1                       # the last entry of a row dropped
    assert ell_compare(prob, r2, col, val, gb, diag, tiles=False)
    assert ell_compare(prob, r2, col, val, gb, diag, tiles=True)      # ... not a zero: wrong on the tile path too
    c2 = col.copy(); c2[0 * M + 4], c2[1 * M + 4] = col[1 * M + 4], col[0 * M + 4]
    assert ell_compare(prob, rownnz, c2, val, gb, diag, tiles=False)  # columns out of order
