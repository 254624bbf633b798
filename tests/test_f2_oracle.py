"""CPU tests of the SURVEY 8f(2) oracle restatement (oracle/orc_reg.c): robust data term over 6-DoF node increments + regulariser.
PARITY UNPINNED by the reference (it defines the pieces and never assembles them); these tests pin the restatement to closed forms and
to the reference-behaviour solver it must reduce to."""
import numpy as np
import pytest

from scenes import node_patch, rot_y


def test_penalties_are_the_references(orc):
    """rho_T' = tukeyPenalty, rho_H = huberPenalty (optimisation.hpp:84-88,134-138): numerical derivative / value checks through the solver's
    energy: one vertex, translation pinned by a huge damping (0 GN steps -> the energy is just rho of the residual)."""
    node_pts = np.array([[0.1 * i, 0.05 * j, 1.0] for i in range(4) for j in range(3)], np.float32)
    for c, x in ((0.01, 0.004), (0.01, 0.02), (0.05, 0.03)):
        nodes = orc.make_nodes(node_pts)
        src = np.array([[0.15, 0.05, 1.0, 0]], np.float32)
        dst = src.copy(); dst[0, 0] += x
        st = orc.solve_f2(nodes, src, dst, orc.f2_params(flags=orc.F2_TUKEY, gn_iters=0, tukey_c=c))
        u = 1 - (x / c) ** 2
        want = c * c / 6 * (1 - u ** 3) if abs(x) <= c else c * c / 6
        assert abs(st[0] - want) <= 2e-5 * want + 1e-12            # (the float32 inputs round the 4 mm residual at the 1e-6 level)


def test_translation_only_reduces_to_the_data_term_solve(orc):
    """flags = 0, lambda = 0: the energy is the reference-behaviour cost (1/2 sum r^2) and the minimiser is the data-term solve's"""
    rng = np.random.default_rng(5)
    node_pts, src = node_patch(rng)
    dst = src.copy(); dst[:, :3] += np.array([0.01, -0.004, 0.006], np.float32)
    a = orc.make_nodes(node_pts, weight=0.08); b = a.copy()
    st = orc.solve_f2(a, src, dst, orc.f2_params(flags=0, gn_iters=3, lm_mu=1e-9))
    so = orc.solve_data_term(b, src, dst, lm_iters=40)
    assert abs(st[0] - so[0]) <= 1e-9 * so[0]
    assert st[1] <= so[1] * (1 + 1e-3) + 1e-12
    ta, tb = orc.node_translations(a)[:, 1:], orc.node_translations(b)[:, 1:]
    assert np.abs(ta - tb).max() < 2e-3 * np.abs(tb).max()
    assert np.array_equal(a[:, 3:7], b[:, 3:7])                      # rotations untouched


def test_twist_explains_a_rotation_that_translations_cannot(orc):
    rng = np.random.default_rng(3)
    node_pts, src = node_patch(rng)
    dst = src.copy(); dst[:, :3] = (src[:, :3] @ rot_y(4.0).T + np.array([0.01, 0, 0.005])).astype(np.float32)
    e = {}
    for flags in (0, orc.F2_TWIST):
        nodes = orc.make_nodes(node_pts, weight=0.08)
        st = orc.solve_f2(nodes, src, dst, orc.f2_params(flags=flags, gn_iters=6))
        assert all(st[8 + i + 1] <= st[8 + i] * (1 + 1e-9) for i in range(6))          # monotone
        e[flags] = st[1]
        if flags:
            q = nodes[:, 3:7]
            ang = 2 * np.arccos(np.clip(np.abs(q[:, 0]), 0, 1))
            assert np.median(ang) == pytest.approx(np.deg2rad(4.0), rel=0.25)            # the nodes picked up the rotation
    assert e[orc.F2_TWIST] < 0.02 * e[0]


def test_tukey_rejects_outliers_and_huber_regulariser_smooths(orc):
    rng = np.random.default_rng(9)
    node_pts, src = node_patch(rng)
    true_t = np.array([0.008, 0.0, -0.004], np.float32)
    dst = src.copy(); dst[:, :3] += true_t
    out = rng.choice(len(src), len(src) // 10, replace=False)
    dst[out, :3] += rng.uniform(0.1, 0.3, (len(out), 3)).astype(np.float32)              # 10 % gross outliers
    err = {}
    for flags in (0, orc.F2_TUKEY):
        nodes = orc.make_nodes(node_pts, weight=0.08)
        orc.solve_f2(nodes, src, dst, orc.f2_params(flags=flags, gn_iters=8, tukey_c=0.05))
        w = src.copy(); n = np.zeros_like(src); n[:, 2] = 1
        orc.warp(nodes, w, n)
        inl = np.setdiff1d(np.arange(len(src)), out)
        err[flags] = np.abs(w[inl, :3] - (src[inl, :3] + true_t)).mean()
    assert err[orc.F2_TUKEY] < 0.2 * err[0]
    # regulariser: a single displaced vertex cluster drags one node; with lambda the neighbours follow (edge differences shrink)
    dst2 = src.copy()
    near = np.linalg.norm(src[:, :2] - node_pts[27, :2], axis=1) < 0.03
    dst2[near, 2] += 0.02
    d = {}
    for lam in (0.0, 20.0):
        nodes = orc.make_nodes(node_pts, weight=0.05)
        st = orc.solve_f2(nodes, src, dst2, orc.f2_params(reg_lambda=lam, flags=orc.F2_HUBER, gn_iters=6, huber_delta=1e-3))
        t = orc.node_translations(nodes)[:, 1:]
        e = orc.f2_edges(nodes, 4)
        d[lam] = np.mean([np.abs(t[i] - t[j]).max() for i in range(len(nodes)) for j in e[i] if j >= 0])
        assert st[6] == e.size
    assert d[20.0] < 0.5 * d[0.0]
