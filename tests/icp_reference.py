"""Float64 reference of the projective ICP's two kernels (csrc/icp.cu), numpy and scipy only.

Sums.  Each inlier pixel contributes a 7-float row r (the oracle exports it, oracle/orc_icp.c orc_icp_rows: its u and v use fmaf, which
numpy cannot restate); icp_accumulate_kernel forms the 27 products r_i * r_j (i = 0..5, j = i..6) in float32 as separate multiplies
(the library is built with -fmad=false), so sums64 forms exactly the same float32 products and adds them in float64.

How far the kernel's sum S of one entry may lie from that float64 sum S64 (sum_bound).  With u = 2^-24 and P = sum |p| over the pixels:
  - thread stage: a thread adds its k <= k_max products one after the other in float.  A running sum s_m = s_{m-1} + p_m is rounded
    with an error <= u |s_m| <= u * (sum of the thread's |p|), and the first addition (0 + p_1) is exact: <= (k_max - 1) u P_thread;
  - warp stage: the 32 thread sums are added by a 5-level butterfly in float.  Every level rounds each node once, with an error <= u
    times the |p| below that node, so <= 5 u P_warp over the tree;
  - the terms above were bounded with the exact partial sums; the rounded ones are larger by at most a factor (1 + k_max u)^2, and the
    two extra units in (k_max + 6) u P cover that with room to spare for every k_max < 2^20;
  - double stages: each block adds its <= 24 warp results in order, the solve or reduce kernel adds <= 160 rows per lane in order and
    then in a 5-level double butterfly, and numpy's pairwise float64 sum over at most 2^22 pixels errs by at most 23 units: all of it
    is below 2^-47 P (64 units of 2^-53).
Hence |S - S64| <= (k_max + 6) 2^-24 P + 2^-47 P, entry by entry (P = abs64 of that entry).

Step.  step64 restates the reference's host step (projective_icp.cpp:195-209) without the oracle's Jacobi code: the sums are rounded to
float, A and b unpacked, the LU determinant gate applied (|det| < 1e-15 or NaN fails), r solved with a pseudo-inverse from
numpy.linalg.eigh (eigenvalues with |w| <= 6 DBL_EPSILON wmax dropped, the threshold cv::solve(DECOMP_SVD) and the device use; blocks
of A that exact zeros decouple are decomposed apart, as the device's Jacobi keeps them, so that a decoupled direction is solved exactly
and its condition does not loosen the bar of the others), then
Rodrigues as opencv2/core/affine.hpp evaluates it (double on float inputs, cast to float) and T <- Tinc T in float32 in the kernel's
operation order.  It also predicts which branch icp_solve_kernel takes: the Cholesky fast path (chol6_solve, pivot d > 1e-13 dmax) or
the LU gate and the eigen pseudo-inverse.
"""
from __future__ import annotations

import math

import numpy as np

U32 = 2.0 ** -24
EPS64 = np.finfo(np.float64).eps                       # DBL_EPSILON
NUM_SMS = 132                                           # DF_NUM_SMS: one partial row per SM at most
RED_ROWS = 160                                          # rows the solve tail stages per pass
PAIRS = [(i, j) for i in range(6) for j in range(i, 7)]
PI = np.array([i for i, _ in PAIRS])
PJ = np.array([j for _, j in PAIRS])
DET_MIN = 1e-15                                         # projective_icp.cpp:197-203
CHOL_PIVOT = 1e-13                                      # chol6_solve's pivot rule
PINV_DROP = 6 * EPS64                                   # eigenvalues with |w| <= PINV_DROP wmax carry nothing
BRANCHES = ("chol", "chol→det-fail", "pinv-kept", "pinv-dropped", "det0/NaN-fail")


# ------------------------------------------------------------------ sums -----------------------------------------------------------------
def products(rows, match):
    """the float32 products r_i * r_j of every inlier (match >= 0), n x 27 in the sums' order"""
    r = np.asarray(rows, np.float32).reshape(-1, 7)[np.asarray(match).reshape(-1) >= 0]
    return r[:, PI] * r[:, PJ]


def sums64(rows, match):
    """(S64, abs64, inliers): the 27 sums of the float32 products in float64, the per-entry sum of |p|, and the inlier count.  An accepted
    row may hold NaN (a NaN previous normal passes the cosine test): match, not the row, says which pixels are inliers."""
    p = products(rows, match).astype(np.float64)
    return p.sum(0), np.abs(p).sum(0), len(p)


def launch_shape(cols, rows):
    """(NT, blocks, k_max) of icp_accumulate_kernel (launch_accumulate): 768-thread blocks on every SM from 132 x 768 pixels on, else
    256-thread blocks, one per 256 pixels up to one per SM.  k_max: pixels of the busiest thread."""
    npix = cols * rows
    if npix >= NUM_SMS * 768:
        nt, blocks = 768, NUM_SMS
    else:
        nt, blocks = 256, max(1, min(-(-npix // 256), NUM_SMS))
    return nt, blocks, max(1, -(-npix // (blocks * nt)))


def sum_bound(shape, abs64):
    """per-entry bar on |S_gpu - S64| for a launch of `shape` = launch_shape(...) (derivation in the module docstring)"""
    k_max = shape[2]
    return ((k_max + 6) * U32 + 2.0 ** -47) * np.asarray(abs64, np.float64)


def fixed_order_sum(table):
    """the solve tail's sum of a partials table (reduce_partials, one pass of <= 160 rows): lane l of the entry's warp adds rows l, l + 32,
    ... in order, then a 5-level xor butterfly; every step a double addition, so this is the kernel's result bit for bit"""
    t = np.asarray(table, np.float64).reshape(-1, 27)
    assert 1 <= len(t) <= RED_ROWS
    out = np.empty(27)
    for s in range(27):
        v = [0.0] * 32
        for lane in range(32):
            for b in range(lane, len(t), 32):
                v[lane] += float(t[b, s])
        for o in (16, 8, 4, 2, 1):
            v = [v[lane] + v[lane ^ o] for lane in range(32)]
        out[s] = v[0]
    return out


def sensitivity(rows, match, bar):
    """min over inliers of max_e |p_e| / bar_e: above 2, dropping or doubling any one correspondence moves some sum by more than twice its
    bar, so a kernel that does either cannot stay within the bar"""
    p = np.abs(products(rows, match).astype(np.float64))
    if not len(p):
        return math.inf
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(bar > 0, p / bar, np.where(p > 0, np.inf, 0.0))
    return float(q.max(1).min())


# ------------------------------------------------------------------ step -----------------------------------------------------------------
def unpack(sums27):
    """A (6 x 6, symmetric) and b from the 27 sums rounded to float, as the reference's float buffer holds them"""
    f = np.asarray(sums27, np.float64).astype(np.float32).astype(np.float64)
    A, b = np.zeros((6, 6)), np.zeros(6)
    for k, (i, j) in enumerate(PAIRS):
        if j == 6:
            b[i] = f[k]
        else:
            A[i, j] = A[j, i] = f[k]
    return A, b


def chol_accepts(A):
    """(accepted, det, pivot margin): chol6_solve's pivot rule, every pivot d > 1e-13 max|A_ii|, and det = (prod L_jj)^2.  The margin is
    how far the pivots up to the first refused one lie from the threshold, in units of their rounding error (eps64 times the sum of
    |A_jj| and the squares subtracted from it): above 1, the device (rsqrt in place of sqrt and division) decides as this does."""
    dmax = float(np.max(np.abs(np.diag(A))))
    L = np.zeros((6, 6))
    ok, dprod, margin = True, 1.0, math.inf
    for j in range(6):
        d = float(A[j, j])
        scale = abs(d)
        for k in range(j):
            d -= L[j, k] * L[j, k]
            scale += L[j, k] * L[j, k]
        thr = dmax * CHOL_PIVOT
        if ok and thr > 0:
            margin = min(margin, abs(d - thr) / (EPS64 * max(scale, thr)))
        if not d > thr:
            ok, d = False, 1.0
        L[j, j] = math.sqrt(d)
        dprod *= L[j, j]
        for i in range(j + 1, 6):
            s = float(A[i, j])
            for k in range(j):
                s -= L[i, k] * L[j, k]
            L[i, j] = s / L[j, j]
    return ok, dprod * dprod, margin


def det_lu(A):
    return float(np.linalg.det(A)) if np.all(np.isfinite(A)) else math.nan


def blocks(A):
    """the index sets of A's decoupled blocks: connected components of its exactly non-zero off-diagonal entries.  No rotation of
    the device's Jacobi ever couples two of them (a rotation of (p, q) leaves an entry that is exactly zero in both columns exactly zero),
    nor does its Cholesky; so each block is solved on its own, to the accuracy its own condition allows."""
    n, seen, out = len(A), set(), []
    for i in range(n):
        if i in seen:
            continue
        comp, stack = [], [i]
        seen.add(i)
        while stack:
            j = stack.pop()
            comp.append(j)
            for k in range(n):
                if k not in seen and k != j and A[j, k] != 0:
                    seen.add(k)
                    stack.append(k)
        out.append(sorted(comp))
    return out


def pinv_solve(A, b):
    """(r, kappa_eff, dropped count, every eigenvalue): the symmetric pseudo-inverse solve from numpy.linalg.eigh, block by block.  The
    drop threshold 6 DBL_EPSILON wmax uses the largest |eigenvalue| of all of A, as the device's does; kappa_eff is the largest over the
    blocks of (block's largest |w|) / (block's smallest kept |w|), the factor by which eigh and the device's solve may disagree."""
    parts = [(ix, *np.linalg.eigh(A[np.ix_(ix, ix)])) for ix in blocks(A)]
    w_all = np.concatenate([w for _, w, _ in parts])
    thr = PINV_DROP * float(np.abs(w_all).max())
    r, kappa, dropped = np.zeros(len(b)), 1.0, 0
    for ix, w, V in parts:
        keep = np.abs(w) > thr
        dropped += int((~keep).sum())
        if keep.any():
            r[ix] = V[:, keep] @ ((V[:, keep].T @ b[ix]) / w[keep])
            kappa = max(kappa, float(np.abs(w).max() / np.abs(w[keep]).min()))
    return r, kappa, dropped, w_all


def rodrigues(rf):
    """cv::Affine3f(rvec, t).rotation(): Rodrigues in double on the float rotation vector, cast to float (opencv2/core/affine.hpp)"""
    rf = np.asarray(rf, np.float32)
    theta = math.sqrt(float(rf[0]) * float(rf[0]) + float(rf[1]) * float(rf[1]) + float(rf[2]) * float(rf[2]))
    if theta < EPS64:
        return np.eye(3, dtype=np.float32)
    c, s = math.cos(theta), math.sin(theta)
    c1, itheta = 1.0 - c, 1.0 / theta
    rx, ry, rz = (np.float32(float(rf[i]) * itheta) for i in range(3))
    rrt = [rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz]
    zero = np.float32(0)
    r_x = [zero, -rz, ry, rz, zero, -rx, -ry, rx, zero]
    return np.array([np.float32(c * (1.0 if i % 4 == 0 else 0.0) + c1 * float(rrt[i]) + s * float(r_x[i])) for i in range(9)],
                    np.float32).reshape(3, 3)


def compose(Rinc, rf, T_in):
    """T <- Tinc * T in float32, in icp_compose_pose's order: ((a0 b0 + a1 b1) + a2 b2) (+ t_inc)"""
    R_in, t_in = (np.asarray(x, np.float32) for x in T_in)
    R_in = R_in.reshape(3, 3)
    Rn, tn = np.empty((3, 3), np.float32), np.empty(3, np.float32)
    for i in range(3):
        for j in range(3):
            Rn[i, j] = Rinc[i, 0] * R_in[0, j] + Rinc[i, 1] * R_in[1, j] + Rinc[i, 2] * R_in[2, j]
        tn[i] = Rinc[i, 0] * t_in[0] + Rinc[i, 1] * t_in[1] + Rinc[i, 2] * t_in[2] + np.float32(rf[3 + i])
    return Rn, tn


class Step:
    """One reference step: ok, T (R, t), the branch the device rule takes on these sums (predicted here: the device reports only ok and
    T), kappa_eff, the T bar and the decision margins.  margins["det"] and margins["eig"] are relative distances of |det| and of every
    |eigenvalue| from their thresholds; pivot_margin is the Cholesky pivots' distance from theirs in rounding units (chol_accepts)."""

    def __init__(self, sums27, T_in, c_kappa=8.0):
        A, b = unpack(sums27)
        R_in, t_in = (np.asarray(x, np.float32) for x in T_in)
        self.T_in = (R_in.reshape(3, 3), t_in.reshape(3))
        self.A, self.b = A, b
        chol_ok, _, self.pivot_margin = chol_accepts(A) if np.all(np.isfinite(A)) else (False, math.nan, math.inf)
        self.det = det_lu(A)
        self.ok = math.isfinite(self.det) and abs(self.det) >= DET_MIN
        self.kappa, self.dropped, self.r = math.nan, 0, None
        self.margins = {}
        if math.isfinite(self.det) and self.det != 0:
            self.margins["det"] = abs(abs(self.det) / DET_MIN - 1.0)
        if not self.ok:
            self.branch = "chol→det-fail" if chol_ok else "det0/NaN-fail"
            self.T = self.T_in
            self.bar = (np.zeros((3, 3)), np.zeros(3))
            return
        r, self.kappa, self.dropped, w = pinv_solve(A, b)
        wmax = float(np.abs(w).max())
        self.margins["eig"] = float(np.min(np.abs(np.abs(w) / (PINV_DROP * wmax) - 1.0)))
        self.branch = "chol" if chol_ok else ("pinv-dropped" if self.dropped else "pinv-kept")
        self.r = r
        rf = r.astype(np.float32)
        Rinc = rodrigues(rf[:3])
        self.T = self.pose_of(r)
        # the bar: a few float ulps of what each entry sums (a float rounding of r or of Rinc that flips moves T by about that much),
        # plus the distance between the device's solve (Cholesky, or Jacobi) and eigh, c kappa_eff eps64 |r|, carried to T
        R0, t0 = self.T_in
        magR = np.abs(Rinc).astype(np.float64) @ np.abs(R0).astype(np.float64)
        magt = np.abs(Rinc).astype(np.float64) @ np.abs(t0).astype(np.float64) + np.abs(rf[3:]).astype(np.float64)
        ulps = 4 * 2.0 ** -23
        drift = c_kappa * self.kappa * EPS64 * float(np.linalg.norm(r)) * (1.0 + float(np.linalg.norm(t0)))
        self.bar = (ulps * np.maximum(magR, 1.0) + drift, ulps * np.maximum(magt, float(np.abs(rf).max())) + drift)

    def pose_of(self, r):
        """T <- Tinc(r) * T_in as the device composes it, for any solution r (the reference's, or a wrong one to hold against the bar)"""
        rf = np.asarray(r, np.float64).astype(np.float32)
        return compose(rodrigues(rf[:3]), rf, self.T_in)

    def within(self, T):
        """|T - T_ref| <= bar entry by entry (NaN where the reference has NaN)"""
        R, t = (np.asarray(x, np.float64) for x in T)
        Rr, tr = (np.asarray(x, np.float64) for x in self.T)
        ok = True
        for got, want, bar in ((R.reshape(3, 3), Rr, self.bar[0]), (t.reshape(3), tr, self.bar[1])):
            nan = np.isnan(want)
            ok &= bool(np.array_equal(np.isnan(got), nan)) and bool(np.all(np.abs(got - want)[~nan] <= np.asarray(bar)[~nan]))
        return ok

    def error(self, T):
        """max over entries of |T - T_ref| / bar (0 where both are NaN)"""
        R, t = (np.asarray(x, np.float64) for x in T)
        e = np.concatenate([np.abs(R.reshape(9) - np.asarray(self.T[0], np.float64).reshape(9)) / np.maximum(self.bar[0].reshape(9), 1e-300),
                            np.abs(t.reshape(3) - np.asarray(self.T[1], np.float64)) / np.maximum(self.bar[1], 1e-300)])
        return float(np.nanmax(e)) if not np.all(np.isnan(e)) else 0.0


def step64(sums27, T_in):
    return Step(sums27, T_in)
