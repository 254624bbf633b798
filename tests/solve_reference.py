"""Float64 reference of the data-term solve (df_solve_data_term), numpy and scipy only.

The data term is linear in the node translations t_k: the residual of vertex v is r_v = b_v - sum_k w_vk t_k with
b_v = live_v - canon_v, so with the N x M weight matrix W the energy is

    E(x) = 1/2 |b - W x|^2 = 1/2 |b|^2 - x.(W^T b) + 1/2 x^T (W^T W) x        (three right-hand sides, one per axis)

and everything the solver assembles (A = W^T W, gb = W^T b, diag A, the non-zero pattern of A) and everything it reports (the energy
before and after) can be recomputed here exactly, or to double rounding, from the neighbour indices and weights of each vertex.  The
minimiser comes from a sparse direct solve of the reduced normal equations, independent of the LM / PCG iteration the kernels run.

Conventions follow the solver: a row (vertex) enters when neither canon nor live has a NaN in x, y, z; b is formed in float32 as
solve_prepare_kernel forms it; neighbour slots with index -1 (fewer nodes than neighbours) carry nothing; a column (node) that no valid
row references has no support and keeps its starting translation.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla
from scipy.spatial import cKDTree

NODE_STRIDE = 12


def valid_rows(canon, live):
    c = np.asarray(canon, np.float32)[:, :3]
    l = np.asarray(live, np.float32)[:, :3]
    return ~(np.isnan(c).any(1) | np.isnan(l).any(1))


def rhs(canon, live, valid):
    """b = float32(live - canon) on the valid rows (N_valid x 3, float64 holding float32 values)"""
    c = np.asarray(canon, np.float32)[valid, :3]
    l = np.asarray(live, np.float32)[valid, :3]
    return (l - c).astype(np.float64)


class Problem:
    """The linear least-squares problem of one solve: W (N_valid x M), b (N_valid x 3)."""

    def __init__(self, M, idx, w, canon, live):
        idx = np.asarray(idx, np.int64).reshape(-1, 8)
        w = np.asarray(w, np.float32).reshape(-1, 8)
        self.M = M
        self.valid = valid_rows(canon, live)
        self.nvalid = int(self.valid.sum())
        iv, wv = idx[self.valid], w[self.valid].astype(np.float64)
        rows = np.repeat(np.arange(self.nvalid), 8).reshape(-1, 8)
        keep = iv >= 0
        # structure (every referenced neighbour, whatever its weight) and values are kept apart: a weight may underflow to 0
        self.S = sp.csr_matrix((np.ones(int(keep.sum())), (rows[keep], iv[keep])), shape=(self.nvalid, M))
        self.W = sp.csr_matrix((wv[keep], (rows[keep], iv[keep])), shape=(self.nvalid, M))
        self.b = rhs(canon, live, self.valid)
        self.A = (self.W.T @ self.W).tocsr()
        self.A.sort_indices()
        self.gb = np.asarray(self.W.T @ self.b)                        # M x 3
        self.diag = self.A.diagonal()
        pattern = (self.S.T @ self.S).tocsr()
        pattern.sort_indices()
        self.pattern = pattern
        self.nnz = int(pattern.nnz)
        self.referenced = np.asarray(self.S.sum(0)).ravel() > 0      # some valid row lists the node
        self.supported = self.diag > 0                               # ... with a weight that did not underflow: the column can move
        absW = abs(self.W)
        self.gb_scale = np.asarray(absW.T @ np.abs(self.b))            # sum_v |w_vi| |b_v|: the size of the terms gb_i sums
        self.half_b2 = 0.5 * float((self.b ** 2).sum())

    def energy(self, x):
        """E(x) = 1/2 |b - W x|^2, x: M x 3"""
        r = self.b - self.W @ np.asarray(x, np.float64)
        return 0.5 * float((r ** 2).sum())

    def gradient(self, x):
        return self.A @ np.asarray(x, np.float64) - self.gb

    def minimiser(self, x0):
        """argmin E with the columns that have no support held at x0 (the reduced system is solved directly)"""
        x = np.array(x0, np.float64, copy=True)
        s = np.flatnonzero(self.supported)
        if len(s):
            Ar = self.A[s][:, s].tocsc()
            x[s] = spla.spsolve(Ar, self.gb[s]).reshape(len(s), 3)
        return x


def node_translations(nodes):
    """t = 2 dual conj(rot) of every 12-float node (rotation normalised), in float64: M x 3"""
    n = np.asarray(nodes, np.float64).reshape(-1, NODE_STRIDE)
    r = n[:, 3:7] / np.linalg.norm(n[:, 3:7], axis=1, keepdims=True)
    d = n[:, 7:11]
    cw, cx, cy, cz = r[:, 0], -r[:, 1], -r[:, 2], -r[:, 3]
    aw, ax, ay, az = 2 * d[:, 0], 2 * d[:, 1], 2 * d[:, 2], 2 * d[:, 3]
    tx = aw * cx + ax * cw + ay * cz - az * cy
    ty = aw * cy - ax * cz + ay * cw + az * cx
    tz = aw * cz + ax * cy - ay * cx + az * cw
    return np.stack([tx, ty, tz], 1)


def encode_nodes(pos, rot, t, weight):
    """12-float nodes: position, unit rotation (w, x, y, z), dual = 1/2 (0, t) rot, weight -- in float64, rounded once to float32"""
    pos = np.asarray(pos, np.float64); rot = np.asarray(rot, np.float64); t = np.asarray(t, np.float64)
    rot = rot / np.linalg.norm(rot, axis=1, keepdims=True)
    rw, rx, ry, rz = rot.T
    tx, ty, tz = 0.5 * t.T
    dual = np.stack([-tx * rx - ty * ry - tz * rz, tx * rw + ty * rz - tz * ry, -tx * rz + ty * rw + tz * rx, tx * ry - ty * rx + tz * rw], 1)
    n = np.zeros((len(pos), NODE_STRIDE), np.float32)
    n[:, 0:3] = pos; n[:, 3:7] = rot; n[:, 7:11] = dual + 0.0; n[:, 11] = weight        # (+ 0.0: a zero translation encodes as +0, not -0)
    return n


def knn8_check(nodes, canon, idx, w, gap=1e-4, w_atol=2e-6):
    """Independent 8-NN of the canonical vertices (cKDTree, float64) against the solver's neighbour indices / weights.

    Index sets are compared where the 8th and 9th distances are clearly apart (relative gap > `gap`: a float32 distance may order a
    closer pair either way); weights exp(-d^2 / (2 r^2)) within `w_atol` (float32 distances and the kernel's exp).  With M < 8 nodes the
    slots past M hold -1; a row whose canonical vertex has a NaN holds -1 everywhere.  Returns (failures as (row, what), rows compared)."""
    n = np.asarray(nodes, np.float64).reshape(-1, NODE_STRIDE)
    M = len(n)
    c = np.asarray(canon, np.float64)[:, :3]
    idx = np.asarray(idx, np.int64).reshape(-1, 8)
    w = np.asarray(w, np.float64).reshape(-1, 8)
    ok_c = ~np.isnan(c).any(1)
    kk = min(8, M)
    fails = [(int(v), "row without a query has neighbours") for v in np.flatnonzero(~ok_c & (idx != -1).any(1))]
    rows = np.flatnonzero(ok_c)
    got = idx[rows]
    bad_slots = (got[:, :kk] < 0).any(1) | (got[:, kk:] != -1).any(1)
    fails += [(int(v), "empty / extra slots") for v in rows[bad_slots]]
    k = min(9, M)
    d, nb = cKDTree(n[:, :3]).query(c[rows], k=k)
    d = d.reshape(-1, k); nb = nb.reshape(-1, k)
    clear = (d[:, 8] - d[:, 7] > gap * np.maximum(d[:, 8], 1e-12)) if M > 8 else np.ones(len(rows), bool)
    clear &= ~bad_slots
    same = np.all(np.sort(got[:, :kk], 1) == np.sort(nb[:, :kk], 1), 1)
    fails += [(int(v), "neighbour set") for v in rows[clear & ~same]]
    chk = ~bad_slots
    g = np.maximum(got[chk, :kk], 0)
    d2 = ((n[g, :3] - c[rows[chk], None, :]) ** 2).sum(-1)
    want = np.exp(-d2 / (2.0 * n[g, 11] ** 2))
    werr = np.abs(want - w[rows[chk], :kk]).max(1)
    fails += [(int(v), "weights") for v in rows[chk][werr > w_atol]]
    return fails, int(clear.sum())


def decode_bound(prob, x, rel=2.0 ** -21):
    """how far E can move when x is perturbed by a float32 rounding of the node encoding: sum |dE/dx| |dx| + 1/2 dx^T A dx with
    |dx| <= rel * |x_k|_inf on every component of node k (a float32 quaternion product and its inverse: a few ulp of the largest component)"""
    x = np.asarray(x, np.float64)
    dx = np.repeat(rel * np.abs(x).max(1, keepdims=True), 3, 1)
    g = np.abs(prob.gradient(x))
    return float((g * dx).sum() + 0.5 * (dx * (abs(prob.A) @ dx)).sum())


def ell_compare(prob, rownnz, col, val, gb, diag, tiles):
    """The read-back of the assembled system (df_solve_normal_system) against the float64 one; returns a list of failures.

    Per-entry assembly: the stored pattern is A's structural pattern (every pair of nodes that share a valid row).  Tile records drop an
    entry whose products are all exact zeros (underflowed weights), so there the stored pattern is a subset and every dropped entry must be
    0 in float64.  Values: products of two float32 are exact in double and every term of A is >= 0, so a row agrees to double rounding of
    its largest entry; gb's terms have both signs and are bounded by sum |w| |b|."""
    M = prob.M
    fails = []
    rownnz = np.asarray(rownnz, np.int64)
    if rownnz.min(initial=0) < 0 or rownnz.max(initial=0) > len(col) // M:
        return [("rownnz out of range", int(rownnz.min()), int(rownnz.max()))]
    cap = len(col) // M
    cols = np.asarray(col, np.int64).reshape(cap, M).T
    vals = np.asarray(val, np.float64).reshape(cap, M).T
    slots = np.arange(cap)[None, :] < rownnz[:, None]
    descending = slots[:, 1:] & (np.diff(cols, axis=1) <= 0)
    if descending.any():
        return [("columns not strictly ascending", int(descending.any(1).sum()))]
    if np.any(slots & ((cols < 0) | (cols >= M))):
        return fails + [("column index out of range", None)]
    indptr = np.concatenate([[0], np.cumsum(rownnz)])
    got = sp.csr_matrix((vals[slots], cols[slots], indptr), shape=(M, M))
    gs = sp.csr_matrix((np.ones(int(rownnz.sum()), np.int8), cols[slots], indptr), shape=(M, M))
    ps = prob.pattern.astype(bool).astype(np.int8)
    if not tiles:
        if not np.array_equal(rownnz, np.diff(prob.pattern.indptr)):
            fails.append(("row lengths differ from the pattern", int(np.sum(rownnz != np.diff(prob.pattern.indptr)))))
        elif not np.array_equal(cols[slots], prob.pattern.indices):
            fails.append(("columns differ from the pattern", None))
    else:
        outside = gs - gs.multiply(ps)
        outside.eliminate_zeros()
        if outside.nnz:
            fails.append(("entries outside the pattern", int(outside.nnz)))
        dropped = ps - ps.multiply(gs)
        dropped.eliminate_zeros()
        if dropped.nnz and abs(prob.A.multiply(dropped)).max() != 0:
            fails.append(("a dropped entry is not zero", float(abs(prob.A.multiply(dropped)).max())))
    rowmax = np.asarray(abs(prob.A).max(1).todense()).ravel()
    err = np.asarray(abs(got - prob.A).max(1).todense()).ravel()
    if np.any(err > 1e-12 * rowmax):
        worst = err / np.maximum(rowmax, 1e-300)
        fails.append(("A values", float(worst.max()), int(np.argmax(worst))))
    egb = np.abs(np.asarray(gb, np.float64).reshape(3, M).T - prob.gb)
    if np.any(egb > 1e-12 * prob.gb_scale):
        fails.append(("gb", float(np.max(egb / np.maximum(prob.gb_scale, 1e-300)))))
    d = np.asarray(diag, np.float64)
    if np.any(np.abs(d - prob.diag) > 1e-12 * np.abs(prob.diag)):
        fails.append(("diag", float(np.max(np.abs(d - prob.diag) / np.maximum(np.abs(prob.diag), 1e-300)))))
    return fails


def consistent_live(nodes, canon, t_true):
    """live = canon + sum_k w_vk t*_k with the float64 8-NN weights: data a translation field reproduces (up to float32 rounding)"""
    n = np.asarray(nodes, np.float64).reshape(-1, NODE_STRIDE)
    c = np.asarray(canon, np.float64)
    live = np.array(c, np.float32, copy=True)
    ok = ~np.isnan(c[:, :3]).any(1)
    kk = min(8, len(n))
    d, nb = cKDTree(n[:, :3]).query(c[ok, :3], k=kk)
    d = d.reshape(-1, kk); nb = nb.reshape(-1, kk)
    wts = np.exp(-d ** 2 / (2.0 * n[nb, 11] ** 2))
    live[ok, :3] = (c[ok, :3] + np.einsum("vk,vkd->vd", wts, np.asarray(t_true, np.float64)[nb])).astype(np.float32)
    return live


def rel_gap(prob, x, x0, xmin):
    """(E(x) - E_min) / (E(x0) - E_min): the share of the reducible energy a solve left"""
    e0, em = prob.energy(x0), prob.energy(xmin)
    return (prob.energy(x) - em) / max(e0 - em, 1e-300)


